"""Host checks of the linear-branch range inputs (tests/sla_linear_branch_inputs.py): every builder reaches its regime by
float64 statistics, the exact output and KVW fit in fp16, and a torch emulation of linear_branch_store's operand
arithmetic shows what the fp16 MMA operand A = T(phi * l / den) does there (NaN, inf, subnormal loss) without a GPU, and
that bf16 and the fp16 per-row power-of-two scaling do not.

Statistics are taken over up to 256 query rows (the dead rows where there are any) on a host restatement of the (128, 64)
block selection, with l_min = sum exp2(s - max s) over the row's selected keys: the kernels' l is at least l_min and at most
2^8 times it (lazy rescale), so max A >= max phi * l_min / den.  The emulation takes l = l_min."""
import math

import pytest
import torch

import sla_linear_branch_inputs as S

F64 = torch.float64
FP16, BF16 = torch.float16, torch.bfloat16
PARAMS = [pytest.param(n, d, id=f"{n}-d{d}") for n, c in S.CASES.items() for d in c[5]]


def _sample_rows(info, l):
    if info["dead"] is not None:
        rows = torch.nonzero(info["dead"]).flatten()
        return rows[torch.linspace(0, len(rows) - 1, min(256, len(rows))).long()]
    return torch.linspace(0, l - 1, min(256, l)).long()


_CACHE = {}


def _case(name, d, dtype=FP16):
    key = (name, d, dtype)
    if key not in _CACHE:
        q, k, v, w, bias, info = S.build(name, d, dtype)
        lut = S.pooled_lut(q, k, 128, 64, info["ratio"])
        rows = _sample_rows(info, q.shape[1])
        _CACHE[key] = (q, k, v, w, bias, info, lut, rows)
    return _CACHE[key]


@pytest.mark.parametrize("name,d", PARAMS)
def test_regime_is_reached(name, d):
    q, k, v, w, bias, info, lut, rows = _case(name, d)
    st = S.stats(q, k, v, w, bias, info, lut, 128, 64, rows=rows)
    ma = st["max_a"]
    print(f"{name} d{d}: max A min / median / max {ma.min():.3g} / {ma.median():.3g} / {ma.max():.3g}, "
          f"A < 2^-14 {st['sub_frac']:.3f}, max |KVW| {st['kvw_max']:.4g}, max |out| {st['out_max']:.4g}")
    assert st["out_max"] < S.FP16_MAX / 4, "the exact output must fit in fp16"
    assert st["kvw_max"] < 2.0 ** 15, "KVW's own range is out of scope: it must fit in fp16"
    if name.startswith("dead_relu"):
        assert (ma > S.FP16_MAX).all()
        j = S.dead_channels(d)
        assert (S.kvw_exact(k, v, w, "relu")[..., j] == 0).all(), "the dead channels' KVW columns are exact zeros"
        pq = S.phi(q[:, rows].to(F64), "relu")
        off = torch.ones(d, dtype=torch.bool)
        off[j] = False
        assert (pq[..., off] == 0).all(), "dead rows are positive only on the dead channels"
    elif name == "partial_dead":
        assert (ma > S.FP16_MAX).float().mean() > 0.3
        lin = _exact_linear(q, k, v, w, "relu", rows)
        assert lin.abs().amax(-1).min() > 0.1, "the exact linear branch of the rows is of order one"
    elif name == "softmax_outlier":
        assert (ma > S.FP16_MAX).float().mean() > 0.9
    elif name.startswith("peaked"):
        assert (ma < S.FP16_MIN_NORMAL).float().mean() > 0.95 and st["sub_frac"] > 0.95, "A subnormal at l = l_min"
        assert 2.0 ** 14 <= st["kvw_max"] < 2.0 ** 15
    else:
        assert (ma > 2.0 ** -10).all() and (ma * 2.0 ** 8 < 2.0 ** S.SCALE_HI).all(), "A far from both ends of fp16"


def _exact_linear(q, k, v, w, feature, rows):
    """float64 phi(q) . KVW^T / den of rows `rows` of batch 0, head 0, with KVW = T(proj_w . kv)."""
    kvw = S.kvw_exact(k, v, w, feature).to(q.dtype)
    pq, _, den = S.head_terms(q, k, feature, 0, 0, rows)
    return (pq @ kvw[0, 0].to(F64).t()) / den[:, None]


def _emulate(name, d, dtype, rescale):
    """(emulated linear branch, exact linear branch) of the sample rows of batch 0, head 0, at dtype."""
    q, k, v, w, bias, info, lut, rows = _case(name, d, dtype)
    feature = info["feature"]
    kvw = S.kvw_exact(k, v, w, feature).to(dtype)[0, 0]
    pq, ksum, den = S.head_terms(q, k, feature, 0, 0, rows)
    l = S.row_l(q, k, lut, 128, 64, 0, 0, rows, d ** -0.5)
    got = S.emulate_linear_branch(pq, ksum, l, kvw, dtype, rescale=rescale)
    want = (pq @ kvw.to(F64).t()) / den[:, None]
    return got, want


def _row_err(got, want):
    return ((got - want).norm(dim=-1) / want.norm(dim=-1).clamp_min(1e-300))


@pytest.mark.parametrize("name", ["dead_relu_alternate", "dead_relu_warp", "dead_relu_ragged"])
def test_emulation_dead_rows(name):
    """fp16: A_J = inf against KVW[:, J] = 0 makes every dead row NaN; bf16 and the rescaled fp16 operand give exact zeros."""
    got, want = _emulate(name, 128, FP16, rescale=False)
    assert (want == 0).all()
    assert torch.isnan(got).any(-1).all(), "every dead row NaN in fp16"
    for dtype, rescale in ((BF16, False), (FP16, True)):
        got, want = _emulate(name, 128, dtype, rescale)
        assert (got == 0).all(), (dtype, rescale)


@pytest.mark.parametrize("name,d", [pytest.param(n, d, id=f"{n}-d{d}") for n in ("partial_dead", "softmax_outlier")
                                    for d in (128, 64)])
def test_emulation_overflow(name, d):
    """fp16: A above 65504 rounds to inf; bf16 and the rescaled fp16 operand stay finite and close to float64."""
    got, _ = _emulate(name, d, FP16, rescale=False)
    bad = (~torch.isfinite(got)).any(-1).float().mean().item()
    print(f"{name} d{d}: fp16 rows with a non-finite linear branch {bad:.3f}")
    assert bad > 0.2
    for dtype, rescale, bar in ((BF16, False, 2e-2), (FP16, True, 4e-3)):
        got, want = _emulate(name, d, dtype, rescale)
        err = _row_err(got, want)
        print(f"  {dtype} rescale={rescale}: row rel err median {err.median():.2e} max {err.max():.2e}")
        assert torch.isfinite(got).all() and err.max() < bar, (dtype, rescale)


@pytest.mark.parametrize("name,d", [pytest.param(n, d, id=f"{n}-d{d}") for n, c in S.CASES.items() if n.startswith("peaked")
                                    for d in c[5]])
def test_emulation_underflow(name, d):
    """Every A subnormal in fp16: the per-row error is above bf16's and 10x the rescaled operand's, which is below bf16's."""
    errs = {}
    for dtype, rescale in ((FP16, False), (BF16, False), (FP16, True)):
        got, want = _emulate(name, d, dtype, rescale)
        err = _row_err(got, want)
        errs[(dtype, rescale)] = err.median().item()
        print(f"{name} d{d} {dtype} rescale={rescale}: row rel err median {err.median():.2e} max {err.max():.2e}")
    assert errs[(FP16, False)] > 10 * errs[(FP16, True)] and errs[(FP16, False)] > 2 * errs[(BF16, False)]
    assert errs[(FP16, True)] < errs[(BF16, False)] / 4


def test_emulation_ordinary_rows_unscaled():
    """Ordinary softmax-map rows are inside the unscaled range, so the fp16 rescale leaves their arithmetic unchanged."""
    q, k, v, w, bias, info, lut, rows = _case("ordinary", 128)
    pq, ksum, _ = S.head_terms(q, k, "softmax", 0, 0, rows)
    l = S.row_l(q, k, lut, 128, 64, 0, 0, rows, 128 ** -0.5)
    kvw = S.kvw_exact(k, v, w, "softmax").to(FP16)[0, 0]
    assert torch.equal(S.emulate_linear_branch(pq, ksum, l, kvw, FP16), S.emulate_linear_branch(pq, ksum, l, kvw, FP16, True))


def test_row_shift_range():
    """The shift puts max A in [2^14, 2^15) and leaves [2^-6, 2^15) and zero rows alone."""
    a = torch.tensor([0.0, 2.0 ** -6, 1.0, 2.0 ** 15 - 1, 2.0 ** 15, 1e7, 1e-9], dtype=F64)
    sh = S.fp16_row_shift(a)
    assert sh[:4].eq(0).all()
    scaled = a[4:] * torch.exp2(sh[4:])
    assert ((scaled >= 2.0 ** 14) & (scaled < 2.0 ** 15)).all(), scaled
    assert S.fp16_row_shift(torch.tensor([1e-60], dtype=F64)).item() == 64
    assert math.isclose(S.fp16_row_shift(torch.tensor([2.0 ** 100], dtype=F64)).item(), -64)
