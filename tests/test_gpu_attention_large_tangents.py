"""GPU checks of the attention JVP, tangent and dense backward kernels where their 16-bit operands run short of range: scores
that rise slowly from one 64-key tile to the next (so the JVP kernel's unnormalised p reaches about 2^8 between lazy rescales)
along keys with a large shared component (so the score tangent S_t reaches hundreds with unit tangents), in both dtypes, at
ragged lengths, against float64.  The inputs are tests/test_attention_large_tangents_host.py's (H), which shows on the CPU that
p * S_t rounded to fp16 overflows on them unless the JVP kernel rescales such rows onto their running maximum first.

Bars are those of tests/test_gpu_dense_attention_jvp.py (DJ) and tests/test_gpu_sla_jvp.py (SJ): primal cos >= 0.999 and
rel-L2 <= 5e-3 against float64; tangent finite and rel-L2 against float64 torch.func.jvp at most 1.5x that of the float32
restatement of the kernel's rounding, plus 1e-7.  Gradients: tests/test_gpu_dense_attention_bwd.py's (DB), rel-L2 against float64
autograd at most 1.5x that of F.scaled_dot_product_attention's backward.  Each test first asserts, from float64 statistics of its
inputs, that they reach the regime it is about."""
import pytest
import torch

import test_attention_large_tangents_host as H
import test_gpu_dense_attention_bwd as DB
import test_gpu_dense_attention_jvp as DJ
import test_gpu_sla_jvp as SJ

pytestmark = pytest.mark.gpu
D, BQ, BK = 128, 128, 64
SM = D ** -0.5
BF16, FP16 = torch.bfloat16, torch.float16
DTYPES = [pytest.param(BF16, id="bf16"), pytest.param(FP16, id="fp16")]
RAMPS = ["slow", "slow-qt-along-u", "alternating"]
SHAPES = [pytest.param(1, 2, 700, 1000, id="b1h2-700x1000"), pytest.param(2, 3, 333, 1000, id="b2h3-333x1000")]
LIMIT = H.FP16_MAX / 16        # "well inside fp16 range" for the normalised |P S_t| and the exact tangent


def _ins(b, h, lq, lk, ramp, dtype, seed, scale=1.0):
    return [t.to(dtype).cuda() for t in H.ramp_inputs(b, lq, lk, h, ramp, seed, tangent_scale=scale)]


def _regime(ins, ramp, what, order=None, mask=None, limit=LIMIT):
    """asserts the inputs reach the overflow regime (fp16 statistics, whatever the dtype run) and that the exact answer is
    representable; returns the fraction of rows whose lazily rescaled p * |S_t| passes 65504"""
    over, norm, lag, _ = H.overflow_stats(ins, order, mask)
    print(f"{what}: rows with p |S_t| > 65504 {over:.3f}, max normalised |P S_t| {norm:.0f}, lag {lag:.2f}")
    assert over > (0.2 if ramp == "slow-qt-along-u" else 0.0) and norm < limit and lag > 7.0, (what, over, norm, lag)
    return over


def _nonfinite(out_t, what):
    """prints how many rows (of d values) of the tangent hold a non-finite value: the failure this file is about"""
    bad = (~torch.isfinite(out_t)).any(-1)
    print(f"{what}: {bad.sum().item()} of {bad.numel()} tangent rows non-finite")


def _check_dense(out_t, ins, what):
    _nonfinite(out_t, what)
    DJ._check_tangent(out_t, ins, what)


def _check_sparse(o, o_t, ins, mask, what):
    _nonfinite(o_t, what)
    SJ._check(o, o_t, ins, mask, what)


def _dense(q, k, v):
    from turbodiffusion_b200 import ops
    return ops.dense_attention(q, k, v)


def _module(dtype):
    """SparseLinearAttention at top-k 0.5 with proj_l zero (its initial state): o is the sparse branch's o_s and o_t its o_s_t"""
    from turbodiffusion_b200.SLA import SparseLinearAttention
    return SparseLinearAttention(D, 0.5, BLKQ=128, BLKK=64, use_bf16=dtype == BF16).cuda()


# ------------------------------------------------------------------------------------------------ dense JVP
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("ramp", RAMPS)
@pytest.mark.parametrize("b,h,lq,lk", SHAPES)
def test_dense_jvp(cuda, b, h, lq, lk, ramp, dtype):
    from turbodiffusion_b200 import ops
    ins = _ins(b, h, lq, lk, ramp, dtype, seed=lq + len(ramp))
    what = f"dense jvp {ramp} ({b}, {h}, {lq}, {lk}) {dtype}"
    _regime(ins, ramp, what)
    out, out_t = ops.dense_attention_jvp(*ins)
    want, _ = DJ.exact_f64(*ins)
    DJ._check_primal(out, want, what)
    _check_dense(out_t, ins, what)


def test_dense_jvp_tangent_scale_sweep_fp16(cuda):
    """Tangents x1 .. x64 on "slow": wherever the normalised |P S_t| and the float64 tangent fit in fp16 with a factor 2 to
    spare (here, every scale), out_t meets the bar: the operator's fp16 range is P * S_t's, not 2^8 times less."""
    from turbodiffusion_b200 import ops
    checked = []
    for scale in (1, 2, 4, 8, 16, 32, 64):
        ins = _ins(1, 2, 700, 1000, "slow", FP16, seed=5, scale=scale)
        _, norm, _, _ = H.overflow_stats(ins)
        _, want_t = DJ.exact_f64(*ins)
        if norm >= H.FP16_MAX / 2 or want_t.abs().max().item() >= H.FP16_MAX / 2:
            continue
        _, out_t = ops.dense_attention_jvp(*ins)
        _check_dense(out_t, ins, f"dense jvp fp16 tangents x{scale}")
        checked.append(scale)
    assert checked == [1, 2, 4, 8, 16, 32, 64], checked


# ------------------------------------------------------------------------------------------------ SLA JVP
def _luts(kind, b, h, l):
    nblk = SJ._nblk(l)
    if kind == "full-ascending":
        return SJ._full_lut(b, h, l)
    if kind == "ascending":
        return SJ._random_lut(b, h, l, nblk - 4, seed=l + 1, ascending=True)
    return SJ._random_lut(b, h, l, nblk - 4, seed=l + 2, tail=True)      # random order, the ragged last block in every row


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("ramp", RAMPS)
@pytest.mark.parametrize("lut_kind", ["ascending", "full-ascending", "random-order"])
def test_sla_jvp_entry_point(cuda, lut_kind, ramp, dtype):
    """tdb200_sla_attn16_jvp over ascending, full ascending and random-order LUTs, against SJ's masked float64 references"""
    b, h, l = (2, 2, 1000) if lut_kind == "ascending" else (1, 2, 1000)
    ins = _ins(b, h, l, l, ramp, dtype, seed=l + len(ramp) + len(lut_kind))
    lut = _luts(lut_kind, b, h, l)
    mask = SJ._mask(lut, l)
    what = f"sla jvp {lut_kind} {ramp} ({b}, {h}, {l}) {dtype}"
    if lut_kind != "random-order":       # random order may visit a row's largest block first: no lag to speak of
        _regime(ins, ramp, what, lut.cpu(), mask)
    o_s, o_s_t = SJ._jvp(*ins, lut)
    _check_sparse(o_s, o_s_t, ins, mask, what)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("ramp", RAMPS)
def test_sla_forward_jvp(cuda, ramp, dtype):
    """SparseLinearAttention.forward_jvp: the block map's ascending LUT; proj_l zero, so o_t is the kernel's o_s_t"""
    b, h, l = 1, 2, 1000
    ins = _ins(b, h, l, l, ramp, dtype, seed=l + len(ramp) + 7)
    mod = _module(dtype)
    mod._keep_selection = {}
    with torch.no_grad():
        o, o_t = mod.forward_jvp(*ins)
    lut = mod._keep_selection["lut"]
    mod._keep_selection = None
    mask = SJ._mask(lut, l)
    what = f"forward_jvp {ramp} {dtype}"
    _regime(ins, ramp, what, lut.cpu(), mask)
    _check_sparse(o, o_t, ins, mask, what)


# ------------------------------------------------------------------------------------------------ the tangent kernels
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("ramp", RAMPS)
def test_dense_func_jvp(cuda, ramp, dtype):
    """torch.func.jvp through ops.dense_attention: the tangent kernel from the lse forward's out and lse"""
    ins = _ins(1, 2, 700, 1000, ramp, dtype, seed=11 + len(ramp))
    what = f"dense func.jvp {ramp} {dtype}"
    _regime(ins, ramp, what)
    out, out_t = torch.func.jvp(_dense, tuple(ins[:3]), tuple(ins[3:]))
    assert torch.equal(out, _dense(*ins[:3]))
    _check_dense(out_t, ins, what)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("ramp", RAMPS)
def test_sla_func_jvp(cuda, ramp, dtype):
    """torch.func.jvp through SparseLinearAttention (proj_l zero): the sparse tangent kernel over the block map's LUT"""
    l = 1000
    ins = _ins(1, 2, l, l, ramp, dtype, seed=13 + len(ramp))
    mod = _module(dtype)
    mod._keep_selection = {}
    o, o_t = torch.func.jvp(mod, tuple(ins[:3]), tuple(ins[3:]))
    lut = mod._keep_selection["lut"]
    mod._keep_selection = None
    mask = SJ._mask(lut, l)
    what = f"sla func.jvp {ramp} {dtype}"
    _regime(ins, ramp, what, lut.cpu(), mask)
    _check_sparse(o, o_t, ins, mask, what)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("path", ["dense", "sparse"])
def test_jvp_kernel_and_tangent_kernel_agree(cuda, path, dtype):
    """On identical inputs where most rows' lazily rescaled p * S_t passes 65504, the JVP kernel's tangent
    (ops.dense_attention_jvp, forward_jvp) and the tangent kernel's (torch.func.jvp) both meet the bar."""
    l = 1000
    ins = _ins(1, 2, l, l, "slow-qt-along-u", dtype, seed=17)
    if path == "dense":
        from turbodiffusion_b200 import ops
        _regime(ins, "slow-qt-along-u", f"agree dense {dtype}")
        _, jvp_t = ops.dense_attention_jvp(*ins)
        _, tan_t = torch.func.jvp(_dense, tuple(ins[:3]), tuple(ins[3:]))
        _check_dense(jvp_t, ins, f"agree dense {dtype}: JVP kernel")
        _check_dense(tan_t, ins, f"agree dense {dtype}: tangent kernel")
    else:
        mod = _module(dtype)
        mod._keep_selection = {}
        with torch.no_grad():
            o, jvp_t = mod.forward_jvp(*ins)
        lut = mod._keep_selection["lut"]
        _, tan_t = torch.func.jvp(mod, tuple(ins[:3]), tuple(ins[3:]))
        assert torch.equal(mod._keep_selection["lut"], lut)
        mod._keep_selection = None
        mask = SJ._mask(lut, l)
        _regime(ins, "slow-qt-along-u", f"agree sparse {dtype}", lut.cpu(), mask)
        _check_sparse(o, jvp_t, ins, mask, f"agree sparse {dtype}: JVP kernel")
        _check_sparse(o, tan_t, ins, mask, f"agree sparse {dtype}: tangent kernel")
    print(f"  JVP kernel vs tangent kernel: rel-L2 {DJ._rel(jvp_t, tan_t):.2e}")


# ------------------------------------------------------------------------------------------------ dense backward
def _steep_ramp(lq, lk, h):
    """DJ's large-score construction: scores climb about 30 log2 units per 64-key tile, so every tile rescales"""
    g = torch.Generator().manual_seed(11)
    u = torch.ones(D) / D ** 0.5
    q, k, v = torch.randn(1, lq, h, D, generator=g), torch.randn(1, lk, h, D, generator=g), torch.randn(1, lk, h, D, generator=g)
    q = 8.0 * (q - (q @ u)[..., None] * u) + 4.0 * u
    k = k + (30.0 * (torch.arange(lk) // BK) / (4.0 * SM * H.LOG2E))[None, :, None, None] * u
    return q, k, v


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("scores", ["steep-ramp", "slow", "large-keys"])
def test_dense_backward_at_large_scores(cuda, scores, dtype):
    """dq, dk and dv of ops.dense_attention's training path against float64 autograd, at DB's bar, on scores whose row maxima
    reach 100 log2 units and more (lse far from 0)"""
    lq, lk, h = 700, 1000, 2
    if scores == "steep-ramp":
        q, k, v = _steep_ramp(lq, lk, h)
    else:
        q, k, v = H.ramp_inputs(1, lq, lk, h, scores, seed=23)[:3]
    d_out = torch.randn(1, lq, h, D, generator=torch.Generator().manual_seed(29))
    ins = [t.to(dtype).cuda() for t in (q, k, v, d_out)]
    s = torch.einsum("bqhd,bkhd->bhqk", ins[0].double(), ins[1].double()) * (SM * H.LOG2E)
    assert s.amax(-1).min().item() > 50, s.amax(-1).min().item()
    _, *grads = DB.ours(*ins)
    _, *want = DB.exact_f64(*ins)
    DB._check_grads(grads, DB.sdpa_grads(*ins), want, f"backward {scores} {dtype}", lk)
