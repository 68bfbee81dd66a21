"""GPU checks of the fused SLA forwards' linear branch where its fp16 MMA operand A = T(phi * l / den) leaves fp16's range:
dead relu channels (A = inf against a KVW column of zeros), near-dead channels and a softmax outlier channel (A above 65504),
and peaked rows over long sequences (every A subnormal).  Inputs and float64 statistics: tests/sla_linear_branch_inputs.py.

Every kernel family that ends in linear_branch_store runs, in fp16 and bf16, through the module on its own block selection
(forward_with_lut): SageSparseLinearAttention at (128, 64) and, with set_served_arch("sm90"), (64, 128), at d = 128 and 64;
SparseLinearAttention at (64, 64); SparseLinearAttention at (128, 64) with the softmax map, and attn_fwd_qk16 called directly
at blkq = 128 with the elu and relu maps on that module's selection (the module sends those maps to the INT8 kernel).

Reference: float64 on the GPU from the call's 16-bit inputs: block-sparse softmax attention over the kernel's LUT (for the
INT8 kernels, scores from the call's own codes and scales, S = (q_i8 . k_i8^T) q_s k_s), plus phi(q) KVW^T / den + b with the
KVW the call was given, phi(q) from q in float64 and ksum the float64 sum of T(phi(k)) (phi(k) is rounded to T where the
reference module rounds it, in kv and ksum alike).  A float32 restatement takes the kernels' rounding points (P rounded to T
before P.V, KVW as passed, output rounded to T) but keeps A unrounded.  Bars: every output finite; per row and over the whole
output, |out - ref| <= 1.5 |restatement - ref| + |T(ref) - ref| + u_T (|P| |v| / l + |phi| |KVW|^T / den) (L2 norms;
u_T = 2^-9 for bf16, 2^-12 for fp16).  The last term bounds rounding A, and P, to T's precision: the restatement leaves A
unrounded, and its largest P is exactly 1, while under the lazy rescale the kernel's is not, so on peaked rows, whose output
rests on one or two keys, the restatement's error alone understates what one rounding of P costs.  Dead rows must also be
bit-identical to the same call with KVW = 0 (proj_l's weight zeroed) and the same bias, since A . KVW adds exact zeros
there.  At (64, 64) the module's training forward (_forward_train) must agree with the fused output, except where the
training path's own rounding points (the reference module's: phi(q) rounded to T, den summed in T) decide the fp16 answer,
which is not this test's subject: on the peaked inputs phi(q) . kvsum overflows fp16, and on softmax_outlier phi(q)_c, about
2e-9, flushes to zero in fp16 although phi(q)_c ksum_c is a large share of den."""
import math

import pytest
import torch

import sla_linear_branch_inputs as S

pytestmark = pytest.mark.gpu
F64 = torch.float64
BF16, FP16 = torch.bfloat16, torch.float16
# family: (module, (BLKQ, BLKK), head dims, served arch)
FAMILIES = {"sage_q128": ("sage", (128, 64), (128, 64), "sm100"), "sage_q64": ("sage", (64, 128), (128, 64), "sm90"),
            "sla_q64": ("sla", (64, 64), (128,), "sm100"), "sla_q128": ("sla", (128, 64), (128,), "sm100")}
PARAMS = [pytest.param(fam, name, d, id=f"{fam}-{name}-d{d}") for fam, f in FAMILIES.items() for name, c in S.CASES.items()
          for d in f[2] if d in c[5]]
DTYPES = [pytest.param(BF16, id="bf16"), pytest.param(FP16, id="fp16")]


def _module(fam, feature, ratio, d, dtype, w, bias):
    from turbodiffusion_b200.SLA import SageSparseLinearAttention, SparseLinearAttention
    kind, (blkq, blkk), _, _ = FAMILIES[fam]
    if kind == "sage":
        mod = SageSparseLinearAttention(d, ratio, feature_map=feature, use_bf16=dtype == BF16)
    else:
        mod = SparseLinearAttention(d, ratio, feature_map=feature, BLKQ=blkq, BLKK=blkk, use_bf16=dtype == BF16)
    mod = mod.cuda()
    with torch.no_grad():
        mod.proj_l.weight.copy_(w)
        mod.proj_l.bias.copy_(bias)
    return mod


def _run(fam, mod, q, k, v, feature, kvw_zero=False):
    """(out, lut, kvw, ksum, int8 prep or None) of one fused forward of family `fam`."""
    from turbodiffusion_b200.SLA.core import attn_fwd_qk16, linear_moments, project_moments, select_prep
    from turbodiffusion_b200.SLA.utils import set_served_arch
    kind, (blkq, blkk), _, arch = FAMILIES[fam]
    prev = set_served_arch(arch)
    try:
        assert mod.block_sizes(0) == (blkq, blkk)
        with torch.no_grad():
            out, sel = mod.forward_with_lut(q, k, v)
            kv, ksum = linear_moments(k, v, S.FEATURE[feature])
            kvw = project_moments(mod.proj_l.weight.detach(), kv, q.dtype)
            if fam == "sla_q128" and feature != "softmax":
                if kvw_zero:
                    kvw = torch.zeros_like(kvw)
                pb = mod.proj_l.bias.detach().float().contiguous()
                out = attn_fwd_qk16(q, k, v, sel["lut"], sel["topk"], kvw, ksum, pb, q.shape[-1] ** -0.5,
                                    feature=S.FEATURE[feature], blkq=128)
            prep = select_prep(q, k, blkq, blkk) if kind == "sage" else None
    finally:
        set_served_arch(prev)
    return out, sel["lut"], kvw, ksum, prep


def _reference(q, k, v, lut, blkq, blkk, feature, kvw, bias, prep):
    """Per row over (b, h): float64 reference, float32 restatement (rounded to T), float64 max_j phi_j l_min / den and the
    rounding bound u_T (|P| |v| / l + |phi| |KVW|^T / den).  Returns (ref [B,L,H,D] f64, restated [B,L,H,D] T, max_a [B,H,L]
    f64, r_bound [B,L,H] f64)."""
    b, l, h, d = q.shape
    dt, sm = q.dtype, d ** -0.5
    ref = torch.empty(b, l, h, d, dtype=F64, device=q.device)
    rest = torch.empty(b, l, h, d, dtype=dt, device=q.device)
    max_a = torch.empty(b, h, l, dtype=F64, device=q.device)
    r_bound = torch.empty(b, l, h, dtype=F64, device=q.device)
    u = 2.0 ** -9 if dt == BF16 else 2.0 ** -12
    nblk = S.cdiv(l, blkk)
    colblk = torch.arange(l, device=q.device) // blkk
    chunk = max(blkq, (1 << 25) // l // blkq * blkq)
    b64 = bias.to(F64)
    for bi in range(b):
        for hi in range(h):
            bm = torch.zeros(lut.shape[2], nblk, dtype=torch.bool, device=q.device).scatter_(-1, lut[bi, hi].long(), True)
            kh, vh = k[bi, :, hi], v[bi, :, hi]
            ks64 = S.phi_k(kh, feature).sum(0)
            ks32 = ks64.float()
            w64, w32 = kvw[bi, hi].to(F64), kvw[bi, hi].float()
            if prep is not None:
                ki = prep.k_i8[bi, hi].to(F64) * prep.k_scale[bi, hi][colblk].to(F64)[:, None]
            for r0 in range(0, l, chunk):
                r1 = min(l, r0 + chunk)
                rows = torch.arange(r0, r1, device=q.device)
                sel = bm[rows // blkq][:, colblk]
                qh = q[bi, r0:r1, hi]
                if prep is None:
                    s64 = qh.to(F64) @ kh.to(F64).t()
                    s32 = qh.float() @ kh.float().t()
                else:
                    qi = prep.q_i8[bi, hi, r0:r1].to(F64) * prep.q_scale[bi, hi][rows // blkq].to(F64)[:, None]
                    s64 = qi @ ki.t()
                    s32 = s64.float()
                s64 = (s64 * sm).masked_fill_(~sel, -math.inf)
                s32 = (s32 * sm).masked_fill_(~sel, -math.inf)
                p64 = torch.exp(s64 - s64.amax(-1, keepdim=True))
                l64 = p64.sum(-1)
                pq64 = S.phi(qh.to(F64), feature)
                den64 = 1e-5 + pq64 @ ks64
                ref[bi, r0:r1, hi] = (p64 @ vh.to(F64)) / l64[:, None] + (pq64 @ w64.t()) / den64[:, None] + b64
                max_a[bi, hi, r0:r1] = pq64.amax(-1) * l64 / den64
                r_bound[bi, r0:r1, hi] = u * (((p64 @ vh.to(F64).abs()) / l64[:, None]).norm(dim=-1)
                                              + ((pq64 @ w64.abs().t()) / den64[:, None]).norm(dim=-1))
                p32 = torch.exp(s32 - s32.amax(-1, keepdim=True))
                o32 = (p32.to(dt).float() @ vh.float()) / p32.sum(-1)[:, None]
                pq32 = S.phi(qh.float(), feature)
                lin32 = (pq32 @ w32.t()) / (1e-5 + pq32 @ ks32)[:, None]
                rest[bi, r0:r1, hi] = (o32 + lin32 + bias.float()).to(dt)
    return ref, rest, max_a, r_bound


def _row_norm(x):
    return x.to(F64).norm(dim=-1)


def _check_bars(out, ref, rest, r_bound, what):
    """Finite, then per row and overall |out - ref| <= 1.5 |restated - ref| + |T(ref) - ref| + r_bound."""
    bad = ~torch.isfinite(out).all(-1)
    nan_rows = int(torch.isnan(out).any(-1).sum())
    assert not bad.any(), f"{what}: {int(bad.sum())} of {bad.numel()} rows non-finite ({nan_rows} with NaN)"
    e_k, e_s = _row_norm(out.to(F64) - ref), _row_norm(rest.to(F64) - ref)
    e_o = _row_norm(ref.to(out.dtype).to(F64) - ref)
    bar = 1.5 * e_s + e_o + r_bound + 1e-30
    ratio = e_k / bar
    rel = lambda e: (e.square().sum().sqrt() / ref.norm()).item()   # noqa: E731
    print(f"{what}: rel-L2 kernel {rel(e_k):.3e} restatement {rel(e_s):.3e} output rounding {rel(e_o):.3e}; worst row "
          f"|err| / bar {ratio.max().item():.3f}")
    worst = int(ratio.flatten().argmax())
    assert (ratio <= 1).all(), (f"{what}: {int((ratio > 1).sum())} rows over the bar, worst row error {e_k.flatten()[worst]:.3e} "
                                f"against bar {bar.flatten()[worst]:.3e} (row norm {_row_norm(ref).flatten()[worst]:.3e})")
    tot = lambda e: e.square().sum().sqrt()   # noqa: E731
    assert tot(e_k) <= 1.5 * tot(e_s) + tot(e_o) + tot(r_bound), what


def _check_regime(name, max_a, dead):
    """The regime, from float64 statistics on the kernel's own selection (l_min <= the kernel's l)."""
    if name.startswith("dead_relu"):
        assert (max_a[:, :, dead] > S.FP16_MAX).all()
    elif name == "partial_dead":
        assert (max_a[:, :, dead] > S.FP16_MAX).float().mean() > 0.3
    elif name == "softmax_outlier":
        assert (max_a > S.FP16_MAX).float().mean() > 0.5
    elif name.startswith("peaked"):
        assert (max_a < S.FP16_MIN_NORMAL).float().mean() > 0.95
    else:
        assert (max_a > 2.0 ** -10).all() and (max_a * 2.0 ** 8 < 2.0 ** S.SCALE_HI).all()


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("fam,name,d", PARAMS)
def test_linear_branch_range(cuda, fam, name, d, dtype):
    q, k, v, w, bias, info = S.build(name, d, dtype)
    feature = info["feature"]
    q, k, v = (t.cuda() for t in (q, k, v))
    w, bias = w.cuda(), bias.cuda()
    mod = _module(fam, feature, info["ratio"], d, dtype, w, bias)
    out, lut, kvw, ksum, prep = _run(fam, mod, q, k, v, feature)
    assert out.dtype == dtype
    blkq, blkk = FAMILIES[fam][1]
    ref, rest, max_a, r_bound = _reference(q, k, v, lut, blkq, blkk, feature, kvw, bias, prep)
    dead = info["dead"].cuda() if info["dead"] is not None else None
    a = max_a if dead is None else max_a[:, :, dead]
    print(f"{fam} {name} d{d} {dtype}: max A (l_min) min / median / max {a.min():.3g} / {a.median():.3g} / {a.max():.3g}, "
          f"max |KVW| {kvw.abs().max().item():.4g}, max |ref| {ref.abs().max().item():.4g}")
    _check_regime(name, max_a, dead)
    assert ref.abs().max() < S.FP16_MAX / 4 and kvw.abs().max() < 2.0 ** 15
    _check_bars(out, ref, rest, r_bound, f"{fam} {name} d{d} {dtype}")

    if name.startswith("dead_relu"):
        with torch.no_grad():
            mod.proj_l.weight.zero_()
        out0 = _run(fam, mod, q, k, v, feature, kvw_zero=True)[0]
        assert torch.isfinite(out0[:, dead]).all(), "dead rows with KVW = 0 non-finite"
        same = (out[:, dead] == out0[:, dead]).all(-1)
        assert same.all(), f"{int((~same).sum())} of {same.numel()} dead rows differ from the KVW = 0 call"
        with torch.no_grad():
            mod.proj_l.weight.copy_(w)

    if fam == "sla_q64" and not name.startswith("peaked") and not (name == "softmax_outlier" and dtype == FP16):
        qg, kg, vg = (t.clone().requires_grad_() for t in (q, k, v))
        train = mod(qg, kg, vg).detach()
        assert torch.isfinite(train).all(), "training forward non-finite"
        e_t = (train.to(F64) - out.to(F64)).norm()
        e_s, e_o = (rest.to(F64) - ref).norm(), (ref.to(dtype).to(F64) - ref).norm()
        print(f"  training forward vs fused: rel-L2 {(e_t / ref.norm()).item():.3e}")
        e_r = r_bound.square().sum().sqrt()
        assert e_t <= 1.5 * e_s + 4 * e_o + e_r, ("training vs fused", e_t.item(), e_s.item(), e_o.item(), e_r.item())
