"""GPU checks of the 16-bit SLA attention kernels (SparseLinearAttention's forward, forward with lse, and backward) where the
ordinary randn cases never go: large score magnitudes, which take the lazy rescale of the online softmax and, on 64-row
query blocks, the merge of two warpgroup states with different maxima; and block lists longer than a CTA's thread count
and than the key-major index's 256-wide scan.

The references are computed here, in float64 on the GPU, from the kernels' own 16-bit inputs: block-sparse softmax attention
over the LUT (dense attention when every key block is selected), its row log-sum-exp, and float64 autograd (or, at long
lengths, the closed-form backward given float64 lse and delta) for the gradients.  They share no LUT handling with the
kernels.

Bars.  Forward output: cos >= 0.9999 and rel-L2 <= 5e-3 (against the fp32 oracle's exact and Triton-rounded statements for
the fused output, against float64 for o_s).  lse: |error| <= 1e-3 + 1e-5 max|s| per row, in log2 units, s being the
row's selected scores scaled by sm_scale * log2(e).  Gradients: cos >= 0.999 and rel-L2 <= 2e-2; proj_l rel-L2 <= 2e-2.
Where a 16-bit restatement of the same computation (fp32 arithmetic on the 16-bit inputs, P rounded to the input type
before P.V) itself misses a gradient bar, the bar becomes the kernel at most 1.5x the restatement's error: peaked softmax
can put a gradient beyond what 16-bit operands resolve.  Every gradient check prints both distances."""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import td_oracle as O

import sla_backward_oracle as B

pytestmark = pytest.mark.gpu
D, BK = 128, 64
LOG2E, LN2 = 1.0 / math.log(2.0), math.log(2.0)
F64 = torch.float64
SM = D ** -0.5
BF16, FP16 = torch.bfloat16, torch.float16
DTYPES = [pytest.param(BF16, id="bf16"), pytest.param(FP16, id="fp16")]


def _cdiv(a, b):
    return (a + b - 1) // b


# ------------------------------------------------------------------------------------------------------------ references
def _stats(got, want):
    a, b = got.to(F64).flatten(), want.to(F64).flatten()
    return {"rel_l2": ((a - b).norm() / b.norm().clamp_min(1e-300)).item(),
            "cos": (torch.dot(a, b) / (a.norm() * b.norm()).clamp_min(1e-300)).item()}


def _bars(got, want, cos, rel, what):
    s = _stats(got, want)
    assert s["cos"] >= cos and s["rel_l2"] <= rel, (what, s)
    return s


def _ref_forward(q, k, v, lut, blkq, sm_scale=SM, d_o=None, entry_max=False):
    """Float64 block-sparse attention of q, k, v [B,L,H,D] (on the GPU) over `lut`, in query chunks.  Returns a dict:
    o [B,L,H,D]; lse and smax [B,H,L] in log2 units (smax = max |s| over the row's selected scores); delta [B,H,L] =
    rowsum(d_o * o) when d_o is given; with entry_max, emax [B,H,L,topk] = the maximum of s over each LUT entry's key
    block, in LUT order."""
    b, l, h, d = q.shape
    nblk = _cdiv(l, BK)
    bm = B.block_mask(lut, nblk)
    dev = q.device
    colblk = torch.arange(l, device=dev) // BK
    out = {"o": torch.empty(b, l, h, d, dtype=F64, device=dev)}
    for name in ("lse", "smax") + (("delta",) if d_o is not None else ()):
        out[name] = torch.empty(b, h, l, dtype=F64, device=dev)
    if entry_max:
        out["emax"] = torch.empty(b, h, l, lut.shape[-1], dtype=F64, device=dev)
    chunk = max(blkq, (1 << 24) // l // blkq * blkq)
    for bi in range(b):
        for hi in range(h):
            qh, kh, vh = (t[bi, :, hi].to(F64) for t in (q, k, v))
            for r0 in range(0, l, chunk):
                r1 = min(l, r0 + chunk)
                rowblk = torch.arange(r0, r1, device=dev) // blkq
                sel = bm[bi, hi][rowblk][:, colblk]
                s = ((qh[r0:r1] @ kh.t()) * (sm_scale * LOG2E)).masked_fill_(~sel, -math.inf)
                lse = torch.logsumexp(s * LN2, -1) / LN2
                out["lse"][bi, hi, r0:r1] = lse
                out["smax"][bi, hi, r0:r1] = s.abs().masked_fill_(~sel, 0.0).amax(-1)
                if entry_max:
                    blk = F.pad(s, (0, nblk * BK - l), value=-math.inf).view(r1 - r0, nblk, BK).amax(-1)
                    out["emax"][bi, hi, r0:r1] = blk.gather(-1, lut[bi, hi][rowblk].long())
                o = torch.exp2(s - lse[:, None]) @ vh
                out["o"][bi, r0:r1, hi] = o
                if d_o is not None:
                    out["delta"][bi, hi, r0:r1] = (o * d_o[bi, r0:r1, hi].to(F64)).sum(-1)
    return out


def _sparse_attention(q, k, v, lut, blkq, sm_scale=SM, p_dtype=None):
    """Differentiable block-sparse attention of [B,L,H,D] tensors over `lut` (one masked dense softmax; short sequences
    only).  p_dtype: P rounded to that type before P.V, the row sum taken from the unrounded P."""
    l = q.shape[1]
    sel = B.block_mask(lut, _cdiv(l, BK))[:, :, torch.arange(l, device=q.device) // blkq][..., torch.arange(l, device=q.device) // BK]
    qh, kh, vh = (t.transpose(1, 2) for t in (q, k, v))
    s = ((qh @ kh.transpose(-1, -2)) * sm_scale).masked_fill(~sel, -math.inf)
    e = torch.exp(s - s.amax(-1, keepdim=True).detach())
    pv = (e if p_dtype is None else e.to(p_dtype).to(e.dtype)) @ vh
    return (pv / e.sum(-1, keepdim=True)).transpose(1, 2)


def _linear_branch(q, k, v, w, bias, rdtype=None):
    """The softmax-feature linear branch and proj_l of [B,L,H,D] tensors, exact in their precision, or with rdtype at the
    reference's 16-bit rounding points (feature maps, moments and proj_l in that type)."""
    qh, kh, vh = (t.transpose(1, 2) for t in (q, k, v))
    if rdtype is None:
        pq, pk = torch.softmax(qh, -1), torch.softmax(kh, -1)
        o = (pq @ (pk.transpose(-1, -2) @ vh)) / (1e-5 + (pq * pk.sum(-2, keepdim=True)).sum(-1, keepdim=True))
        return (o @ w.t() + bias).transpose(1, 2)
    pq, pk, vd = torch.softmax(qh, -1).to(rdtype), torch.softmax(kh, -1).to(rdtype), vh.to(rdtype)
    o = (pq @ (pk.transpose(-1, -2) @ vd)) / (1e-5 + (pq * pk.sum(-2, keepdim=True)).sum(-1, keepdim=True))
    return F.linear(o, w.to(rdtype), bias.to(rdtype)).float().transpose(1, 2)


def _ref_grads(q, k, v, d_o, lut, blkq, sm_scale=SM, w=None, bias=None, rdtype=None):
    """Gradients of sum(d_o * out) for out = block-sparse attention (+ the linear branch and proj_l when w is given):
    float64 autograd, or with rdtype the 16-bit restatement (fp32 arithmetic on the 16-bit inputs, P rounded to rdtype).
    Returns [dq, dk, dv] (+ [dw, dbias])."""
    ct = F64 if rdtype is None else torch.float32
    leaves = [t.to(ct).requires_grad_() for t in (q, k, v)]
    if w is not None:
        leaves += [w.to(ct).requires_grad_(), bias.to(ct).requires_grad_()]
    o = _sparse_attention(*leaves[:3], lut, blkq, sm_scale, p_dtype=rdtype)
    if w is not None:
        o = o + _linear_branch(*leaves, rdtype=rdtype)
    (o * d_o.to(ct)).sum().backward()
    return [t.grad for t in leaves]


def _check_lse(lse, ref, what):
    """Per row: |lse - lse_ref| <= 1e-3 + 1e-5 max|s| (log2 units).  Returns the worst error and its bar."""
    err = (lse.to(F64) - ref["lse"]).abs()
    bar = 1e-3 + 1e-5 * ref["smax"]
    worst = (err - bar).argmax()
    assert (err <= bar).all(), (what, "lse rows over the bar:", int((err > bar).sum()), "worst", err.flatten()[worst].item(),
                                "bar there", bar.flatten()[worst].item())
    return err.max().item()


def _check_grad(name, got, want, restated, what, cos=0.999, rel=2e-2):
    """The gradient bar, or 1.5x the 16-bit restatement's error where the restatement itself misses that bar."""
    s, r = _stats(got, want), _stats(restated, want)
    print(f"{what} {name}: kernel rel-L2 {s['rel_l2']:.2e} cos {s['cos']:.7f} | restatement rel-L2 {r['rel_l2']:.2e} "
          f"cos {r['cos']:.7f}")
    if r["cos"] >= cos and r["rel_l2"] <= rel:
        assert s["cos"] >= cos and s["rel_l2"] <= rel, (what, name, s, "restatement", r)
    else:
        # 1 - cos grows as the square of a small error: 1.5x the restatement's error is 2.25x its 1 - cos
        assert s["rel_l2"] <= 1.5 * r["rel_l2"] and 1 - s["cos"] <= 2.25 * (1 - r["cos"]), (what, name, s, "restatement", r)


def _rescale_fraction(emax, blkq):
    """Fraction of rows whose running maximum, in the LUT order one warpgroup sees, grows by more than 8 (log2 units): every
    entry at 128-row blocks, entries j = g mod 2 for warpgroup g at 64-row blocks.  Such a row takes the lazy rescale."""
    orders = [emax] if blkq == 128 else [emax[..., 0::2], emax[..., 1::2]]
    grows = torch.zeros(emax.shape[:-1], dtype=torch.bool, device=emax.device)
    for e in orders:
        if e.shape[-1] > 1:
            run = torch.cummax(e, -1).values
            grows |= ((run[..., 1:] - run[..., :-1]) > 8).any(-1)
    return grows.float().mean().item()


# ------------------------------------------------------------------------------------------------------------ inputs
# The input builders (large-score and entry-split patterns, long lists) are sla_backward_oracle's.
SCALED, SPLIT = B.SCALED, B.SPLIT
MIN_FRACTION = {"all": 0.2, "ragged_last": 0.3, "half_warp": 0.08, "one_warp": 0.04, "split_dominant": 0.9, "split_merge": 0.9}


def _module(blkq, ratio, dtype, seed=5, **kw):
    from turbodiffusion_b200.SLA import SparseLinearAttention
    mod = SparseLinearAttention(D, ratio, BLKQ=blkq, BLKK=BK, use_bf16=dtype == BF16, **kw).cuda()
    assert mod.block_sizes(0) == (blkq, BK)
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        mod.proj_l.weight.copy_(torch.randn(D, D, generator=g) * 0.05)
        mod.proj_l.bias.copy_(torch.randn(D, generator=g) * 0.05)
    return mod


def _case(name, blkq, dtype):
    """(q, k, v on the GPU in dtype, lut or None (the module selects), ratio)."""
    if name in SPLIT:
        q, k, v, lut = B.split_case(name, blkq)
        ratio, lut = 1.0, lut.cuda()
    else:
        q, k, v, ratio = B.scaled_case(name, blkq)
        lut = None
    return [t.to(dtype).cuda() for t in (q, k, v)], lut, ratio


def _fused(mod, q, k, v, lut, blkq):
    """The fused inference forward: through the module when it selects the blocks, else attn_fwd_qk16 on `lut` with the
    module's linear-branch operands.  Returns (out, lut)."""
    from turbodiffusion_b200.SLA.core import attn_fwd_qk16, linear_moments, project_moments
    with torch.no_grad():
        if lut is None:
            out, sel = mod.forward_with_lut(q, k, v)
            return out, sel["lut"]
        kv, ksum = linear_moments(k, v, 0)
        kvw = project_moments(mod.proj_l.weight.detach(), kv, q.dtype)
        pb = mod.proj_l.bias.detach().float().contiguous()
        return attn_fwd_qk16(q, k, v, lut, lut.shape[-1], kvw, ksum, pb, SM, blkq=blkq), lut


def _direct(q, k, v, lut, blkq, sm_scale=SM, seed=1):
    from turbodiffusion_b200.SLA.core import attn_bwd_qk16, attn_fwd_qk16_lse
    topk = lut.shape[-1]
    o_s, lse = attn_fwd_qk16_lse(q, k, v, lut, topk, sm_scale, blkq=blkq)
    g = torch.Generator(device=q.device).manual_seed(seed)
    d_o = torch.randn(q.shape, generator=g, device=q.device).to(q.dtype)
    return o_s, lse, d_o, attn_bwd_qk16(q, k, v, o_s, d_o, lse, lut, topk, sm_scale, blkq=blkq)


# ------------------------------------------------------------------------------------------------------------ 1. forward
FWD = [pytest.param(128, n, id=f"q128-{n}") for n in SCALED] + [pytest.param(64, n, id=f"q64-{n}") for n in (*SCALED, *SPLIT)]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("blkq,name", FWD)
def test_large_scores_forward(cuda, blkq, name, dtype):
    """The fused inference output against the fp32 oracle (exact and Triton-rounded), and attn_fwd_qk16_lse's o_s and
    per-row lse against float64, on inputs where the lazy rescale (and at 64 rows the merge) is taken."""
    (q, k, v), lut, ratio = _case(name, blkq, dtype)
    mod = _module(blkq, ratio, dtype)
    out, lut = _fused(mod, q, k, v, lut, blkq)
    assert out.dtype == dtype and torch.isfinite(out).all()
    ref = _ref_forward(q, k, v, lut, blkq, entry_max=True)
    frac = _rescale_fraction(ref["emax"], blkq)
    assert frac > MIN_FRACTION[SCALED[name][0] if name in SCALED else name], ("rows taking the lazy rescale", frac)

    w, bias = mod.proj_l.weight.detach().cpu(), mod.proj_l.bias.detach().cpu()
    qc, kc, vc, lc = q.cpu(), k.cpu(), v.cpu(), lut.cpu()
    exact = O.sla_forward(qc, kc, vc, w, bias, ratio, blkq, BK, dtype=dtype, mode="exact", lut=lc)
    tri = O.sla_forward(qc, kc, vc, w, bias, ratio, blkq, BK, dtype=dtype, mode="triton", lut=lc)
    s_exact = _bars(out, exact.cuda(), 0.9999, 5e-3, ("fused vs exact", name))
    s_tri = _bars(out, tri.cuda(), 0.9999, 5e-3, ("fused vs triton", name))

    from turbodiffusion_b200.SLA.core import attn_fwd_qk16_lse
    o_s, lse = attn_fwd_qk16_lse(q, k, v, lut, lut.shape[-1], SM, blkq=blkq)
    s_os = _bars(o_s, ref["o"], 0.9999, 5e-3, ("o_s vs float64", name))
    worst = _check_lse(lse, ref, name)
    print(f"{name} q{blkq} {dtype}: rescale rows {frac:.3f}, fused rel-L2 {s_exact['rel_l2']:.2e} (exact) "
          f"{s_tri['rel_l2']:.2e} (triton), o_s {s_os['rel_l2']:.2e}, lse max |err| {worst:.2e} (max|s| "
          f"{ref['smax'].max().item():.0f})")


# ------------------------------------------------------------------------------------------------------------ 2. backward
BWD = [pytest.param(bq, n, id=f"q{bq}-{n}") for bq in (128, 64) for n in ("all_x8", "ragged_last", "split_dominant")]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("blkq,name", BWD)
def test_large_scores_backward(cuda, blkq, name, dtype):
    """attn_bwd_qk16's dq, dk, dv against float64 autograd (its lse and delta are float64's, not the kernel's); where the
    module selects the blocks, also the module's gradients (forward_with_lut + backward, proj_l included)."""
    (q, k, v), lut, ratio = _case(name, blkq, dtype)
    mod = _module(blkq, ratio, dtype)
    if lut is None:
        lut = _fused(mod, q, k, v, None, blkq)[1]
    o_s, lse, d_o, grads = _direct(q, k, v, lut, blkq)
    want = _ref_grads(q, k, v, d_o, lut, blkq)
    restated = _ref_grads(q, k, v, d_o, lut, blkq, rdtype=dtype)
    for nm, gt, wt, rs in zip(("dq", "dk", "dv"), grads, want, restated):
        _check_grad(nm, gt, wt, rs, f"{name} q{blkq} {dtype} direct")
    if name in SPLIT:
        return
    qg, kg, vg = (t.clone().requires_grad_() for t in (q, k, v))
    out, sel = mod.forward_with_lut(qg, kg, vg)
    assert torch.equal(sel["lut"], lut)
    gout = torch.randn(out.shape, generator=torch.Generator(device="cuda").manual_seed(9), device="cuda").to(dtype)
    out.backward(gout)
    w, bias = mod.proj_l.weight.detach(), mod.proj_l.bias.detach()
    want = _ref_grads(q, k, v, gout, lut, blkq, w=w, bias=bias)
    restated = _ref_grads(q, k, v, gout, lut, blkq, w=w, bias=bias, rdtype=dtype)
    got = [qg.grad, kg.grad, vg.grad, mod.proj_l.weight.grad, mod.proj_l.bias.grad]
    for nm, gt, wt, rs in zip(("dq", "dk", "dv", "dW", "db"), got, want, restated):
        if nm in ("dW", "db"):
            s = _stats(gt, wt)
            print(f"{name} q{blkq} {dtype} module {nm}: kernel rel-L2 {s['rel_l2']:.2e} | restatement "
                  f"{_stats(rs, wt)['rel_l2']:.2e}")
            assert s["rel_l2"] <= 2e-2, (nm, s)
        else:
            _check_grad(nm, gt, wt, rs, f"{name} q{blkq} {dtype} module")


# ------------------------------------------------------------------------------------------------------------ 4. LUT order, sm_scale
@pytest.mark.parametrize("blkq,name", [pytest.param(bq, n, id=f"q{bq}-{n}") for bq in (128, 64)
                                       for n in ("all_x16", "split_dominant")])
def test_permuted_lut_rows(cuda, blkq, name):
    """The kernels take a LUT row in any order.  A random permutation of every row changes which warpgroup and which step
    sees each row's maximum; forward and backward stay within the same bars of float64."""
    (q, k, v), lut, ratio = _case(name, blkq, BF16)
    if lut is None:
        lut = _fused(_module(blkq, ratio, BF16), q, k, v, None, blkq)[1]
    g = torch.Generator().manual_seed(blkq)
    perm = torch.argsort(torch.rand(lut.shape, generator=g), -1).cuda()
    plut = lut.gather(-1, perm).contiguous()
    assert not torch.equal(plut, lut) and torch.equal(plut.sort(-1).values, lut.sort(-1).values)
    o_s, lse, d_o, grads = _direct(q, k, v, plut, blkq)
    ref = _ref_forward(q, k, v, plut, blkq, entry_max=True)
    assert _rescale_fraction(ref["emax"], blkq) > 0.3
    _bars(o_s, ref["o"], 0.9999, 5e-3, "o_s")
    _check_lse(lse, ref, name)
    want = _ref_grads(q, k, v, d_o, plut, blkq)
    restated = _ref_grads(q, k, v, d_o, plut, blkq, rdtype=BF16)
    for nm, gt, wt, rs in zip(("dq", "dk", "dv"), grads, want, restated):
        _check_grad(nm, gt, wt, rs, f"{name} q{blkq} permuted")


@pytest.mark.parametrize("blkq", [128, 64])
def test_sm_scale_other_than_head_dim(cuda, blkq):
    """The ABI takes the softmax scale; the module only ever passes d^-0.5.  0.5 / sqrt(d) through the forward with lse and
    the backward, on a large-score case."""
    sm_scale = 0.5 / D ** 0.5
    (q, k, v), lut, ratio = _case("all_x16", blkq, BF16)
    lut = _fused(_module(blkq, ratio, BF16), q, k, v, None, blkq)[1]
    o_s, lse, d_o, grads = _direct(q, k, v, lut, blkq, sm_scale=sm_scale)
    ref = _ref_forward(q, k, v, lut, blkq, sm_scale=sm_scale, entry_max=True)
    assert _rescale_fraction(ref["emax"], blkq) > 0.1
    _bars(o_s, ref["o"], 0.9999, 5e-3, "o_s")
    _check_lse(lse, ref, "sm_scale")
    want = _ref_grads(q, k, v, d_o, lut, blkq, sm_scale=sm_scale)
    restated = _ref_grads(q, k, v, d_o, lut, blkq, sm_scale=sm_scale, rdtype=BF16)
    for nm, gt, wt, rs in zip(("dq", "dk", "dv"), grads, want, restated):
        _check_grad(nm, gt, wt, rs, f"sm_scale q{blkq}")


# ------------------------------------------------------------------------------------------------------------ 3. long lists
def _check_long(q, k, v, lut, blkq, q_blocks, k_blocks, what):
    """Forward with lse and backward on `lut`: o_s and lse of every row against float64 attention, dQ of q_blocks and dK /
    dV of k_blocks against the closed-form float64 backward (float64 lse and delta), on every head."""
    b, l, h, _ = q.shape
    o_s, lse, d_o, (dq, dk, dv) = _direct(q, k, v, lut, blkq)
    ref = _ref_forward(q, k, v, lut, blkq, d_o=d_o)
    s_os = _bars(o_s, ref["o"], 0.9999, 5e-3, (what, "o_s"))
    row_err = (o_s.to(F64) - ref["o"]).norm(dim=-1) / ref["o"].norm(dim=-1)
    assert row_err.max() <= 2e-2, (what, "o_s row", row_err.max().item())
    worst = _check_lse(lse, ref, what)
    bm = B.block_mask(lut, _cdiv(l, BK))
    lines = [f"{what}: o_s rel-L2 {s_os['rel_l2']:.2e} (worst row {row_err.max().item():.2e}), lse max |err| {worst:.2e}"]
    for hi in range(h):
        for mi in q_blocks:
            r0, r1 = mi * blkq, min(l, (mi + 1) * blkq)
            s = _bars(dq[0, r0:r1, hi], B.ref_dq(q, k, v, d_o, bm, blkq, ref, 0, hi, mi), 0.999, 2e-2, (what, "dq", hi, mi))
            lines.append(f"  dq h{hi} qblk {mi}: rel-L2 {s['rel_l2']:.2e}")
        for ni in k_blocks:
            c0, c1 = ni * BK, min(l, (ni + 1) * BK)
            wk, wv = B.ref_dkdv(q, k, v, d_o, bm, blkq, ref, 0, hi, ni)
            sk = _bars(dk[0, c0:c1, hi], wk, 0.999, 2e-2, (what, "dk", hi, ni))
            sv = _bars(dv[0, c0:c1, hi], wv, 0.999, 2e-2, (what, "dv", hi, ni))
            lines.append(f"  dk / dv h{hi} kblk {ni} (list {int(bm[0, hi, :, ni].sum())}): rel-L2 {sk['rel_l2']:.2e} / "
                         f"{sv['rel_l2']:.2e}")
    print("\n".join(lines))


LONG_DENSE = [
    # blkq, L, dtype: nblk = 290 > 288 threads (sla_attn_fwd_kernel, sla_bwd_dq_kernel) and > 256 (the key-major index),
    # last key block 4 keys, last query block 68 rows; or nblk = 386 > 384 threads (the 64-row kernels), last key block 60
    pytest.param(128, 18500, BF16, id="q128-L18500-bf16"),
    pytest.param(128, 18500, FP16, id="q128-L18500-fp16"),
    pytest.param(64, 24700, BF16, id="q64-L24700-bf16"),
]


@pytest.mark.parametrize("blkq,l,dtype", LONG_DENSE)
def test_long_dense_block_lists(cuda, blkq, l, dtype):
    """Dense selection (topk = nblk) past every loop's single iteration: the LUT loaders, the key-major index's entry loop
    and its chunked scan, and dK / dV lists mblk long.  Checked against dense float64 attention."""
    h = 2
    mblk, nblk = _cdiv(l, blkq), _cdiv(l, BK)
    assert nblk > (288 if blkq == 128 else 384) and nblk > 256
    q, k, v = B.long_inputs(l, h, dtype, seed=l)
    lut = torch.arange(nblk, dtype=torch.int32, device="cuda").expand(1, h, mblk, nblk).contiguous()
    _check_long(q, k, v, lut, blkq, (0, mblk // 2, mblk - 1), (0, nblk // 2, nblk - 1), f"dense q{blkq} L{l} {dtype}")


@pytest.mark.parametrize("blkq", [128, 64])
def test_long_sparse_hand_made_lut(cuda, blkq):
    """Shape A's length, L = 32760 (512 key blocks, the last 56 keys): 400 of 512 key blocks per row, random and ascending,
    every row holding key block 0 and the last one, whose dK / dV lists are therefore mblk long."""
    l, h, topk = 32760, 2, 400
    mblk, nblk = _cdiv(l, blkq), _cdiv(l, BK)
    q, k, v = B.long_inputs(l, h, BF16, seed=blkq)
    g = torch.Generator().manual_seed(31 + blkq)
    lut = torch.empty(1, h, mblk, topk, dtype=torch.int32)
    for hi in range(h):
        for mi in range(mblk):
            mid = 1 + torch.randperm(nblk - 2, generator=g)[:topk - 2]
            lut[0, hi, mi] = torch.cat([torch.tensor([0, nblk - 1]), mid]).sort().values
    lut = lut.cuda()
    _check_long(q, k, v, lut, blkq, (0, mblk // 2, mblk - 1), (0, nblk // 2, nblk - 1), f"sparse q{blkq} L{l}")


@pytest.mark.parametrize("family,l", [pytest.param("sla16", 18500, id="sla16-q128-L18500"),
                                      pytest.param("sla16", 24700, id="sla16-q64-L24700"),
                                      pytest.param("sage", 18500, id="sage-q128-k64-L18500"),
                                      pytest.param("sage", 50000, id="sage-q64-k128-L50000")])
def test_long_dense_lists_fused_forward(cuda, family, l):
    """The fused forwards at topk = 1.0 past their CTA's thread count: SparseLinearAttention at (128, 64) and (64, 64), and the
    INT8 families at (128, 64) (nblk = 290 > 288) and (64, 128) (nblk = 391 > 384).  Sampled query blocks (first, middle,
    ragged last) of both heads against the fp32 oracle's per-block statement on the module's own selection."""
    from turbodiffusion_b200.SLA import SageSparseLinearAttention
    from turbodiffusion_b200.SLA.utils import set_served_arch
    h = 2
    if family == "sla16":
        blkq, blkk = (128, 64) if l == 18500 else (64, 64)
        mod = _module(blkq, 1.0, BF16)
        bars = (0.9999, 5e-3)
    else:
        blkq, blkk = (128, 64) if l == 18500 else (64, 128)
        mod = SageSparseLinearAttention(D, 1.0).cuda()
        g = torch.Generator().manual_seed(5)
        with torch.no_grad():
            mod.proj_l.weight.copy_(torch.randn(D, D, generator=g) * 0.05)
            mod.proj_l.bias.copy_(torch.randn(D, generator=g) * 0.05)
        bars = (0.999, 2e-2)                    # the INT8 families' bars against the exact oracle (test_gpu_sla.py)
    q, k, v = B.long_inputs(l, h, BF16, seed=l + 1)
    prev = set_served_arch("sm90" if (blkq, blkk) == (64, 128) else "sm100")
    try:
        assert mod.block_sizes(0) == (blkq, blkk)
        with torch.no_grad():
            out, sel = mod.forward_with_lut(q, k, v)
    finally:
        set_served_arch(prev)
    mblk, nblk = _cdiv(l, blkq), _cdiv(l, blkk)
    assert sel["topk"] == nblk and nblk > (288 if blkq == 128 else 384)
    w, bias = mod.proj_l.weight.detach().cpu(), mod.proj_l.bias.detach().cpu()
    for hi in range(h):
        qc, kc, vc = (t[:, :, hi:hi + 1].cpu() for t in (q, k, v))
        for m in (0, mblk // 2, mblk - 1):
            ref = O.sla_forward_block(qc, kc, vc, w, bias, 0, m, sel["lut"][0, hi, m].cpu(), blkq, blkk, mode="exact")
            s = _bars(out[0, m * blkq:min(l, (m + 1) * blkq), hi], ref.cuda(), *bars, (family, l, hi, m))
            print(f"{family} ({blkq}, {blkk}) L{l} h{hi} qblk {m}: rel-L2 {s['rel_l2']:.2e} cos {s['cos']:.7f}")
