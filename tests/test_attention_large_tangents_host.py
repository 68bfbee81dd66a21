"""CPU checks of the inputs tests/test_gpu_attention_large_tangents.py runs the attention JVP kernels on, through a torch
emulation of dense_attn_jvp_kernel's tile arithmetic (no GPU needed).

The inputs: log2-domain scores that climb along a shared key direction u by about 3.9 from one 64-key tile to the next, below
the lazy rescale's threshold (8), so the kernel rescales only every third tile and in between keeps p = exp2(s - m_used) with
m_used lagging the row maximum by up to 7.8: p reaches about 2^7.8; keys carry a large component along u (norms near 1800, the
"massive activation" pattern), so the score tangent S_t = sm_scale (q_t.k^T + q.k_t^T) reaches hundreds with unit tangents.  Then p * S_t, which the kernel rounds to the
16-bit type as an MMA operand, passes fp16's largest finite value 65504 while the normalised P * S_t and the exact tangent stay
far inside it.

The emulation follows the kernel: per 64-key tile the maxima, the lazy rescale of O, A, l and mu, and the products' operands p
and p * S_t rounded to the 16-bit type.  With `overflow_rescale` (the kernel in fp16) a row where some |p * S_t| of the tile
would round to inf is first rescaled onto its running maximum, so p <= 1 and |p * S_t| <= |S_t|; without it (the kernel in bf16,
whose range needs no such step, and in fp16 before it had the step) the lazy rule alone decides."""
import math

import pytest
import torch

import test_gpu_dense_attention_jvp as DJ

D, BK = 128, 64
SM = D ** -0.5
LOG2E = 1.0 / math.log(2.0)
F64 = torch.float64
BF16, FP16 = torch.bfloat16, torch.float16
FP16_MAX = 65504.0
THRESHOLD = 8.0

# name: (rises of the row maximum per 64-key tile in log2 units, cycled; base offset along u in log2 units; q_t's component
# along u).  "slow": every rise below the threshold.  "slow-qt-along-u": S_t also carries q_t.u times the keys' large component.
# "alternating": two slow rises, then one above the threshold, so tiles the running maximum leaps onto meet lagging ones in a
# row.  "large-keys": the same large component on every key, no ramp.
RAMPS = {
    "slow": ((3.9,), 0.0, 0.0),
    "slow-qt-along-u": ((3.9,), 0.0, 3.0),
    "alternating": ((3.9, 3.9, 10.0), 0.0, 1.0),
    "large-keys": ((0.0,), 58.0, 0.0),
}


def ramp_inputs(b, lq, lk, h, ramp, seed, tangent_scale=1.0):
    """q, k, v, q_t, k_t, v_t (float32, CPU) of the RAMPS entry `ramp`.  q = q_perp / 2 + u / 4 with q_perp orthogonal to
    u = ones / sqrt(D), so the score noise is about 0.7 log2 units; key j gets (offset of its tile) / (sm_scale log2e / 4) u.
    The tangents are unit randn (q_t plus its component along u), times tangent_scale."""
    rises, base, q_t_u = RAMPS[ramp]
    g = torch.Generator().manual_seed(seed)
    u = torch.ones(D) / D ** 0.5
    a = 0.25
    q = torch.randn(b, lq, h, D, generator=g)
    q = 0.5 * (q - (q @ u)[..., None] * u) + a * u
    n_tiles = -(-lk // BK)
    off = base + torch.tensor([0.0] + [rises[i % len(rises)] for i in range(n_tiles - 1)]).cumsum(0)
    k = torch.randn(b, lk, h, D, generator=g) + (off[torch.arange(lk) // BK] / (a * SM * LOG2E))[None, :, None, None] * u
    v = torch.randn(b, lk, h, D, generator=g)
    q_t = torch.randn(b, lq, h, D, generator=g) + q_t_u * u
    k_t, v_t = torch.randn(b, lk, h, D, generator=g), torch.randn(b, lk, h, D, generator=g)
    return [q, k, v] + [tangent_scale * t for t in (q_t, k_t, v_t)]


def _scores(ins):
    """float64 log2-domain scores s and natural-log score tangents S_t, [B, H, Lq, Lk], on the inputs' device"""
    q, k, _, q_t, k_t, _ = (t.to(F64) for t in ins)
    s = torch.einsum("bqhd,bkhd->bhqk", q, k) * (SM * LOG2E)
    st = (torch.einsum("bqhd,bkhd->bhqk", q_t, k) + torch.einsum("bqhd,bkhd->bhqk", q, k_t)) * SM
    return s, st


def _tiles(x, order):
    """[B, H, Lq, Lk] -> [B, H, Lq, n, 64] in visiting order: key tiles 0, 1, ... or, with `order` [B, H, Mblk, topk] (a LUT
    over 128-row query blocks), the listed tiles in list order; keys >= Lk are -inf"""
    lk = x.shape[-1]
    t = torch.nn.functional.pad(x, (0, -lk % BK), value=-math.inf).unflatten(-1, (-1, BK))
    if order is None:
        return t
    rows = order.to(x.device).long()[:, :, torch.arange(x.shape[2], device=x.device) // 128]      # [B, H, Lq, topk]
    return torch.gather(t, 3, rows[..., None].expand(*rows.shape, BK))


def overflow_stats(ins, order=None, mask=None):
    """float64 statistics of the inputs (dense, or over the keys `order` lists, `mask` [B, H, Lq, Lk] its key mask):
    (fraction of rows where the lazily rescaled p * |S_t| of some key exceeds 65504, the largest normalised |P * S_t|, the
    largest lag of the lazy maximum m_used behind the row's running maximum (the log2 of the largest p), the fraction of
    tile-to-tile rises of the running maximum above the threshold)"""
    s, st = _scores(ins)
    if mask is not None:
        s = s.masked_fill(~mask, -math.inf)
    st_t, s_t = _tiles(st.masked_fill(~torch.isfinite(s), 0.0), order), _tiles(s, order)
    worst = torch.zeros(s.shape[:3], dtype=F64, device=s.device)
    lag, steep = 0.0, 0.0
    for j in range(s_t.shape[3]):
        mx = s_t[..., j, :].amax(-1)
        if j == 0:
            m_used, m_run = mx, mx
        else:
            steep += (mx > m_run + THRESHOLD).double().mean().item() / (s_t.shape[3] - 1)
            m_used = torch.where(mx > m_used + THRESHOLD, mx, m_used)
            m_run = torch.maximum(m_run, mx)
            lag = max(lag, (m_run - m_used).max().item())
        p = torch.exp2(s_t[..., j, :] - m_used[..., None])
        worst = torch.maximum(worst, (p * st_t[..., j, :].abs()).nan_to_num(0.0).amax(-1))
    norm = (torch.softmax(s / LOG2E, -1) * st.abs()).amax().item()
    return (worst > FP16_MAX).double().mean().item(), norm, lag, steep


def emulate_jvp(ins, dtype, overflow_rescale):
    """(out, out_t) of dense_attn_jvp_kernel's arithmetic in float32 torch on the dtype-rounded inputs"""
    q, k, v, q_t, k_t, v_t = (t.to(dtype).float().transpose(1, 2) for t in ins)      # [B, H, L, D]
    s = (q @ k.transpose(-1, -2)) * (SM * LOG2E)
    st = (q_t @ k.transpose(-1, -2) + q @ k_t.transpose(-1, -2)) * SM
    lk = k.shape[2]
    rows = s.shape[:3]
    o, a = torch.zeros(*rows, D), torch.zeros(*rows, D)
    l, mu = torch.zeros(rows), torch.zeros(rows)
    for j in range(-(-lk // BK)):
        keys = slice(j * BK, min(lk, (j + 1) * BK))
        mx = s[..., keys].amax(-1)
        if j == 0:
            m_used, m_run = mx, mx
        else:
            alpha = torch.where(mx > m_used + THRESHOLD, torch.exp2(m_used - mx), torch.ones_like(mx))
            o, a, l, mu = o * alpha[..., None], a * alpha[..., None], l * alpha, mu * alpha
            m_used, m_run = torch.where(mx > m_used + THRESHOLD, mx, m_used), torch.maximum(m_run, mx)
        p = torch.exp2(s[..., keys] - m_used[..., None])
        l = l + p.sum(-1)
        x = p * st[..., keys]
        if overflow_rescale:
            alpha = torch.where(x.abs().amax(-1) > FP16_MAX, torch.exp2(m_used - m_run), torch.ones_like(mx))
            o, a, l, mu = o * alpha[..., None], a * alpha[..., None], l * alpha, mu * alpha
            p, x, m_used = p * alpha[..., None], x * alpha[..., None], torch.where(alpha < 1, m_run, m_used)
        mu = mu + x.sum(-1)
        p_r = p.to(dtype).float()
        o = o + p_r @ v[..., keys, :]
        a = a + x.to(dtype).float() @ v[..., keys, :] + p_r @ v_t[..., keys, :]
    out = (o / l[..., None]).to(dtype)
    out_t = ((a - (mu / l)[..., None] * o) / l[..., None]).to(dtype)
    return out.transpose(1, 2), out_t.transpose(1, 2)


# ------------------------------------------------------------------------------------------------------------ the inputs
LQ, LK, H = 256, 1000, 2


@pytest.mark.parametrize("ramp", ["slow", "slow-qt-along-u", "alternating"])
def test_rises_and_overflow_regime(ramp):
    """The lazy maximum lags the running one by more than 7 (p near 2^8); on "slow" no rise of the running maximum passes the
    threshold, on "alternating" a third do; the lazily rescaled p * |S_t| passes 65504 in some rows while P * |S_t| stays below
    65504 / 32."""
    ins = [t.to(FP16).float() for t in ramp_inputs(1, LQ, LK, H, ramp, seed=1)]
    over, norm, lag, steep = overflow_stats(ins)
    print(f"{ramp}: rows over 65504 {over:.3f}, max normalised |P S_t| {norm:.0f}, largest lag {lag:.2f}, steep rises {steep:.3f}")
    assert over > (0.2 if ramp == "slow-qt-along-u" else 0.0) and norm < FP16_MAX / 32, (over, norm)
    assert 7.0 < lag <= THRESHOLD
    assert (0.25 < steep < 0.4) if ramp == "alternating" else steep == 0.0, steep


@pytest.mark.parametrize("ramp", ["slow", "slow-qt-along-u", "alternating"])
def test_fp16_overflows_with_the_lazy_rule_alone_and_not_with_the_overflow_rescale(ramp):
    """fp16: with the lazy rescale alone out_t has non-finite rows; with the overflow rescale (the kernel's arithmetic) out_t
    is finite and meets the GPU tests' bar against float64, the primal meets DJ's, and the rows the lazy rule kept finite keep
    their bits."""
    ins = [t.to(FP16) for t in ramp_inputs(1, LQ, LK, H, ramp, seed=1)]
    lazy, lazy_t = emulate_jvp(ins, FP16, overflow_rescale=False)
    out, out_t = emulate_jvp(ins, FP16, overflow_rescale=True)
    bad = (~torch.isfinite(lazy_t)).any(-1)
    want, want_t = DJ.exact_f64(*ins)
    ours, ref = DJ._rel(out_t, want_t), DJ._rel(DJ.restated(*ins), want_t)
    print(f"{ramp}: lazy rule: {bad.sum().item()} of {LQ * H} rows non-finite; overflow rescale: rel-L2 {ours:.2e}, "
          f"restatement {ref:.2e}")
    assert bad.any()
    assert torch.equal(out[~bad], lazy[~bad]) and torch.equal(out_t[~bad], lazy_t[~bad])
    DJ._check_primal(out, want, ramp)
    assert torch.isfinite(out_t).all() and ours <= 1.5 * ref + 1e-7, (ours, ref)


@pytest.mark.parametrize("ramp", ["slow", "slow-qt-along-u", "alternating"])
def test_bf16_has_the_range(ramp):
    """bf16 has the range: with the lazy rule alone out_t is finite and meets the bar."""
    ins = [t.to(BF16) for t in ramp_inputs(1, LQ, LK, H, ramp, seed=1)]
    _, out_t = emulate_jvp(ins, BF16, overflow_rescale=False)
    _, want_t = DJ.exact_f64(*ins)
    ours, ref = DJ._rel(out_t, want_t), DJ._rel(DJ.restated(*ins), want_t)
    print(f"{ramp} bf16: rel-L2 {ours:.2e}, restatement {ref:.2e}")
    assert torch.isfinite(out_t).all() and ours <= 1.5 * ref + 1e-7, (ours, ref)


def test_tangent_scale_sweep_stays_representable():
    """The fp16 sweep of the GPU tests: at tangent scales 1 .. 64 of "slow" the normalised |P * S_t| and the float64 out_t stay
    below 65504 / 2, and the kernel's fp16 arithmetic keeps out_t finite at every scale."""
    for scale in (1, 4, 16, 64):
        ins = [t.to(FP16) for t in ramp_inputs(1, LQ, LK, H, "slow", seed=1, tangent_scale=scale)]
        _, norm, _, _ = overflow_stats(ins)
        _, want_t = DJ.exact_f64(*ins)
        _, out_t = emulate_jvp(ins, FP16, overflow_rescale=True)
        print(f"x{scale}: max normalised |P S_t| {norm:.0f}, max |out_t| {want_t.abs().max().item():.1f}")
        assert norm < FP16_MAX / 2 and want_t.abs().max().item() < FP16_MAX / 2
        assert torch.isfinite(out_t).all()


def test_lut_order_follows_the_listed_tiles():
    """overflow_stats over a LUT visits the listed tiles in list order: the full ascending LUT gives the dense statistics, and
    the reversed one (the maximum found first) never exceeds the threshold lag, so nothing overflows."""
    ins = [t.to(FP16).float() for t in ramp_inputs(1, LQ, LK, H, "slow-qt-along-u", seed=1)]
    nblk, mblk = -(-LK // BK), -(-LQ // 128)
    full = torch.arange(nblk, dtype=torch.int32).expand(1, H, mblk, nblk)
    assert overflow_stats(ins, full) == overflow_stats(ins)
    over, _, _, _ = overflow_stats(ins, full.flip(-1))
    assert over == 0.0
