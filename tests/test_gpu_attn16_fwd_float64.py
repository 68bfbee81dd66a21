"""The 16-bit attention forwards, JVP and tangent kernels against float64 on the kernel's own inputs, query block by query block
and row by row: sla_attn_fwd_kernel<T, 128, kQK16> (128 x 64 blocks) and sla_attn_fwd_q64_kernel<T, 128, kQK16, 64> (64 x 64)
behind tdb200_sla_attn16_fwd (fused: sparse branch + linear branch + proj_b) and tdb200_sla_attn16_fwd_lse; dense_attn_fwd_kernel
behind tdb200_attn_dense_fwd(_lse); dense_attn_jvp_kernel behind tdb200_attn_dense_jvp(_lse) and tdb200_sla_attn16_jvp(_lse);
attn_tangent_kernel behind tdb200_attn_dense_tangent and tdb200_sla_attn16_tangent.  Every output is a sentinel-filled buffer
longer than the output, so rows past l (past lq for dense) of out, out_t and lse are checked untouched.

Two references per row, built from what the kernel is given (16-bit q, k, v and tangents, the LUT, the fused forward's own
kvw, ksum and proj_b, the tangent kernel's out and lse from the lse forward):
  * R64, the float64 closed form: softmax(S sm) V (+ phi(q) KVW^T / den + proj_b), lse = log2 sum 2^(S sm log2e), and the
    tangent out_t = sum P S_t v - (sum P S_t) o + P v_t with S_t = sm (q_t k^T + q k_t^T).
  * R32, the kernel's rounding points: s = fl(fl(q.k) sc), sc = fl(sm log2e) (softmax_p); p = exp2(fl(s - m)) in fp32 against
    the maximum the kernel uses at that entry (B.running_max: the 2^8 lazy rescale in list order, one sequence per row on
    128-row blocks, one per warpgroup over alternate entries on 64-row blocks and then their merge; dense: ascending 128-key
    tiles for the forward, 64-key tiles for the JVP, whose fp16 instantiation also rescales a row onto its running maximum
    where |p S_t| would pass 65504); the row sum from the unrounded p, P rounded to T as the P.V operand, each entry weighted
    exactly into the final maximum; out = T(fl(O) fl(1/l)).  Fused: A = T(phi l / den) with fp16's power-of-two row scaling
    (B.round_operand), O + A KVW^T, then / l + proj_b.  JVP: x = fl(p fl(fl(S_t / sm) sm)), mu from the unrounded x, T(p)
    and T(x) as operands, out_t = T((A - (mu / l) O) / l).  Tangent: P = exp2(fl(s - lse)) with the kernel's lse, the same
    products, out_t = T(A - mu out) with the kernel's rounded out.  lse = fl(m + fl(log2 l)).

Bars (the backward file's forms).  Per (batch, head, query block) rel-L2 against R64 <= 1.5x R32's.  Per row of o, o_s and
out_t: |kernel - R64| <= 2 max(|R32 - R64| + acc + allow, |T(R64) - R64|) + sqrt(d) sub, sub one subnormal step of T.
acc: one fp32 rounding (2^-24) per 16-key P.V MMA step, relative to the accumulator it rounds, bounded by the largest
partial sum |O| (|A| for out_t) the accumulator reaches over the list (_peak, per warpgroup on 64-row blocks), over l; it
matters only at the limit-length lists.  allow: what R32's exact-then-rounded S and S_t do not model: the kernel's fp32 MMA
chains are within 2^-20 of their |terms| sums, and ex2.approx within 2^-22 relative, so each p carries a relative error
e_p = 2^-20 sc ln2 (|q|.|k|) + 2^-22 and each S_t an absolute one 2^-20 sm (|q_t|.|k| + |q|.|k_t|), carried through the
normalisation (sum P e_p (|v| + |o|)).  The block bar takes allow but not acc: R32 sums exactly, so its error leaves the
accumulation out, and 1.5x of it leaves that room where the P.V chains are long.
Per row of lse, in log2 units:
    |lse - R64| <= 2 (|R32 - R64| + acc_l) + ulp(lse) + lg2,
  acc_l = (keys / 8 2^-24 + sum P e_p) / ln2 is l's relative error in log2 units (each thread adds its 8 pairs of p per 64
  keys into one fp32 partial sum, one rounding each, and every p carries e_p); ulp(lse) covers the fp32 rounding of
  m + log2(l), the kernel's and R32's alike; lg2 = max(2^-22, 2 ulp(log2 l)) is __log2f's documented error (lg2.approx.f32:
  2^-22 absolute for l in [0.5, 2], 2 ulp elsewhere; CUDA C++ Programming Guide, intrinsic functions).
Always: every output and every reference finite, and every sentinel past the last row untouched.  At the limit lengths a
zero output and half of the list dropped are shown to fail every row (_limit_faults).  Every hand-made case first asserts from float64
statistics of its inputs that it reaches the regime it is named for.  Every test prints its worst row as a fraction of its bar.

test_bars_reject_kernel_faults shows what these bars catch that the whole-tensor bars of the other tests accept.
"""
import math
import time
from types import SimpleNamespace

import pytest
import torch

import sla_backward_oracle as B
import test_attention_large_tangents_host as LT

pytestmark = pytest.mark.gpu
D, BK = 128, 64
SM = D ** -0.5
LN2 = math.log(2.0)
F64, F32 = torch.float64, torch.float32
BF16, FP16 = torch.bfloat16, torch.float16
DTYPES = [pytest.param(BF16, id="bf16"), pytest.param(FP16, id="fp16")]
GEOMS = [pytest.param(128, id="q128"), pytest.param(64, id="q64")]
SM32 = float(torch.tensor(SM, dtype=F32))
SC32 = float(torch.tensor(SM, dtype=F32) * torch.tensor(1.4426950408889634, dtype=F32))   # p.sm_scale * kLog2e in fp32
SUB = {BF16: 2.0 ** -133, FP16: 2.0 ** -24}
PAD_ROWS = 37
SENTINEL = -1234.0
FP32_SUM = 2.0 ** -20   # the kernel's fp32 S and S_t against their |terms| sums
EX2 = 2.0 ** -22        # ex2.approx.ftz.f32, relative
LG2 = 2.0 ** -22        # lg2.approx.f32, absolute on [0.5, 2]
CHUNK = 1 << 15         # keys per float64 tile of the references (a multiple of every key tile)
LOG2_FP16_MAX = math.log2(65504.0)
# The 16-bit forwards' largest top-k (derived in tests/test_sla_q64_16bit_host.py beside the validation table), and the JVP
# and tangent kernels' (jvp::kMaxLutIds: the LUT row fills the last 34,560 bytes of shared memory).
FWD_TOPK_LIMIT = {128: 11220, 64: 13952}
JVP_TOPK_LIMIT = 8640

_WORST = []


@pytest.fixture(autouse=True)
def _report_worst(request):
    _WORST.clear()
    yield
    if _WORST:
        print(f"\n{request.node.name}: worst row at {max(_WORST):.3f} of its bar")


# ------------------------------------------------------------------------------------------------------------ kernel calls
def _lib():
    from turbodiffusion_b200 import _lib
    return _lib


_last_error = B.last_error


def _ok(rc):
    torch.cuda.synchronize()
    assert rc == 0, _last_error()


def _bufs(x, *names, lse=False):
    """Sentinel-filled outputs named `names` ([b, lq, h, d]) and, with lse, x.lse ([b, h, lq] fp32), PAD_ROWS rows longer."""
    views, pads = B.sentinel_buffers(x.dtype, x.q.device, PAD_ROWS, SENTINEL, *[x.q.shape] * len(names))
    for n, v, p in zip(names, views, pads):
        setattr(x, n, v)
        x.pads[n] = p
    if lse:
        (x.lse,), (x.pads["lse"],) = B.sentinel_buffers(F32, x.q.device, PAD_ROWS, SENTINEL, (x.b, x.h, x.lq, 1))
        x.lse = x.lse.view(x.b, x.h, x.lq)


def _linear_inputs(x, seed=9):
    """The fused forward's kvw, ksum (of the keys' feature map) and proj_b, as the module computes them."""
    from turbodiffusion_b200.SLA.core import linear_moments, project_moments
    kv, x.ksum = linear_moments(x.k, x.v, x.feature)
    g = torch.Generator().manual_seed(seed)
    w = (torch.randn(D, D, generator=g) * 0.05).to(x.q.device)
    x.proj_b = (torch.randn(D, generator=g) * 0.05).float().to(x.q.device).contiguous()
    x.kvw = project_moments(w, kv, x.dtype)


def _run(x, kind):
    """One kernel call into sentinel buffers.  kind: "fused", "lse" (SLA forwards), "dense", "dense_lse", "jvp", "jvp_lse",
    "tangent" (after an lse forward, whose out and lse it reads)."""
    L = _lib()
    lib, p, tag, st = L.lib(), L.ptr, L.DTYPE_TAG[x.dtype], L.stream_ptr(x.q.device)
    sparse = x.lut is not None
    topk = x.lut.shape[-1] if sparse else 0
    x.pads = {}
    t0 = time.perf_counter()
    if kind == "fused":
        if getattr(x, "kvw", None) is None:
            _linear_inputs(x)
        _bufs(x, "out")
        _ok(lib.tdb200_sla_attn16_fwd(p(x.q), p(x.k), p(x.v), tag, p(x.lut), topk, p(x.kvw), p(x.ksum), p(x.proj_b), p(x.out),
                                      x.b, x.lq, x.lk, x.h, D, SM, x.feature, x.blkq, BK, st))
    elif kind == "lse":
        _bufs(x, "o_s", lse=True)
        _ok(lib.tdb200_sla_attn16_fwd_lse(p(x.q), p(x.k), p(x.v), tag, p(x.lut), topk, p(x.o_s), p(x.lse), x.b, x.lq, x.h, D, SM,
                                          x.blkq, BK, st))
    elif kind in ("dense", "dense_lse"):
        _bufs(x, "o_s", lse=kind == "dense_lse")
        if kind == "dense":
            _ok(lib.tdb200_attn_dense_fwd(p(x.q), p(x.k), p(x.v), tag, p(x.o_s), x.b, x.lq, x.lk, x.h, D, SM, st))
        else:
            _ok(lib.tdb200_attn_dense_fwd_lse(p(x.q), p(x.k), p(x.v), tag, p(x.o_s), p(x.lse), x.b, x.lq, x.lk, x.h, D, SM, st))
    elif kind in ("jvp", "jvp_lse"):
        _bufs(x, "o_s", "out_t", lse=kind == "jvp_lse")
        ins = (p(x.q), p(x.k), p(x.v), p(x.qt), p(x.kt), p(x.vt), tag)
        lse = (p(x.lse),) if kind == "jvp_lse" else ()
        if sparse:
            fn = lib.tdb200_sla_attn16_jvp_lse if lse else lib.tdb200_sla_attn16_jvp
            _ok(fn(*ins, p(x.lut), topk, p(x.o_s), p(x.out_t), *lse, x.b, x.lq, x.h, D, SM, 128, BK, st))
        else:
            fn = lib.tdb200_attn_dense_jvp_lse if lse else lib.tdb200_attn_dense_jvp
            _ok(fn(*ins, p(x.o_s), p(x.out_t), *lse, x.b, x.lq, x.lk, x.h, D, SM, st))
    elif kind == "tangent":
        _run(x, "lse" if sparse else "dense_lse")
        t0 = time.perf_counter()
        _bufs(x, "out_t")
        ins = (p(x.q), p(x.k), p(x.v), p(x.qt), p(x.kt), p(x.vt), p(x.o_s), p(x.lse), tag)
        if sparse:
            _ok(lib.tdb200_sla_attn16_tangent(*ins, p(x.lut), topk, p(x.out_t), x.b, x.lq, x.h, D, SM, 128, BK, st))
        else:
            _ok(lib.tdb200_attn_dense_tangent(*ins, p(x.out_t), x.b, x.lq, x.lk, x.h, D, SM, st))
    else:
        raise ValueError(kind)
    x.kind, x.seconds = kind, time.perf_counter() - t0
    return x


def _case(q, k, v, lut, blkq=128, tangents=None, feature=0):
    """The inputs of one call on the GPU (lut None: dense attention); tangents = (q_t, k_t, v_t) for the JVP and tangent."""
    x = SimpleNamespace(q=q.contiguous(), k=k.contiguous(), v=v.contiguous(), lut=lut, blkq=blkq, dtype=q.dtype,
                        feature=feature, pads={}, kvw=None)
    x.qt, x.kt, x.vt = (None, None, None) if tangents is None else (t.contiguous() for t in tangents)
    x.b, x.lq, x.h, _ = q.shape
    x.lk = k.shape[1]
    x.mblk = B.cdiv(x.lq, blkq)
    return x


_randn = B.randn


def _inputs(b, lq, lk, h, dtype, seed):
    """q, k, v and the tangents q_t, k_t, v_t (half scale) on the GPU."""
    shapes = [(b, lq, h, D), (b, lk, h, D), (b, lk, h, D)]
    prim = [_randn(s, dtype, seed + i) for i, s in enumerate(shapes)]
    return prim, [_randn(s, dtype, seed + 10 + i, 0.5) for i, s in enumerate(shapes)]


# ------------------------------------------------------------------------------------------------------------ references
def _tiles_of(x, kind, bi, hi, m, lut_row=None):
    """(start key of each entry in visiting order, keys per entry, one running maximum per warpgroup over alternate entries)."""
    dev = x.q.device
    if x.lut is None:
        tw = 128 if kind in ("dense", "dense_lse") else 64
        return torch.arange(0, x.lk, tw, device=dev), tw, False
    ids = (x.lut[bi, hi, m] if lut_row is None else torch.as_tensor(lut_row)).long().to(dev)
    return ids * BK, BK, x.blkq == 64 and kind in ("fused", "lse")


def _running_max_jvp(ent_max, ent_g):
    """dense_attn_jvp_kernel's maximum per tile ([R, tiles] float32, visiting order): the lazy rule, and with ent_g (fp16: the
    log2 of each tile's largest |exp2(s) S_t|) the overflow rescale onto the running maximum where |p S_t| would pass 65504."""
    m = ent_max.clone()
    run = ent_max[:, 0].clone()
    for j in range(1, ent_max.shape[1]):
        prev = m[:, j - 1]
        mj = torch.where(ent_max[:, j] > prev + 8.0, ent_max[:, j], prev)
        run = torch.maximum(run, ent_max[:, j])
        if ent_g is not None:
            mj = torch.where(ent_g[:, j] - mj.double() > LOG2_FP16_MAX, run, mj)
        m[:, j] = mj
    return m


def _refs(x, kind, bi, hi, rows, lut_row=None, drop_keys=None, lse_rows=None, out_rows=None):
    """The references of query rows `rows` (one query block) of batch bi, head hi for the call `kind`:
    {output name: (R64, R32, |terms| sum, MMA steps, allowance) [R, d] as _judge takes them; "lse": (R64, R32, bar extra) [R]}.
    lut_row / drop_keys (a mask over the keys visited) / lse_rows, out_rows (the rows whose lse and out the tangent reads)
    replace what the kernel would read: the sensitivity test's faults."""
    dev, dt = x.q.device, x.dtype
    rows = rows.to(dev)
    R = len(rows)
    m_blk = int(rows[0]) // x.blkq
    starts, tw, two_wg = _tiles_of(x, kind, bi, hi, m_blk, lut_row)
    keys = (starts[:, None] + torch.arange(tw, device=dev)).flatten()
    dead = keys >= x.lk
    if drop_keys is not None:
        dead = dead | drop_keys(keys)
    keys = keys.clamp_max(x.lk - 1)
    tangent = kind in ("jvp", "jvp_lse", "tangent")
    q = x.q[bi, rows, hi].double()
    qt = x.qt[bi, rows, hi].double() if tangent else None

    def chunks():
        for c0 in range(0, keys.numel(), CHUNK):
            kk, dd = keys[c0:c0 + CHUNK], dead[c0:c0 + CHUNK]
            kc = x.k[bi, kk, hi].double()
            dot = q @ kc.t()
            t = SimpleNamespace(c0=c0, kk=kk, kc=kc)
            t.s64 = (dot * (SM / LN2)).masked_fill(dd, -math.inf)
            t.s32 = (dot.float() * SC32).masked_fill(dd, -math.inf)
            t.e_p = FP32_SUM * SC32 * LN2 * (q.abs() @ kc.abs().t()) + EX2
            if tangent:
                ktc = x.kt[bi, kk, hi].double()
                sd = qt @ kc.t() + q @ ktc.t()
                t.st64 = (SM * sd).masked_fill(dd, 0.0)
                t.st32 = (sd.float() * SM32).masked_fill(dd, 0.0)
                t.e_st = SM * FP32_SUM * (qt.abs() @ kc.abs().t() + q.abs() @ ktc.abs().t())
            yield t

    # pass 1: the float64 row maxima and each entry's fp32 maximum, for the maxima the kernel uses
    m64 = torch.full((R,), -math.inf, dtype=F64, device=dev)
    ent_max, ent_g = [], []
    fp16_jvp = kind in ("jvp", "jvp_lse") and dt == FP16
    for t in chunks():
        m64 = torch.maximum(m64, t.s64.amax(-1))
        ent_max.append(t.s32.view(R, -1, tw).amax(-1))
        if fp16_jvp:
            ent_g.append((t.s32.double() + t.st32.double().abs().log2()).view(R, -1, tw).amax(-1))
    ent_max = torch.cat(ent_max, 1).cpu()
    if kind == "tangent":
        m_ent = None
    elif tangent:
        m_ent = _running_max_jvp(ent_max, torch.cat(ent_g, 1).cpu() if fp16_jvp else None).to(dev)
    else:
        m_ent = B.running_max(ent_max, two_wg).to(dev)
    if m_ent is not None:
        m_top = m_ent[:, -2:].amax(-1) if two_wg else m_ent[:, -1]
        w_ent = torch.exp2(m_ent.double() - m_top.double()[:, None])
    else:
        lse_in = x.lse[bi, hi, rows if lse_rows is None else lse_rows.to(dev)]

    z = lambda: torch.zeros(R, D, dtype=F64, device=dev)
    zr = lambda: torch.zeros(R, dtype=F64, device=dev)
    l64, l32, al_l, mu64, mu32, al_mu = zr(), zr(), zr(), zr(), zr(), zr()
    o64, o32, pk_o, al_o, a64, a32, pk_a, al_a = z(), z(), z(), z(), z(), z(), z(), z()
    run_o = torch.zeros(2 if two_wg else 1, R, D, dtype=F64, device=dev)   # each accumulator's running sum of O and of A
    run_a = torch.zeros(1, R, D, dtype=F64, device=dev)
    for t in chunks():
        vc = x.v[bi, t.kk, hi].double()
        p64 = torch.exp2(t.s64 - m64[:, None])
        if m_ent is None:
            p32 = torch.exp2(t.s32 - lse_in[:, None])
            w = 1.0
        else:
            e0, ne = t.c0 // tw, t.s32.shape[1] // tw
            p32 = torch.exp2(t.s32 - m_ent[:, e0:e0 + ne].repeat_interleave(tw, 1))
            w = w_ent[:, e0:e0 + ne].repeat_interleave(tw, 1)
        pw = p32.double() * w
        pr = p32.to(dt).double() * w
        l64 += p64.sum(-1)
        o64 += p64 @ vc
        l32 += pw.sum(-1)
        o32 += pr @ vc
        pk_o = torch.maximum(pk_o, _peak(run_o, ((pr, vc),), t.c0 // tw, tw))
        e = pw * t.e_p
        al_l += e.sum(-1)
        al_o += e @ vc.abs()
        if tangent:
            vtc = x.vt[bi, t.kk, hi].double()
            x32 = p32 * t.st32
            xr = x32.to(dt).double() * w
            mu64 += (p64 * t.st64).sum(-1)
            a64 += (p64 * t.st64) @ vc + p64 @ vtc
            mu32 += (x32.double() * w).sum(-1)
            a32 += xr @ vc + pr @ vtc
            pk_a = torch.maximum(pk_a, _peak(run_a, ((xr, vc), (pr, vtc)), 0, tw))
            est = pw * t.e_st
            al_a += (e * t.st64.abs() + est) @ vc.abs() + e @ vtc.abs()
            al_mu += (e * t.st64.abs() + est).sum(-1)

    steps = B.cdiv(keys.numel(), 16)
    o = o64 / l64[:, None]
    refs = {}
    if kind == "tangent":
        out_in = x.o_s[bi, rows if out_rows is None else out_rows.to(dev), hi].double()
        mu = mu64 / l64
        ot64 = a64 / l64[:, None] - mu[:, None] * o
        ot32 = (a32 - mu32[:, None] * out_in).to(dt).double()
        mag = pk_a + mu32.abs()[:, None] * out_in.abs()
        refs["out_t"] = (ot64, ot32, mag, steps, al_a + al_mu[:, None] * o.abs())
        return refs
    inv32 = (1.0 / l32.float()).double()
    allow_o = (al_o + al_l[:, None] * o.abs()) / l32[:, None]   # al_* sum R32's p, in l32's units
    if kind == "fused":
        phi = _phi(x.q[bi, rows, hi].double(), x.feature)
        den = phi @ x.ksum[bi, hi].double() + 1e-5
        kvw, pb = x.kvw[bi, hi].double(), x.proj_b.double()
        a = B.round_operand(phi * (l32 / den)[:, None], dt)
        r64 = o + (phi @ kvw.t()) / den[:, None] + pb
        r32 = ((o32 + a @ kvw.t()) / l32[:, None] + pb).to(dt).double()
        mag = (pk_o + (a @ kvw.t()).abs()) / l32[:, None]
        refs["out"] = (r64, r32, mag, steps + D // 16, allow_o)
        return refs
    refs["o_s"] = (o, (o32.float().double() * inv32[:, None]).float().to(dt).double(), pk_o / l32[:, None], steps, allow_o)
    if tangent:
        mu = mu64 / l64
        ot64 = a64 / l64[:, None] - mu[:, None] * o
        mu_l = mu32 * inv32
        ot32 = ((a32 - mu_l[:, None] * o32) * inv32[:, None]).to(dt).double()
        mag = (pk_a + mu_l.abs()[:, None] * pk_o) / l32[:, None]
        allow = ((al_a + al_mu[:, None] * o.abs()) / l32[:, None]
                 + (al_l / l32)[:, None] * (ot64.abs() + mu.abs()[:, None] * o.abs()))
        refs["out_t"] = (ot64, ot32, mag, steps, allow)
    lse64 = m64 + torch.log2(l64)
    lse32 = (m_top.float() + torch.log2(l32.float())).double()
    acc_l = (keys.numel() / 8 * 2.0 ** -24 + al_l / l32) / LN2
    lg2 = torch.maximum(torch.full_like(l64, LG2), 2 * _ulp32(torch.log2(l64)))
    refs["lse"] = (lse64, lse32, 2 * acc_l + _ulp32(lse64) + lg2)
    return refs


def _peak(run, products, e0, tw):
    """The largest |partial sum| [R, d] an accumulator reaches while it adds, entry by entry in list order, the sum of the
    products p [R, n tw] . v [n tw, d]: run [G, R, d] holds the running sum of each of the G accumulators (G = 2: the 64-row
    kernels' warpgroups, which take the entries j = g mod 2; e0 is the first entry's index) and is updated."""
    n = products[0][0].shape[1] // tw
    terms = sum(torch.einsum("rnt,ntd->rnd", p.view(p.shape[0], n, tw), v.view(n, tw, -1)) for p, v in products)
    peak = torch.zeros_like(run[0])
    for g in range(run.shape[0]):
        part = terms[:, (g - e0) % run.shape[0]::run.shape[0]]
        if part.shape[1] == 0:
            continue
        sums = part.cumsum(1) + run[g][:, None]
        peak = torch.maximum(peak, sums.abs().amax(1))
        run[g] = sums[:, -1]
    return peak


def _ulp32(a):
    return torch.ldexp(torch.ones_like(a), torch.frexp(a.abs().clamp_min(2.0 ** -126)).exponent - 24)


_phi = B.phi


# ------------------------------------------------------------------------------------------------------------ bars
def _judge(got, ref, dtype, what, record=True):
    """The bars on one block of rows.  Returns (block passes, per-row pass) and prints the distances."""
    r64, r32, mag, steps, allow = ref
    assert bool(torch.isfinite(r64).all() and torch.isfinite(r32).all()), (what, "reference not finite")
    got = got.double()
    e_k = (got - r64).norm(dim=-1)
    e_32 = (r32 - r64).norm(dim=-1)
    e_t = (r64.to(dtype).double() - r64).norm(dim=-1)
    allow = allow.norm(dim=-1)
    acc = steps * 2.0 ** -24 * mag.norm(dim=-1) + allow
    floor = SUB[dtype] * math.sqrt(D)
    bar = 2 * torch.maximum(e_32 + acc, e_t) + floor
    rows_ok = e_k <= bar
    block_ok = e_k.norm() <= 1.5 * e_32.norm() + allow.norm() + floor * math.sqrt(len(e_k))
    ratio = e_k / bar
    worst = int(torch.argmax(ratio))
    if record:
        _WORST.append(float(ratio[worst]))
    nrm = r64.norm().clamp_min(1e-300)
    if not (block_ok and rows_ok.all()) or record is None:
        print(f"{what}: rel-L2 kernel {float(e_k.norm() / nrm):.3e} R32 {float(e_32.norm() / nrm):.3e}; worst row {worst} at "
              f"{float(ratio[worst]):.3f} of its bar; rows failing {int((~rows_ok).sum())}/{len(rows_ok)}")
    return bool(block_ok), rows_ok


def _judge_lse(got, ref, what):
    r64, r32, extra = ref
    assert bool(torch.isfinite(r64).all() and torch.isfinite(r32).all()), (what, "lse reference not finite")
    e_k = (got.double() - r64).abs()
    bar = 2 * (r32 - r64).abs() + extra
    ok = e_k <= bar
    ratio = e_k / bar
    _WORST.append(float(ratio.max()))
    if not ok.all():
        print(f"{what} lse: worst row {int(ratio.argmax())} at {float(ratio.max()):.3f} of its bar; rows failing "
              f"{int((~ok).sum())}/{len(ok)}")
    return ok


OUTPUTS = {"fused": ("out",), "lse": ("o_s",), "dense": ("o_s",), "dense_lse": ("o_s",), "jvp": ("o_s", "out_t"),
           "jvp_lse": ("o_s", "out_t"), "tangent": ("out_t",)}


def _check_common(x, what):
    for name, pad in x.pads.items():
        assert torch.equal(pad, torch.full_like(pad, SENTINEL)), f"{what}: {name} written past its last row"
    for name in OUTPUTS[x.kind] + (("lse",) if x.kind in ("lse", "dense_lse", "jvp_lse") else ()):
        assert torch.isfinite(getattr(x, name).float()).all(), (what, name)


def _check(x, what, q_blocks=None, bh=None):
    """All bars on every (or the sampled) query block of every (or the sampled) (batch, head)."""
    what = f"{what} {x.kind} {str(x.dtype)[6:]}"
    _check_common(x, what)
    bh = [(bi, hi) for bi in range(x.b) for hi in range(x.h)] if bh is None else bh
    q_blocks = range(x.mblk) if q_blocks is None else q_blocks
    for bi, hi in bh:
        for m in q_blocks:
            rows = torch.arange(m * x.blkq, min(x.lq, (m + 1) * x.blkq), device=x.q.device)
            refs = _refs(x, x.kind, bi, hi, rows)
            w = f"{what} b{bi} h{hi} m{m}"
            for name in OUTPUTS[x.kind]:
                block_ok, rows_ok = _judge(getattr(x, name)[bi, rows, hi], refs[name], x.dtype, f"{w} {name}")
                assert block_ok and bool(rows_ok.all()), (w, name, "rows failing", (~rows_ok).nonzero().flatten().tolist()[:16])
            if x.kind in ("lse", "dense_lse", "jvp_lse"):
                ok = _judge_lse(x.lse[bi, hi, rows], refs["lse"], w)
                assert bool(ok.all()), (w, "lse rows failing", (~ok).nonzero().flatten().tolist()[:16])


def _check_kinds(x, kinds, what, **kw):
    for kind in kinds:
        _check(_run(x, kind), what, **kw)


SPARSE_KINDS = {128: ("fused", "lse", "jvp", "jvp_lse", "tangent"), 64: ("fused", "lse")}
DENSE_KINDS = ("dense", "dense_lse", "jvp", "jvp_lse", "tangent")


# ------------------------------------------------------------------------------------------------------------ block-map LUTs
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("blkq", GEOMS)
def test_block_map_luts(cuda, blkq, dtype):
    """The module's selection at b = 2, h = 3, L = 1000: ragged last query block (104 or 40 rows) and last key block (40 keys),
    5 of 16 key blocks per row.  The fused forward with each feature map, the lse forward and, on 128-row blocks, the sparse
    JVP (both entry points) and tangent.  Every block of every head."""
    (q, k, v), tan = _inputs(2, 1000, 1000, 3, dtype, 11)
    lut = B.block_map_lut(q, k, blkq, 5)
    for feature in (0, 1, 2):
        qf = q if feature == 0 else (q.float() * 0.5).to(dtype)
        _check(_run(_case(qf, k, v, lut, blkq, feature=feature), "fused"), f"block map q{blkq} feature {feature}")
    _check_kinds(_case(q, k, v, lut, blkq, tan), SPARSE_KINDS[blkq][1:], f"block map q{blkq}")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("blkq", GEOMS)
@pytest.mark.parametrize("lq,lk", [(333, 1000), (1000, 77)])
def test_fused_lengths_differ(cuda, lq, lk, blkq, dtype):
    """The fused forward at lq != lk (its rows past lq in the sentinel), on the module's selection of a third of the key
    blocks (every one at lk = 77: two key blocks, the second with 13 keys)."""
    (q, k, v), _ = _inputs(1, lq, lk, 2, dtype, 40 + lq)
    nblk = B.cdiv(lk, BK)
    lut = B.block_map_lut(q, k, blkq, max(2, nblk // 3))
    _check(_run(_case(q, k, v, lut, blkq), "fused"), f"{lq}x{lk} q{blkq}")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("lq,lk", [(333, 1000), (1000, 77)])
def test_dense_lengths_differ(cuda, lq, lk, dtype):
    """Dense forward (both entry points), JVP (both) and tangent at lq = 333 / lk = 1000 and lq = 1000 / lk = 77 (fewer keys
    than one tile), b = 2, h = 2: every block of every head, sentinel rows past lq."""
    (q, k, v), tan = _inputs(2, lq, lk, 2, dtype, 60 + lq)
    _check_kinds(_case(q, k, v, None, 128, tan), DENSE_KINDS, f"dense {lq}x{lk}")


# ------------------------------------------------------------------------------------------------------------ hand-made LUTs
R = 7                 # the ragged key block of the hand-made cases: L = 7 * 64 + valid keys, 8 key blocks
HAND = {
    # name: (entries, valid keys of the ragged block)
    "one": ([3], 40), "two": ([2, 5], 40), "three": ([1, 3, 5], 40), "four": ([0, 2, 3, 5], 40),
    "ragged_alone_1": ([R], 1), "ragged_alone_63": ([R], 63),
    "ragged_first_1": ([R, 2, 5], 1), "ragged_first_63": ([R, 2, 5], 63),         # warpgroup 0's first entry
    "ragged_last_1": ([1, 4, R], 1), "ragged_last_63": ([1, 4, R], 63),           # the last entry, warpgroup 0's
    "ragged_wg1_1": ([2, R], 1), "ragged_wg1_63": ([2, R, 5], 63),                # warpgroup 1's only entry
    "permuted": ([5, 0, 6, 2, 7, 3], 40), "descending": ([7, 6, 5, 3, 2, 1], 40),
    # boosted entries (positions in BOOST): the row maximum rises by more than 2^8 (log2) only there
    "rise_wg1": ([0, 1, 2, 3, 4, 5], 40), "rise_wg0": ([0, 1, 2, 3, 4, 5], 40), "rise_next": ([0, 2, 3, 4, 5, 6], 40),
    "rise_last": ([0, 2, 3, 4, 5, 6], 40),
    "negative_first": ([0, 2, 4, 6], 40), "peaked": ([1, 3, 5], 40),
}
BOOST = {"rise_wg1": (3, 5), "rise_wg0": (2, 4), "rise_next": (1,), "rise_last": (5,)}


def _hand_inputs(name, dtype):
    """q, k, v, tangents [1, L, 2, D] and the entries of a HAND case; the scores of the boosted / negative / peaked blocks are
    moved along u = ones / sqrt(d), which every query carries."""
    entries, valid = HAND[name]
    l = R * BK + valid
    (q, k, v), tan = _inputs(1, l, l, 2, torch.float32, 300 + len(name) + valid)
    u = B.U.cuda()
    if name in BOOST or name == "negative_first":
        q, k = q * 0.25 + 6.0 * u, k * 0.25
        for pos in BOOST.get(name, ()):
            k[:, entries[pos] * BK:(entries[pos] + 1) * BK] += 24.0 * u
        if name == "negative_first":
            k[:, entries[0] * BK:(entries[0] + 1) * BK] -= 16.0 * u
    if name == "peaked":                            # one key 8 * 150 / sqrt(d) log2e above the rest
        q, k = q * 0.1 + 8.0 * u, k * 0.25
        k[:, entries[1] * BK + 5] = 150.0 * u
    return [t.to(dtype) for t in (q, k, v)], [t.to(dtype) for t in tan], entries


def _premise(q, k, name, entries, blkq):
    """The scores do what the case is named for (float64, the first query block of head 0)."""
    qs = q[0, :blkq, 0].double() * (SM / LN2)
    lk = k.shape[1]
    ent_max = []
    for e in entries:
        s = qs @ k[0, e * BK:min(lk, (e + 1) * BK), 0].double().t()
        ent_max.append(s.amax(-1))
        if name == "negative_first" and e == entries[0]:
            assert (s.amax(-1) < 0).float().mean() > 0.9
        if name == "peaked" and e == entries[1]:
            top2 = s.topk(2, -1).values
            assert (top2[:, 0] - top2[:, 1] > 130).float().mean() > 0.9
    if name in BOOST:
        ent_max = torch.stack(ent_max, -1)
        boosted = torch.zeros(len(entries), dtype=torch.bool)
        boosted[list(BOOST[name])] = True
        rise = ent_max[:, boosted].amin(-1) - ent_max[:, ~boosted].amax(-1)
        assert (rise > 8).float().mean() > 0.5, rise
        if name.startswith("rise_wg"):   # on 64-row blocks the boosted entries are all one warpgroup's
            assert len({p % 2 for p in BOOST[name]}) == 1
    if name.startswith("ragged"):
        pos = entries.index(R)
        assert lk - R * BK == int(name.split("_")[-1])
        assert pos == {"alone": 0, "first": 0, "last": len(entries) - 1, "wg1": 1}[name.split("_")[1]]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("blkq", GEOMS)
@pytest.mark.parametrize("name", list(HAND))
def test_hand_made_luts(cuda, name, blkq, dtype):
    """topk = 1; the ragged key block alone with 1 and 63 valid keys, first, last, or warpgroup 1's entry; lists of 2, 3 and 4
    entries (the three-slot rings +-1, the pipelined S_{j+1} prologue, the last-entry path); permuted and descending rows;
    maxima that rise by more than 2^8 only in one warpgroup's entries, at the pipelined next step or the last entry; a first
    entry far below the rest; peaked rows (l ~ 1).  b = 1, h = 2, every row of the same list.  The fused and lse forwards
    and, on 128-row blocks, the sparse JVP and tangent."""
    (q, k, v), tan, entries = _hand_inputs(name, dtype)
    _premise(q, k, name, entries, blkq)
    mblk = B.cdiv(q.shape[1], blkq)
    lut = torch.tensor(entries, dtype=torch.int32, device="cuda").expand(1, 2, mblk, len(entries)).contiguous()
    _check_kinds(_case(q, k, v, lut, blkq, tan), SPARSE_KINDS[blkq], f"{name} q{blkq}")


@pytest.mark.parametrize("blkq", GEOMS)
def test_fused_dead_relu_channel_fp16(cuda, blkq):
    """relu feature map with a key channel that is negative on every key (ksum = 0 there, den down to 1e-5): the fp16 row
    scaling of the linear branch's operand under the row bar."""
    (q, k, v), _ = _inputs(1, 1000, 1000, 2, torch.float32, 70)
    k[..., 0] = -k[..., 0].abs() - 0.1
    q, k, v = (t.to(FP16) for t in (q, k, v))
    x = _case(q, k, v, B.block_map_lut(q, k, blkq, 5), blkq, feature=2)
    _run(x, "fused")
    a = torch.relu(q[..., 0].float())
    assert float(x.ksum[..., 0].abs().max()) == 0.0 and bool((a > 0).any())
    _check(x, f"dead relu q{blkq}")


# ------------------------------------------------------------------------------------------------------------ large scores
LARGE = [pytest.param(n, id=n) for n in ("all_x8", "ragged_last", "split_dominant", "split_merge")]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("blkq", GEOMS)
@pytest.mark.parametrize("name", LARGE)
def test_large_score_and_entry_split_inputs(cuda, name, blkq, dtype):
    """The large-score (q scaled by 8 or 12, the maximum in the ragged last key block) and entry-split (row maxima in
    warpgroup 1's entries, 140+ log2 units above warpgroup 0's; both warpgroups rescaling into the merge) inputs of
    sla_backward_oracle, under the row bars: fused and lse forwards and, on 128-row blocks, the sparse JVP and tangent."""
    if name in B.SPLIT:
        q, k, v, lut = B.split_case(name, blkq)
        lut = lut.cuda()
        q, k, v = (t.to(dtype).cuda() for t in (q, k, v))
    else:
        q, k, v, ratio = B.scaled_case(name, blkq)
        q, k, v = (t.to(dtype).cuda() for t in (q, k, v))
        nblk = B.cdiv(q.shape[1], BK)
        lut = B.block_map_lut(q, k, blkq, max(1, min(nblk, int(ratio * nblk))))
    tan = [_randn(t.shape, dtype, 90 + i, 0.25) for i, t in enumerate((q, k, v))]
    _check_kinds(_case(q, k, v, lut, blkq, tan), SPARSE_KINDS[blkq], f"{name} q{blkq}")


def test_slow_ramp_fp16_jvp_and_tangent(cuda):
    """fp16 on the "slow" ramp of the large-tangent tests: the lazily rescaled p |S_t| passes 65504 in some rows (the JVP's
    overflow rescale onto the running maximum), dense (lq = 256, lk = 1000) and sparse over every key block (L = 1000)."""
    ins = [t.to(FP16) for t in LT.ramp_inputs(1, 256, 1000, 2, "slow", seed=1)]
    over, norm, lag, _ = LT.overflow_stats([t.float() for t in ins])
    print(f"slow ramp: rows with p |S_t| > 65504 {over:.3f}, max normalised |P S_t| {norm:.0f}, lag {lag:.2f}")
    assert over > 0.0 and norm < LT.FP16_MAX / 32 and lag > 7.0
    ins = [t.cuda() for t in ins]
    _check_kinds(_case(*ins[:3], None, 128, ins[3:]), DENSE_KINDS, "slow ramp dense")
    sq = [t.cuda() for t in LT.ramp_inputs(1, 1000, 1000, 2, "slow", seed=2)]
    sq = [t.to(FP16) for t in sq]
    over, *_ = LT.overflow_stats([t.float() for t in sq])
    assert over > 0.0
    lut = torch.arange(16, dtype=torch.int32, device="cuda").expand(1, 2, 8, 16).contiguous()
    _check_kinds(_case(*sq[:3], lut, 128, sq[3:]), ("jvp", "jvp_lse", "tangent"), "slow ramp sparse")


# ------------------------------------------------------------------------------------------------------------ full shapes
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("blkq", GEOMS)
def test_shape_a_sampled(cuda, blkq, dtype):
    """Shape A (Wan2.1-1.3B at 480p): L = 32760, 12 heads, top-k 0.1 of 512 key blocks by the module's selection.  First,
    middle and last query blocks of heads 0, 5 and 11: fused and lse forwards and, on 128-row blocks, the sparse JVP and
    tangent."""
    l, h = 32760, 12
    (q, k, v), tan = _inputs(1, l, l, h, dtype, 32760)
    lut = B.block_map_lut(q, k, blkq, 51)
    mblk = B.cdiv(l, blkq)
    _check_kinds(_case(q, k, v, lut, blkq, tan), SPARSE_KINDS[blkq], f"shape A q{blkq}", q_blocks=(0, mblk // 2, mblk - 1),
                 bh=[(0, 0), (0, 5), (0, 11)])


@pytest.mark.parametrize("dtype", DTYPES)
def test_dense_shape_a_cross_attention(cuda, dtype):
    """Shape A cross-attention: 32760 queries over 512 text keys, 12 heads.  First, middle and last query blocks of heads 0,
    5 and 11: dense forward, JVP and tangent."""
    (q, k, v), tan = _inputs(1, 32760, 512, 12, dtype, 77)
    mblk = B.cdiv(32760, 128)
    _check_kinds(_case(q, k, v, None, 128, tan), DENSE_KINDS, "dense shape A cross", q_blocks=(0, mblk // 2, mblk - 1),
                 bh=[(0, 0), (0, 5), (0, 11)])


# ------------------------------------------------------------------------------------------------------------ limits
@pytest.mark.parametrize("blkq", GEOMS)
def test_largest_topk(cuda, blkq):
    """topk = 11,220 (128-row blocks) or 13,952 (64-row blocks), the largest the on-chip LUT takes, every key block of a
    ragged L = 64 topk - 17 listed (the lse forward runs lq = lk = L): fused and lse forwards, bf16, on the ramped inputs of
    the long-list tests so every part of the list carries weight.  The first, a middle and the last query block."""
    topk = FWD_TOPK_LIMIT[blkq]
    l = 64 * topk - 17
    q, k, v = B.long_inputs(l, 1, BF16, topk)
    mblk = B.cdiv(l, blkq)
    lut = torch.arange(topk, dtype=torch.int32, device="cuda").expand(1, 1, mblk, topk).contiguous()
    x = _case(q, k, v, lut, blkq)
    for kind in ("fused", "lse"):
        _run(x, kind)
        print(f"topk {topk} q{blkq} {kind}: {x.seconds:.2f} s")
        _check(x, f"topk {topk} q{blkq}", q_blocks=(0, mblk // 2, mblk - 1))
        _limit_faults(x, f"topk {topk} q{blkq}")


def test_jvp_and_tangent_largest_topk(cuda):
    """The sparse JVP and tangent at topk = 8,640 (jvp::kMaxLutIds: the LUT row fills the last 34,560 bytes of shared memory),
    L = 552,960, every key block listed, bf16, ramped inputs.  The first, a middle and the last query block."""
    topk = JVP_TOPK_LIMIT
    l = 64 * topk
    q, k, v = B.long_inputs(l, 1, BF16, topk)
    tan = [_randn((1, l, 1, D), BF16, 8640 + i, 0.25) for i in range(3)]
    mblk = B.cdiv(l, 128)
    lut = torch.arange(topk, dtype=torch.int32, device="cuda").expand(1, 1, mblk, topk).contiguous()
    x = _case(q, k, v, lut, 128, tan)
    for kind in ("jvp_lse", "tangent"):
        _run(x, kind)
        print(f"topk {topk} {kind}: {x.seconds:.2f} s")
        _check(x, f"topk {topk}", q_blocks=(0, mblk // 2, mblk - 1))
        _limit_faults(x, f"topk {topk}")


def _limit_faults(x, what, m=0):
    """At a limit-length list the row bars still reject, on every row of query block m, a zero output and R64 of a kernel
    that read only the second half of the list (the part the ramp of B.long_inputs weighs most)."""
    rows = torch.arange(m * x.blkq, min(x.lq, (m + 1) * x.blkq), device=x.q.device)
    out = OUTPUTS[x.kind][-1]
    ref = _refs(x, x.kind, 0, 0, rows)[out]
    half = x.lut[0, 0, m, x.lut.shape[-1] // 2:]
    for name, bad in (("zero output", torch.zeros_like(ref[0])),
                      ("first half of the list dropped", _refs(x, x.kind, 0, 0, rows, lut_row=half)[out][0])):
        _, rows_ok = _judge(bad.to(x.dtype), ref, x.dtype, f"{what} {x.kind} fault: {name}", record=None)
        assert not bool(rows_ok.any()), (what, x.kind, name, int(rows_ok.sum()))


@pytest.mark.parametrize("blkq", GEOMS)
def test_largest_key_block_count(cuda, blkq):
    """nblk = 65,535 (L = 4,194,240, h = 1, bf16), every LUT row {0, 32767, 32768, 65534}: ids past 32767 through the
    producers' uint16 LUT.  The lse forward (lq = L) on sampled query blocks, and the fused forward on 300 query rows."""
    l = 64 * 65535
    ids = [0, 32767, 32768, 65534]
    q, k, v = (_randn((1, l, 1, D), BF16, 65535 + i) for i in range(3))
    lut = torch.tensor(ids, dtype=torch.int32, device="cuda").expand(1, 1, B.cdiv(l, blkq), 4).contiguous()
    x = _run(_case(q, k, v, lut, blkq), "lse")
    _check(x, f"nblk 65535 q{blkq}", q_blocks=(0, 1, x.mblk // 2, x.mblk - 1))
    x = _case(q[:, :300], k, v, lut[:, :, :B.cdiv(300, blkq)].contiguous(), blkq)
    _check(_run(x, "fused"), f"nblk 65535 q{blkq}")


# ------------------------------------------------------------------------------------------------------------ exact properties
def _counter_inputs(b, lq, lk, h, dtype):
    """q = q_t = k_t = 0, so every score and score tangent is 0 and p = exp2(0) = 1 exactly; v and v_t channel c < 20 = bit c
    of the key index, channel 20 + i = key index mod (i + 2) (i < 8), the rest 1: every P.V sum is a small integer, exact in
    fp32."""
    j = torch.arange(lk, device="cuda")
    cols = [(j >> c) & 1 for c in range(20)] + [j % (i + 2) for i in range(8)]
    cols += [torch.ones_like(j)] * (D - len(cols))
    v = torch.stack(cols, -1).to(dtype)[None, :, None].expand(b, lk, h, D).contiguous()
    z = torch.zeros(b, lq, h, D, dtype=dtype, device="cuda")
    k = _randn((b, lk, h, D), dtype, 5)
    return z, k, v, (z, torch.zeros_like(k), v)


def _counts(x, kind, bi, hi, m):
    """The exact sum of v over the keys query block m reads, and their number ([d] float64, int)."""
    starts, tw, _ = _tiles_of(x, kind, bi, hi, m)
    keys = (starts[:, None] + torch.arange(tw, device="cuda")).flatten()
    keys = keys[keys < x.lk]
    return x.v[bi, keys, hi].double().sum(0), len(keys)


def _counter_check(x, name, exact=True):
    """o (and out_t) of every row of block m = T(fl(count fl(1/n))), bit for bit; the tangent (exact=False): there is one
    rounded P per row, t in {T(1/n) and its two neighbours}, with out_t = T(count t)."""
    for bi in range(x.b):
        for hi in range(x.h):
            for m in range(x.mblk):
                rows = torch.arange(m * x.blkq, min(x.lq, (m + 1) * x.blkq), device="cuda")
                cnt, n = _counts(x, x.kind, bi, hi, m)
                inv = float(torch.tensor(1.0 / n, dtype=F32))
                want = (cnt.float() * inv).to(x.dtype)
                for nm in OUTPUTS[x.kind]:
                    got = getattr(x, nm)[bi, rows, hi]
                    if exact:
                        assert bool((got == want).all()), (name, nm, bi, hi, m, n)
                        continue
                    bits = torch.tensor([1.0 / n], dtype=F32).to(x.dtype).view(torch.int16)   # T(1/n) and its T neighbours
                    ok = torch.zeros(len(rows), dtype=torch.bool, device="cuda")
                    for t in (bits - 1, bits, bits + 1):
                        t = t.view(x.dtype)
                        ok |= (got == (cnt.float() * float(t.float())).to(x.dtype)).all(-1)
                    assert bool(ok.all()), (name, nm, bi, hi, m, n)


@pytest.mark.parametrize("blkq", GEOMS)
def test_key_counter(cuda, blkq):
    """q = 0 (and q_t = k_t = 0): o_s, the fused out (kvw = proj_b = 0), o and out_t of every row are T(count / n) with the
    kernel's reciprocal-and-multiply epilogue, bit for bit, where count sums the small-integer channels of v (and v_t) over
    exactly the keys the row's list names: LUT entries in any order, the ragged block's 1 or 40 valid keys, both
    warpgroups' shares on 64-row blocks, keys < lk for dense.  The tangent reads the lse the forward wrote."""
    for dtype in (BF16, FP16):
        for l in (7 * 64 + 1, 1000):
            q, k, v, tan = _counter_inputs(2, l, l, 3, dtype)
            nblk, mblk = B.cdiv(l, BK), B.cdiv(l, blkq)
            g = torch.Generator().manual_seed(l + blkq)
            lut = torch.stack([torch.randperm(nblk, generator=g)[:5] for _ in range(2 * 3 * mblk)]).view(2, 3, mblk, 5)
            lut[..., 0] = nblk - 1                          # the ragged block in every list
            lut = lut.int().cuda()
            x = _case(q, k, v, lut, blkq, tan)
            x.kvw = torch.zeros(2, 3, D, D, dtype=dtype, device="cuda")
            x.ksum = torch.ones(2, 3, D, dtype=F32, device="cuda")
            x.proj_b = torch.zeros(D, dtype=F32, device="cuda")
            for kind in SPARSE_KINDS[blkq]:
                _counter_check(_run(x, kind), f"q{blkq} {kind} L{l}", exact=kind != "tangent")
            if blkq == 128:
                for lq, lk in ((333, 1000), (1000, 77)):
                    q, k, v, tan = _counter_inputs(1, lq, lk, 2, dtype)
                    x = _case(q, k, v, None, 128, tan)
                    for kind in DENSE_KINDS:
                        _counter_check(_run(x, kind), f"dense {kind} {lq}x{lk}", exact=kind != "tangent")


@pytest.mark.parametrize("blkq", GEOMS)
def test_power_of_two_v_bf16(cuda, blkq):
    """bf16: scaling v by 2^s (and v_t, and the out the tangent reads) scales o_s, o and out_t by 2^s bit for bit, s from -40
    to 40, on randn inputs and the module's selection (on 128-row blocks the sparse JVP and tangent too; dense at
    333 x 1000)."""
    (q, k, v), tan = _inputs(1, 1000, 1000, 2, BF16, 31)
    cases = [(_case(q, k, v, B.block_map_lut(q, k, blkq, 5), blkq, tan), ("lse",) + SPARSE_KINDS[blkq][2:])]
    if blkq == 128:
        (qd, kd, vd), tand = _inputs(1, 333, 1000, 2, BF16, 32)
        cases.append((_case(qd, kd, vd, None, 128, tand), DENSE_KINDS))
    for x, kinds in cases:
        base = {}
        for kind in kinds:
            _run(x, kind)
            base[kind] = {n: getattr(x, n).clone() for n in OUTPUTS[kind]}
            base[kind]["src"] = x.o_s.clone() if kind == "tangent" else None
        v0, vt0 = x.v, x.vt
        for s in (-40, -17, -1, 3, 40):
            x.v = (v0.double() * 2.0 ** s).to(BF16)
            x.vt = (vt0.double() * 2.0 ** s).to(BF16)
            for kind in kinds:
                _run(x, kind)
                if kind == "tangent":   # the out the tangent reads is the scaled forward's
                    assert torch.equal(x.o_s.double(), base[kind]["src"].double() * 2.0 ** s)
                for n in OUTPUTS[kind]:
                    assert torch.equal(getattr(x, n).double(), base[kind][n].double() * 2.0 ** s), (kind, n, s)
        x.v, x.vt = v0, vt0


# ------------------------------------------------------------------------------------------------------------ sensitivity
def _old_bar(got, want):
    a, b = got.double().flatten(), want.flatten()
    rel = float((a - b).norm() / b.norm())
    cos = float(torch.dot(a, b) / (a.norm() * b.norm()))
    return cos >= 0.9999 and rel <= 5e-3


def _merge_fault(x, bi, hi, rows):
    """R64 of the 64-row kernel whose merge scales warpgroup 1's state with warpgroup 0's exponent: O = O0 a0 + O1 a0."""
    starts, tw, _ = _tiles_of(x, "lse", bi, hi, int(rows[0]) // x.blkq)
    parts = []
    for g in (0, 1):
        keys = (starts[g::2, None] + torch.arange(tw, device="cuda")).flatten()
        keys = keys[keys < x.lk]
        s = (x.q[bi, rows, hi].double() @ x.k[bi, keys, hi].double().t()) * (SM / LN2)
        m = s.amax(-1, keepdim=True)
        p = torch.exp2(s - m)
        parts.append((m, p.sum(-1, keepdim=True), p @ x.v[bi, keys, hi].double()))
    (m0, l0, o0), (m1, l1, o1) = parts
    a0 = torch.exp2(m0 - torch.maximum(m0, m1))
    return (o0 * a0 + o1 * a0) / (l0 * a0 + l1 * a0)


@pytest.mark.parametrize("blkq", GEOMS)
def test_bars_reject_kernel_faults(cuda, blkq):
    """R64 as faulty kernels would compute it (rounded to T as their output would be), judged by the row bars: each must fail
    on at least half of the rows it changes.  Prints whether the whole-tensor bars in use today (cos >= 0.9999, rel-L2 <=
    5e-3 on the block) accept each.  L = 1000, bf16, b = 1, h = 2; the list of query block 2 holds 6 key blocks, the ragged
    one last.  The fused forward's den fault runs on keys whose channel 0 dominates ksum and queries whose odd rows put
    phi(q) on that channel, so that neighbouring rows' den differ severalfold (on randn inputs they agree to a few percent,
    and a kernel that swapped them would be within rounding of the right one).  The JVP whose mu sums T(p) S_t instead of
    the unrounded p S_t runs on _mu_case, where T(p) - p has one sign on every key that carries S_t (on randn inputs the
    shift sum (T(p) - p) S_t / l o is a sum of roundings of either sign, within the kernel's own rounding of A)."""
    l, h = 1000, 2
    (q, k, v), tan = _inputs(1, l, l, h, BF16, 41)
    nblk = B.cdiv(l, BK)
    entries = [0, 3, 5, 8, 11, nblk - 1]
    mblk = B.cdiv(l, blkq)
    lut = torch.tensor(entries, dtype=torch.int32, device="cuda").expand(1, h, mblk, 6).contiguous()
    m, hi = 2, 1
    rows = torch.arange(m * blkq, (m + 1) * blkq, device="cuda")
    nbr = m * blkq + ((rows - m * blkq) ^ 1)
    x = _case(q, k, v, lut, blkq, tan)
    _run(x, "lse")
    # the fused forward on keys whose channel 0 dominates ksum, and queries whose odd rows put phi on it: den of neighbouring
    # rows differs severalfold
    xf = _case((q.float() + 4.0 * (torch.arange(l, device="cuda") % 2)[None, :, None, None] * (torch.arange(D, device="cuda") == 0))
               .to(BF16), (k.float() + 3.0 * (torch.arange(D, device="cuda") == 0)).to(BF16), v, lut, blkq)
    _run(xf, "fused")
    phi = torch.softmax(xf.q[0, rows, hi].double(), -1)
    den = phi @ xf.ksum[0, hi].double()
    assert float((den / den[(rows - m * blkq) ^ 1]).log2().abs().median()) > 1.0
    faults = {  # name: (inputs, kind, output, rows, faulty R64)
        "dropped entry of warpgroup 1's share" if blkq == 64 else "dropped entry":
            (x, "lse", "o_s", rows, lambda: _refs(x, "lse", 0, hi, rows, lut_row=entries[:3] + entries[4:])["o_s"][0]),
        "ragged block's last valid key masked":
            (x, "lse", "o_s", rows, lambda: _refs(x, "lse", 0, hi, rows, drop_keys=lambda kk: kk == l - 1)["o_s"][0]),
        "row normalised by its neighbour's l":
            (x, "lse", "o_s", rows, lambda: _neighbour_l(x, 0, hi, rows, nbr)),
        "fused den of the neighbour row":
            (xf, "fused", "out", rows, lambda: _neighbour_den(xf, 0, hi, rows, nbr)),
    }
    if blkq == 64:
        faults["warpgroup 1 merged with warpgroup 0's exponent"] = (x, "lse", "o_s", rows, lambda: _merge_fault(x, 0, hi, rows))
    else:
        xt = _run(_case(q, k, v, lut, blkq, tan), "tangent")
        faults["tangent reading the next row's out"] = (xt, "tangent", "out_t", rows,
                                                        lambda: _tangent_fault(xt, 0, hi, rows, out_rows=nbr))
        faults["tangent reading the other head's lse"] = (xt, "tangent", "out_t", rows,
                                                          lambda: _tangent_fault(xt, 0, hi, rows, head=1 - hi))
        xm = _mu_case()
        _check(_run(xm, "jvp"), "mu case")           # the right kernel meets the bars there
        rows0 = torch.arange(0, 128, device="cuda")
        faults["JVP mu summed from T(p) S_t"] = (xm, "jvp", "out_t", rows0, lambda: _mu_fault(xm, 0, hi, rows0))
    accepted = []
    for name, (src, kind, out, idx, faulty) in faults.items():
        ref = _refs(src, kind, 0, hi, idx)[out]
        bad = faulty().to(BF16)
        changed = (bad.double() != ref[0].to(BF16).double()).any(-1)
        _, rows_ok = _judge(bad, ref, BF16, f"q{blkq} fault: {name}", record=None)
        rejected = int((~rows_ok & changed).sum())
        assert int(changed.sum()) > 0 and rejected >= 0.5 * int(changed.sum()), (name, rejected, int(changed.sum()))
        old = _old_bar(bad, ref[0])
        print(f"q{blkq} {name}: row bars reject {rejected}/{int(changed.sum())} changed rows; the whole-tensor bar "
              f"{'accepts' if old else 'rejects'} it")
        if old:
            accepted.append(name)
    print(f"q{blkq}: faults the whole-tensor bars accept: {accepted}")


def _neighbour_l(x, bi, hi, rows, nbr):
    """o_s of rows normalised by their neighbour row's l (the same maximum: the unnormalised sums of both against one m)."""
    keys = _counts_keys(x, bi, hi, rows)
    s = (x.q[bi, rows, hi].double() @ x.k[bi, keys, hi].double().t()) * (SM / LN2)
    sn = (x.q[bi, nbr, hi].double() @ x.k[bi, keys, hi].double().t()) * (SM / LN2)
    mx = torch.maximum(s.amax(-1, keepdim=True), sn.amax(-1, keepdim=True))
    return (torch.exp2(s - mx) @ x.v[bi, keys, hi].double()) / torch.exp2(sn - mx).sum(-1, keepdim=True)


def _counts_keys(x, bi, hi, rows):
    starts, tw, _ = _tiles_of(x, "lse", bi, hi, int(rows[0]) // x.blkq)
    keys = (starts[:, None] + torch.arange(tw, device="cuda")).flatten()
    return keys[keys < x.lk]


def _neighbour_den(x, bi, hi, rows, nbr):
    r64 = _refs(x, "fused", bi, hi, rows)["out"][0]
    phi, phin = _phi(x.q[bi, rows, hi].double(), 0), _phi(x.q[bi, nbr, hi].double(), 0)
    ks, kvw = x.ksum[bi, hi].double(), x.kvw[bi, hi].double()
    lin = phi @ kvw.t()
    return r64 - lin / (phi @ ks + 1e-5)[:, None] + lin / (phin @ ks + 1e-5)[:, None]


def _tangent_fault(x, bi, hi, rows, out_rows=None, head=None):
    """R64 of a tangent kernel reading another row's out (out_t = A - mu out[nbr]) or another head's lse (P = exp2(s - lse'))."""
    keys = _counts_keys(x, bi, hi, rows)
    q, qt = x.q[bi, rows, hi].double(), x.qt[bi, rows, hi].double()
    kc, ktc = x.k[bi, keys, hi].double(), x.kt[bi, keys, hi].double()
    vc, vtc = x.v[bi, keys, hi].double(), x.vt[bi, keys, hi].double()
    s = (q @ kc.t()) * (SM / LN2)
    st = SM * (qt @ kc.t() + q @ ktc.t())
    if head is None:
        p = torch.softmax(s * LN2, -1)
    else:
        p = torch.exp2(s - x.lse[bi, head, rows].double()[:, None])
    a = (p * st) @ vc + p @ vtc
    mu = (p * st).sum(-1, keepdim=True)
    o = torch.softmax(s * LN2, -1) @ vc if out_rows is None else x.o_s[bi, out_rows, hi].double()
    return a - mu * o


def _mu_case():
    """Sparse JVP inputs (bf16, L = 128, h = 2, LUT [1, 0]) on which a mu summed from T(p) S_t moves out_t past rounding:
    every query is e_0, so the scores are k[:, 0] sm log2e.  Key block 1 (listed first: it sets the maximum) has
    k[:, 0] = 1 + 2^-6, so p = 1, S_t = 0 and v = v0 + noise; key block 0 has k[:, 0] = 1 or 1 + 2^-7, so p = 0.99862 or
    0.99931, which bf16 rounds up to 1, S_t = 8 sm (k_t[:, 0] = 8, q_t = 0) and v = 0.  Then T(p) - p > 0 wherever S_t is,
    the kernel's A = sum T(p S_t) v + T(p) v_t has no rounding of a p below 1 in it, and v_t of block 1 = T(mu v) cancels
    -mu o to a bf16 rounding: out_t is small, and (mu' - mu) o is several times larger."""
    l, h = 128, 2
    dev = "cuda"
    keys = torch.arange(l, device=dev)
    a = keys < 64
    q = torch.zeros(1, l, h, D, device=dev)
    q[..., 0] = 1.0
    k = B.randn((1, l, h, D), F32, 801)
    k[..., 0] = torch.where(a, 1.0 + 2.0 ** -7 * (keys % 2), torch.full_like(keys, 1.0 + 2.0 ** -6, dtype=F32))[None, :, None]
    kt = B.randn((1, l, h, D), F32, 802)
    kt[..., 0] = torch.where(a, 8.0, 0.0)[None, :, None]
    v = (B.randn((1, 1, h, D), F32, 803) + 0.25 * B.randn((1, l, h, D), F32, 804)) * (~a)[None, :, None, None]
    p = torch.exp2((k[0, :, 0, 0].double() - 1.0 - 2.0 ** -6) * SC32)
    st = SM * kt[0, :, 0, 0].double()
    mu = float((p * st).sum() / p.sum())
    vt = mu * v
    q, k, v, kt, vt = (t.to(BF16) for t in (q, k, v, kt, vt))
    pa = p[a]
    assert bool((pa < 1).all() and (pa.to(BF16) == 1).all() and (p[~a] == 1).all()), "p rounds up wherever S_t is"
    lut = torch.tensor([1, 0], dtype=torch.int32, device=dev).expand(1, h, 1, 2).contiguous()
    return _case(q, k, v, lut, 128, (torch.zeros_like(q), kt, vt))


def _mu_fault(x, bi, hi, rows):
    """R64 of a JVP whose mu sums T(p) S_t (p against the row maximum) instead of the unrounded p S_t."""
    keys = _counts_keys(x, bi, hi, rows)
    q, qt = x.q[bi, rows, hi].double(), x.qt[bi, rows, hi].double()
    kc, ktc = x.k[bi, keys, hi].double(), x.kt[bi, keys, hi].double()
    vc, vtc = x.v[bi, keys, hi].double(), x.vt[bi, keys, hi].double()
    s = (q @ kc.t()) * (SM / LN2)
    st = SM * (qt @ kc.t() + q @ ktc.t())
    p = torch.exp2(s - s.amax(-1, keepdim=True))
    l = p.sum(-1, keepdim=True)
    o = p @ vc / l
    mu = (p.to(BF16).double() * st).sum(-1, keepdim=True) / l
    return ((p * st) @ vc + p @ vtc) / l - mu * o
