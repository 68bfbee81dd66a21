"""The INT8 SageSLA forwards (tdb200_sla_attn_fwd: sla_attn_fwd_kernel on 128 x 64 blocks, sla_attn_fwd_q64_kernel on 64 x 128)
against float64 on the kernel's own inputs, query block by query block and row by row.

Both references start from what the kernel is given: the INT8 codes and scales of tdb200_sla_quant_qk, the 16-bit q and v,
kvw, ksum and proj_b.  So INT8 quantisation is not an error here, and the moments have float64 tests of their own.
  * float64: s = (q_i8 . k_i8^T) q_scale[row block] k_scale[key block] sm_scale on the LUT's keys < lk, softmax . V, plus
    phi(q) . kvw^T / (phi(q) . ksum + 1e-5) + proj_b with phi of the 16-bit q.
  * the float32 restatement at the kernel's rounding points: sc = fl(fl(q_scale sm_scale) log2e) k_scale (sla_attn.cu, qsc
    times s_ksc), s = fl(float(acc) sc), p = exp2(fl(s - m)) with m the exact row maximum, the row sum from the unrounded p,
    P rounded to T for P.V, the linear-branch operand A = T(phi l / den) (in fp16 with the kernel's power-of-two range
    scaling), and the output rounded to T.
Bars, fixed from those rounding points: per (batch, head, query block) rel-L2 against float64 <= 1.5x the restatement's;
per row <= 2x max(the restatement's plus 2^-24 per P.V MMA step, the row's own rounding |T(ref) - ref| / |ref|); all finite, and the rows >= lq of a
sentinel-filled buffer untouched.  test_bars_reject_a_wrong_scale_entry_or_key shows what those bars catch that the
cosine >= 0.999 / rel-L2 <= 2e-2 bars of the other SageSLA tests let pass.

The FP8 P.V forwards (tdb200_sla_attn_fwd_fp8v on the codes and channel scales of tdb200_sla_quant_v_fp8, "-fp8" in the
test ids; d = 128 only) run the same cases.  Their restatement rounds P and reads V as e4m3 where the kernel does.  Bars:
  (a) the ones above against float64, with the e4m3 restatement and the chain allowance below in place of 2^-24 per step;
  (b) faithfulness, per row, relative to the row's float64 norm: |kernel - R32| <= 2 |T(R32) - R32| + flip + chain, R32 the
      restatement before its rounding to T.  flip: each P within FLIP_REL (ex2.approx against torch's exp2) of an e4m3
      rounding midpoint adds one e4m3 step times |v| / l.  chain: per key block, 2^-CHAIN_BITS (the e4m3 wgmma chain's
      accumulation width) plus 2^-24 (the block's fp32 add into O) times sum |p v| / l.
test_fp8_chain_accumulation_width measures the chain's width through the kernel and holds it to CHAIN_BITS.
"""
import math

import pytest
import torch

import sla_backward_oracle as B

pytestmark = pytest.mark.gpu

FAMILIES = {"sm100": (128, 64), "sm90": (64, 128)}   # (BLKQ, BLKK): sla_attn_fwd_kernel, sla_attn_fwd_q64_kernel
DTYPES = {"bf16": torch.bfloat16, "fp16": torch.float16}
FEATURES = {"softmax": 0, "elu": 1, "relu": 2}
LOG2E32 = torch.tensor(1.4426950408889634, dtype=torch.float32)   # kLog2e as the kernel holds it
PAD_ROWS = 37          # rows of the buffer after the output, which the kernel must leave alone
SENTINEL = -1234.0     # exact in bf16 and fp16
CHUNK = 1 << 16        # keys per float64 score tile of the references
ERR_UNSUPPORTED = -2   # TDB200_ERR_UNSUPPORTED
E4M3 = torch.float8_e4m3fn
# ex2.approx.ftz.f32 (the kernel's P) and exp2f (torch's, which the restatement's P comes from) each within 2 ulp of 2^x
FLIP_REL = 2.0 ** -21
# The e4m3 wgmma chain's relative accumulation error is at most 2^-CHAIN_BITS of sum |p v| (test_fp8_chain_accumulation_width).
# On an H100 80GB HBM3 (700 W limit) that probe measured 9.996 bits (128 x 64) and 9.9995 (64 x 128): the chain truncates
# each product to 13 bits below the leading bit of the K = 32 step's largest one (a 14-bit significand), so 30 products
# just under that grid beside +-448 are lost whole, 2^-9.996 of the sum.
CHAIN_BITS = 9

# (d, P.V) and (family, P.V): the 16-bit P.V cases keep their ids, the FP8 ones add "-fp8" (d = 128 only)
D_PV = [pytest.param(128, "bf16", id="128"), pytest.param(64, "bf16", id="64"), pytest.param(128, "fp8", id="128-fp8")]
FAMILY_PV = [pytest.param(f, pv, id=f + ("-fp8" if pv == "fp8" else "")) for pv in ("bf16", "fp8") for f in sorted(FAMILIES)]

# ------------------------------------------------------------------------------------------------------------ top-k limits
# launch() refuses a LUT whose on-chip copy does not fit: 1024 (alignment) + Lay::kOffLut + round16(2 topk) (uint16 ids)
# + 4 topk (k_scale of each entry) <= 227 KB.  Lay (INT8 Q/K): Q BQ*HD | 3 K stages BK*HD | 3 V stages BK*HD*2 (e4m3: BK*HD)
# | KVW HD*HD*2 | 16-bit Q rows BQ*HD*2 | 256 B of barriers.
#   128x64, d=128:  16384 + 3*8192 + 3*16384 + 32768 + 32768 + 256 = 155904; 232448 - 1024 - 155904 = 75520 = 6*12584 + 16
#   128x64, d=64:    8192 + 3*4096 + 3*8192 + 8192 + 16384 + 256 = 69888;    161536 -> 6*26920 = 161520
#   64x128, d=128:   8192 + 3*16384 + 3*32768 + 32768 + 16384 + 256 = 205056; 26368 -> 6*4392 = 26352
#   64x128, d=64:    4096 + 3*8192 + 3*16384 + 8192 + 8192 + 256 = 94464;    136960 -> 6*22824 = 136944
#   FP8 P.V (d=128 only), V stages of BK*HD bytes:
#   128x64:         16384 + 3*8192 + 3*8192 + 32768 + 32768 + 256 = 131328;  100096 -> 6*16680 = 100080
#   64x128:          8192 + 3*16384 + 3*16384 + 32768 + 16384 + 256 = 155904; 75520 -> 6*12584 = 75504
# In each case topk + 1 needs 6 (topk + 1) + 16 bytes more than there are (round16 of 2 topk + 2 rounds up by 14).
TOPK_LIMIT = {("sm100", 128): 12584, ("sm100", 64): 26920, ("sm90", 128): 4392, ("sm90", 64): 22824}
TOPK_LIMIT_FP8 = {"sm100": 16680, "sm90": 12584}


def _lay_lut_offset(hd, bq, bk, fp8v=False):
    v_bytes = bk * hd if fp8v else bk * hd * 2
    return bq * hd + 3 * bk * hd + 3 * v_bytes + hd * hd * 2 + bq * hd * 2 + 256


def _largest_topk(hd, bq, bk, fp8v=False):
    room = 227 * 1024 - 1024 - _lay_lut_offset(hd, bq, bk, fp8v)
    t = room // 6
    while ((2 * t + 15) & ~15) + 4 * t > room:
        t -= 1
    return t


# ------------------------------------------------------------------------------------------------------------ inputs
CONTRAST = [0, 2, -2, 1, -1]   # log2 magnitude of successive blocks: neighbours differ by up to 2^4


def _contrast(x, blk, shift):
    """x [b, l, h, d] with block i of `blk` rows of (batch bi, head hi) scaled by 2^CONTRAST[(i + 3 bi + hi + shift) % 5]."""
    b, l, h, _ = x.shape
    i = torch.arange(l, device=x.device) // blk
    e = torch.tensor(CONTRAST, dtype=x.dtype, device=x.device)
    idx = (i[None, :, None] + 3 * torch.arange(b, device=x.device)[:, None, None]
           + torch.arange(h, device=x.device)[None, None, :] + shift) % len(CONTRAST)
    return x * torch.exp2(e[idx])[..., None]


def _qkv(b, lq, lk, h, d, seed, dev, family=None, contrast=True, v_contrast=False):
    """Float32 q [b, lq, h, d], k, v [b, lk, h, d] on `dev`, keys with a channel mean; with `contrast`, per-block magnitudes
    that vary by 2^-2..2^2 over the family's query and key blocks; with `v_contrast`, V channel c of (batch bi, head hi)
    scaled by 2^CONTRAST[(c + 3 bi + hi) % 5], so that a channel scale read from the pair neighbour, the next head or the
    next batch is off by 2x or more."""
    g = torch.Generator(device=dev).manual_seed(seed)
    q = torch.randn(b, lq, h, d, generator=g, device=dev)
    k = torch.randn(b, lk, h, d, generator=g, device=dev) + torch.randn(1, 1, h, d, generator=g, device=dev) * 2.0
    v = torch.randn(b, lk, h, d, generator=g, device=dev)
    if contrast:
        blkq, blkk = FAMILIES[family]
        q, k = _contrast(q, blkq, 0), _contrast(k, blkk, 1)
    if v_contrast:
        e = torch.tensor(CONTRAST, dtype=v.dtype, device=dev)
        idx = (torch.arange(d, device=dev)[None, None, :] + 3 * torch.arange(b, device=dev)[:, None, None]
               + torch.arange(h, device=dev)[None, :, None]) % len(CONTRAST)
        v = v * torch.exp2(e[idx])[:, None]
    return q, k, v


class Inputs:
    """What tdb200_sla_attn_fwd (tdb200_sla_attn_fwd_fp8v when pv == "fp8") is given (GPU tensors), and the call's sizes."""


def _prepare(q, k, v, family, dtype, feature=0, seed=9, pv="bf16", proj=None):
    """pv = "fp8": also v_fp8, v_scale of tdb200_sla_quant_v_fp8 and v_codes, v_fp8 with its keys in plain order.
    proj = (weight [d, d], bias [d]): proj_l's parameters instead of random ones."""
    from turbodiffusion_b200.SLA.core import linear_moments, project_moments
    from turbodiffusion_b200.SLA.utils import quant_qk
    x = Inputs()
    x.blkq, x.blkk = FAMILIES[family]
    x.family, x.dtype, x.feature, x.pv = family, dtype, feature, pv
    x.q, x.k, x.v = (t.to(dtype).contiguous() for t in (q, k, v))
    x.b, x.lq, x.h, x.d = x.q.shape
    x.lk = x.k.shape[1]
    x.prep = quant_qk(x.q, x.k, x.lk, x.blkq, x.blkk)
    x.mblk, x.nblk = x.prep.mblk, x.prep.nblk
    kv, x.ksum = linear_moments(x.k, x.v, feature)
    if proj is None:
        g = torch.Generator().manual_seed(seed)
        w = (torch.randn(x.d, x.d, generator=g) * 0.05).to(q.device)
        x.proj_b = (torch.randn(x.d, generator=g) * 0.05).float().to(q.device).contiguous()
    else:
        w, x.proj_b = proj[0].float().contiguous(), proj[1].float().contiguous()
    x.kvw = project_moments(w, kv, dtype)
    x.sm_scale = x.d ** -0.5
    if pv == "fp8":
        _quant_v(x)
    return x


def _quant_v(x):
    from turbodiffusion_b200 import _ops
    x.v_fp8, x.v_scale = _ops.sla_quant_v_fp8(x.v, x.lk, x.blkk)
    x.v_codes = x.v_fp8[..., torch.argsort(_key_of_position(x.v_fp8.shape[-1])).to(x.v.device)]


def _block_map_lut(x, topk):
    from turbodiffusion_b200.SLA.utils import block_map_from_pools
    return block_map_from_pools(x.prep.q_pool, x.prep.k_pool, min(topk, x.nblk))[1]


def _hand_lut(x, entries):
    return torch.tensor(entries, dtype=torch.int32, device=x.q.device).view(1, 1, 1, -1).expand(
        x.b, x.h, x.mblk, len(entries)).contiguous()


def _run(x, lut, k_seq_major=False, lk=None, topk=None):
    """One tdb200_sla_attn_fwd (or tdb200_sla_attn_fwd_fp8v) call into a buffer PAD_ROWS rows longer than the output,
    filled with SENTINEL.  Returns (return code, out [b, lq, h, d], pad rows)."""
    from turbodiffusion_b200._lib import DTYPE_TAG, lib, ptr, stream_ptr
    lk = x.lk if lk is None else lk
    topk = lut.shape[-1] if topk is None else topk
    k_i8 = x.prep.k_i8.permute(0, 2, 1, 3).contiguous() if k_seq_major else x.prep.k_i8
    n = x.b * x.lq * x.h * x.d
    buf = torch.full((n + PAD_ROWS * x.h * x.d,), SENTINEL, dtype=x.dtype, device=x.q.device)
    head = (ptr(x.prep.q_i8), ptr(x.prep.q_scale), ptr(k_i8), ptr(x.prep.k_scale))
    tail = (ptr(x.q), DTYPE_TAG[x.dtype], ptr(lut), topk, ptr(x.kvw), ptr(x.ksum), ptr(x.proj_b), ptr(buf), x.b, x.lq, lk, x.h,
            x.d, x.sm_scale, x.feature, x.blkq, x.blkk, int(k_seq_major), stream_ptr(x.q.device))
    if x.pv == "fp8":
        rc = lib().tdb200_sla_attn_fwd_fp8v(*head, ptr(x.v_fp8), ptr(x.v_scale), *tail)
    else:
        rc = lib().tdb200_sla_attn_fwd(*head, ptr(x.v), *tail)
    torch.cuda.synchronize()
    return rc, buf[:n].view(x.b, x.lq, x.h, x.d), buf[n:]


_last_error = B.last_error


# ------------------------------------------------------------------------------------------------------------ references
_phi = B.phi


def _flip_step(p):
    """For P (float32, >= 0): one e4m3 step where P lies within FLIP_REL of a rounding midpoint of e4m3 (so the kernel's
    ex2.approx and torch's exp2 may round it to neighbouring codes), else 0.  e4m3 steps: 2^(e - 3) in [2^e, 2^(e + 1)),
    2^-9 below 2^-6 (subnormals)."""
    pd = p.double()
    step = torch.exp2(torch.floor(torch.log2(pd.clamp_min(2.0 ** -126))).clamp_min(-6) - 3)
    r = pd / step
    near = (r - torch.floor(r) - 0.5).abs() * step <= FLIP_REL * pd
    return torch.where(near, step, torch.zeros_like(step))


def _references(x, bi, hi, rows, entries, q_scale=None, entry_k_scale=None, key_limit=None, fp8=None, p_dtype=E4M3,
                l_from_rounded_p=False):
    """(float64 reference, float32 restatement, fp8 terms) of query rows `rows` (one query block) of batch bi, head hi over
    the key blocks `entries`, [len(rows), d] float64.  The keyword arguments replace what the kernel would read (the
    sensitivity tests): the row block's q_scale, each entry's k_scale, the number of keys.  fp8 = (v_fp8 in key order
    [d, lk_pad], v_scale [d]): the restatement rounds P to p_dtype (e4m3, as tdb200_sla_attn_fwd_fp8v does) and reads V as
    e4m3, and the fp8 terms are {"r32": the restatement before its rounding to T, "flip", "chain": bar (b)'s allowances
    [len(rows), d] in output units}; without fp8 they are None.  l_from_rounded_p: l summed from the rounded P."""
    dev, bk, d = x.q.device, x.blkk, x.d
    rows = rows.to(dev)
    entries = torch.as_tensor(entries, dtype=torch.int64, device=dev)
    m = int(rows[0]) // x.blkq
    qs = float(x.prep.q_scale[bi, hi, m]) if q_scale is None else float(q_scale)
    eks = x.prep.k_scale[bi, hi, entries] if entry_k_scale is None else torch.as_tensor(entry_k_scale, device=dev)
    key_limit = x.lk if key_limit is None else key_limit
    keys = (entries[:, None] * bk + torch.arange(bk, device=dev)).flatten()    # BK keys per entry, CHUNK a multiple of BK
    kscale = eks.float().repeat_interleave(bk)
    dead = keys >= key_limit
    keys = keys.clamp_max(x.lk - 1)

    qi = x.prep.q_i8[bi, hi, rows].double()
    sc_q = (torch.tensor(qs, dtype=torch.float32) * torch.tensor(x.sm_scale, dtype=torch.float32)) * LOG2E32   # qsc
    sm64 = qs * x.d ** -0.5

    def tiles():
        for c0 in range(0, keys.numel(), CHUNK):
            kk, ks, dd = keys[c0:c0 + CHUNK], kscale[c0:c0 + CHUNK], dead[c0:c0 + CHUNK]
            acc = qi @ x.prep.k_i8[bi, hi, kk].double().t()             # exact integers
            s64 = (acc * (sm64 * ks.double())).masked_fill(dd, -math.inf)
            s32 = (acc.float() * (sc_q.to(dev) * ks)).masked_fill(dd, -math.inf)   # fl(float(acc) * fl(qsc * k_scale))
            yield c0 // bk, kk, s64, s32

    # pass 1: the float64 row maxima, and each entry's float32 maximum for the kernel's running maxima
    m64 = torch.full((len(rows), 1), -math.inf, dtype=torch.float64, device=dev)
    ent_max = []
    for _, _, s64, s32 in tiles():
        m64 = torch.maximum(m64, s64.amax(-1, keepdim=True))
        ent_max.append(s32.view(len(rows), -1, bk).amax(-1))
    m_ent = B.running_max(torch.cat(ent_max, 1).cpu(), x.blkq == 64).to(dev)
    m_top = m_ent[:, -2:].amax(-1, keepdim=True).double()   # the maximum after the last entry (and the warpgroups' merge)
    w_ent = torch.exp2(m_ent.double() - m_top)               # exact rescale factor of each entry's P into that maximum
    # pass 2: float64 softmax . V; P against the running maximum, rounded to T, weighted into the final maximum
    l64 = torch.zeros(len(rows), 1, dtype=torch.float64, device=dev)
    l32 = torch.zeros_like(l64)
    o64 = torch.zeros(len(rows), d, dtype=torch.float64, device=dev)
    o32 = torch.zeros_like(o64)
    flip, chain = torch.zeros_like(o64), torch.zeros_like(o64)
    for e0, kk, s64, s32 in tiles():
        v64 = x.v[bi, kk, hi].double()
        p64 = torch.exp(s64 - m64)
        l64 += p64.sum(-1, keepdim=True)
        o64 += p64 @ v64
        ne = s32.shape[1] // bk
        p32 = torch.exp2(s32 - m_ent[:, e0:e0 + ne].repeat_interleave(bk, 1))
        w = w_ent[:, e0:e0 + ne].repeat_interleave(bk, 1)
        if fp8 is None:
            l32 += (p32.double() * w).sum(-1, keepdim=True)
            o32 += (p32.to(x.dtype).double() * w) @ v64
        else:
            v_codes, v_scale = fp8
            v8 = (v_codes[:, kk].view(E4M3).double() * v_scale.double()[:, None]).t()
            pw = p32.to(p_dtype).double() * w
            l32 += (pw if l_from_rounded_p else p32.double() * w).sum(-1, keepdim=True)
            o32 += pw @ v8
            chain += pw.abs() @ v8.abs()
            flip += (_flip_step(p32) * w) @ v8.abs()

    q16 = x.q[bi, rows, hi].double()
    phi = _phi(q16, x.feature)
    den = phi @ x.ksum[bi, hi].double() + 1e-5
    kvw = x.kvw[bi, hi].double()
    pb = x.proj_b.double()
    ref = o64 / l64 + (phi @ kvw.t()) / den[:, None] + pb
    a = B.round_operand(phi * (l32 / den[:, None]), x.dtype)
    r32 = (o32 + a @ kvw.t()) / l32 + pb
    rest = r32.to(x.dtype).double()
    if fp8 is None:
        return ref, rest, None
    # every key block's e4m3 chain and its fp32 add into O: relative 2^-CHAIN_BITS + 2^-24 of the block's sum |p v|
    return ref, rest, {"r32": r32, "flip": flip / l32, "chain": (2.0 ** -CHAIN_BITS + 2.0 ** -24) * chain / l32}


def _distances(got, ref, rest, dtype):
    got = got.double()
    err = lambda a: (a - ref).norm(dim=-1)
    nrm = ref.norm(dim=-1)
    return {"kernel": float(err(got).norm() / nrm.norm()), "restatement": float(err(rest).norm() / nrm.norm()),
            "row_kernel": err(got) / nrm, "row_restatement": err(rest) / nrm,
            "row_rounding": err(ref.to(dtype).double()) / nrm}


_WORST_FAITH = []   # bar (b): each judged group's worst row / its bar, reported per test by _report_faithfulness


@pytest.fixture(autouse=True)
def _report_faithfulness(request):
    _WORST_FAITH.clear()
    yield
    if _WORST_FAITH:
        print(f"\n{request.node.name}: bar (b), worst row at {max(_WORST_FAITH):.3f} of its bar")


def _faithfulness(got, rest, fp8, nrm):
    """Bar (b) per row: (|kernel - R32|, its bar), both relative to the row's float64 norm `nrm`."""
    r32 = fp8["r32"]
    dist = (got.double() - r32).norm(dim=-1) / nrm
    bar = (2 * (rest - r32).norm(dim=-1) + fp8["flip"].norm(dim=-1) + fp8["chain"].norm(dim=-1)) / nrm
    return dist, bar


def _judge(got, ref, rest, dtype, what, entries=0, blkk=64, fp8=None):
    """The bars.  Returns (the group passes, per-row pass [R] bool, per-row pass of bar (b) or None without fp8) and
    prints the distances.  The 16-bit restatement sums P.V exactly, where the kernel adds each of the entries * blkk / 16
    MMA steps into its fp32 accumulator: the row bar counts one fp32 rounding (2^-24 relative) per step on top of the
    restatement's row error.  Below 100 entries that is < 3e-5; it matters at the top-k limits, where 26,920 entries
    (107,680 steps) put single rows 1.2x past the bar without it.  fp8 (the third value of _references): the e4m3
    restatement, the chain allowance in place of that count, and bar (b)."""
    s = _distances(got, ref, rest, dtype)
    nrm = ref.norm(dim=-1)
    acc = entries * blkk // 16 * 2.0 ** -24 if fp8 is None else fp8["chain"].norm(dim=-1) / nrm
    row_bar = 2 * torch.maximum(s["row_restatement"] + acc, s["row_rounding"])
    rows_ok = s["row_kernel"] <= row_bar
    block_ok = s["kernel"] <= 1.5 * s["restatement"]
    worst = int(torch.argmax(s["row_kernel"] / row_bar))
    msg = (f"{what}: rel-L2 kernel {s['kernel']:.3e} restatement {s['restatement']:.3e}; worst row {worst}: kernel "
           f"{float(s['row_kernel'][worst]):.3e} bar {float(row_bar[worst]):.3e}; rows failing {int((~rows_ok).sum())}/"
           f"{rows_ok.numel()}")
    faith_ok = None
    if fp8 is not None:
        dist, bar = _faithfulness(got, rest, fp8, nrm)
        faith_ok = dist <= bar
        ratio = dist / bar.clamp_min(1e-300)
        wf = int(torch.argmax(ratio))
        _WORST_FAITH.append(float(ratio[wf]))
        msg += (f"; bar (b) worst row {wf}: {float(dist[wf]):.3e} bar {float(bar[wf]):.3e} (float64 bar "
                f"{float(row_bar[wf]):.3e}), failing {int((~faith_ok).sum())}/{faith_ok.numel()}")
    print(msg)
    return block_ok, rows_ok, faith_ok


def _check_group(x, out, bi, hi, rows, entries, what, **kw):
    if x.pv == "fp8":
        kw.setdefault("fp8", (x.v_codes[bi, hi], x.v_scale[bi, hi]))
    ref, rest, fp8 = _references(x, bi, hi, rows, entries, **kw)
    got = out[bi, rows.to(out.device), hi]
    block_ok, rows_ok, faith_ok = _judge(got, ref, rest, x.dtype, what, len(entries), x.blkk, fp8)
    if faith_ok is not None:
        rows_ok = rows_ok & faith_ok
    assert block_ok and bool(rows_ok.all()), (what, "rows", rows[~rows_ok.cpu()].tolist(), "entries", entries)


def _check_all(x, lut, out, pad, what):
    """Every (batch, head, query block) of a call, every row."""
    assert torch.equal(pad, torch.full_like(pad, SENTINEL)), f"{what}: the kernel wrote past row lq"
    assert torch.isfinite(out.float()).all(), what
    lut_cpu = lut.cpu()
    for bi in range(x.b):
        for hi in range(x.h):
            for m in range(x.mblk):
                rows = torch.arange(m * x.blkq, min(x.lq, (m + 1) * x.blkq))
                _check_group(x, out, bi, hi, rows, lut_cpu[bi, hi, m].tolist(), f"{what} b{bi} h{hi} m{m}")


# ------------------------------------------------------------------------------------------------------------ the cases
@pytest.mark.parametrize("feature", sorted(FEATURES))
@pytest.mark.parametrize("d,pv", D_PV)
@pytest.mark.parametrize("dtype", sorted(DTYPES))
@pytest.mark.parametrize("family", sorted(FAMILIES))
def test_block_map_lut_scale_contrast(cuda, family, dtype, d, pv, feature):
    """b = 2, h = 3, l = 1000 (ragged last query and key blocks) on the block map's LUT (a third of the key blocks), with
    per-block magnitudes that differ by up to 16x between neighbours, so a scale read from the wrong block, head or batch
    entry moves the output far past the bars.  FP8: V channels of each (batch, head) differ by up to 16x too, for v_scale."""
    q, k, v = _qkv(2, 1000, 1000, 3, d, 100 + d + FEATURES[feature], cuda, family, v_contrast=pv == "fp8")
    if feature != "softmax":
        q = q * 0.5
    x = _prepare(q, k, v, family, DTYPES[dtype], FEATURES[feature], pv=pv)
    lut = _block_map_lut(x, max(1, x.nblk // 3))
    rc, out, pad = _run(x, lut)
    assert rc == 0, _last_error()
    _check_all(x, lut, out, pad, f"block map {family} {dtype} d={d} {pv} P.V {feature}")


L_HAND = 7 * 64 + 40, 7 * 128 + 40   # lk of the hand-made LUT cases (sm100, sm90): 8 key blocks, the last one ragged
R = 7                                # the ragged block
HAND_LUTS = {
    # 1 to 4 entries: the 3-slot rings' depth +-1; in the 64-row kernel warpgroup 1 with no entry (1) or one fewer (3)
    "one": [3], "two": [2, 5], "three": [1, 3, 5], "four": [0, 2, 3, 5],
    # the ragged block alone, as the last entry of warpgroup 0 (odd length) and as warpgroup 1's first entry
    "ragged_alone": [R], "ragged_last_wg0": [1, 4, R], "ragged_first_wg1": [2, R],
    # boosted entries (positions in BOOST): the row maximum rises by more than 2^8 (log2) only there
    "rise_wg1": [0, 1, 2, 3, 4, 5], "rise_wg0": [0, 1, 2, 3, 4, 5], "rise_next": [0, 2, 3, 4, 5, 6],
    "rise_last": [0, 2, 3, 4, 5, 6],
    # every score of the first entry negative; peaked rows (exp2 underflows for all keys but one)
    "negative_first": [0, 2, 4, 6], "peaked": [1, 3, 5],
}
BOOST = {"rise_wg1": (3, 5), "rise_wg0": (2, 4), "rise_next": (1,), "rise_last": (5,)}


def _hand_inputs(name, family, d, dtype, seed, valid=None, pv="bf16"):
    blkq, blkk = FAMILIES[family]
    lk = L_HAND[family == "sm90"] if valid is None else R * blkk + valid
    dev = torch.device("cuda")
    q, k, v = _qkv(1, lk, lk, 2, d, seed, dev, family)
    entries = HAND_LUTS[name]
    u = torch.ones(d, device=dev) / d ** 0.5
    if name in BOOST or name == "negative_first":   # queries share a component along u; whole key blocks along or against it
        q, k = q * 0.25 + 6.0 * u, k * 0.25
        for pos in BOOST.get(name, ()):
            k[:, entries[pos] * blkk:(entries[pos] + 1) * blkk] += 24.0 * u
        if name == "negative_first":
            k[:, entries[0] * blkk:(entries[0] + 1) * blkk] -= 16.0 * u
    if name == "peaked":                            # one key far along u: 8 * 150 / sqrt(d) above the rest
        q, k = q * 0.1 + 8.0 * u, k * 0.25
        k[:, entries[1] * blkk + 5] = 150.0 * u
    return _prepare(q, k, v, family, dtype, pv=pv), entries


def _premise(x, name, entries):
    """The scores do what the case is named for (first row block of head 0, float64 on the kernel's codes)."""
    bk = x.blkk
    rows = torch.arange(0, min(x.lq, x.blkq), device=x.q.device)
    qi = x.prep.q_i8[0, 0, rows].double() * float(x.prep.q_scale[0, 0, 0]) * x.sm_scale / math.log(2.0)
    ent_max = []
    for e in entries:
        kk = torch.arange(e * bk, min(x.lk, (e + 1) * bk), device=x.q.device)
        s = qi @ (x.prep.k_i8[0, 0, kk].double() * float(x.prep.k_scale[0, 0, e])).t()
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


@pytest.mark.parametrize("d,pv", D_PV)
@pytest.mark.parametrize("dtype", sorted(DTYPES))
@pytest.mark.parametrize("family", sorted(FAMILIES))
@pytest.mark.parametrize("name", list(HAND_LUTS))
def test_hand_made_luts(cuda, name, family, dtype, d, pv):
    x, entries = _hand_inputs(name, family, d, DTYPES[dtype], 300 + len(name) + d, pv=pv)
    _premise(x, name, entries)
    lut = _hand_lut(x, entries)
    rc, out, pad = _run(x, lut)
    assert rc == 0, _last_error()
    _check_all(x, lut, out, pad, f"hand LUT {name} {family} {dtype} d={d} {pv} P.V")


@pytest.mark.parametrize("valid", ["1", "BK-1"])
@pytest.mark.parametrize("name", ["ragged_alone", "ragged_last_wg0", "ragged_first_wg1"])
@pytest.mark.parametrize("family,pv", FAMILY_PV)
def test_ragged_block_one_or_all_but_one_key(cuda, family, pv, name, valid):
    blkk = FAMILIES[family][1]
    n = 1 if valid == "1" else blkk - 1
    for dtype in DTYPES.values():
        x, entries = _hand_inputs(name, family, 128, dtype, 400 + n, valid=n, pv=pv)
        assert x.lk - R * blkk == n
        lut = _hand_lut(x, entries)
        rc, out, pad = _run(x, lut)
        assert rc == 0, _last_error()
        _check_all(x, lut, out, pad, f"ragged {name} valid={n} {family} {dtype} {pv} P.V")


@pytest.mark.parametrize("lq,lk", [(200, 5000), (3000, 300)])
@pytest.mark.parametrize("family,pv", FAMILY_PV)
def test_query_and_key_lengths_differ(cuda, family, pv, lq, lk):
    cases = [(torch.bfloat16, 128), (torch.float16, 64 if pv == "bf16" else 128)]
    for i, (dtype, d) in enumerate(cases):
        q, k, v = _qkv(1, lq, lk, 2, d, 500 + lq + d, cuda, family)
        x = _prepare(q, k, v, family, dtype, pv=pv)
        lut = _block_map_lut(x, max(1, x.nblk // 3) + i)
        rc, out, pad = _run(x, lut)
        assert rc == 0, _last_error()
        _check_all(x, lut, out, pad, f"lq={lq} lk={lk} {family} {dtype} d={d} {pv} P.V")


@pytest.mark.parametrize("family,pv", FAMILY_PV)
def test_sequence_major_keys_equal_head_major(cuda, family, pv):
    """k_i8 in the [1, lk, h, d] layout sequence-parallel ranks gather: the same bits as head-major K, and the bars."""
    q, k, v = _qkv(1, 700, 1500, 3, 128, 600, cuda, family)
    x = _prepare(q, k, v, family, torch.bfloat16, pv=pv)
    lut = _block_map_lut(x, max(1, x.nblk // 3))
    rc, out, pad = _run(x, lut)
    assert rc == 0, _last_error()
    rc, out_seq, pad_seq = _run(x, lut, k_seq_major=True)
    assert rc == 0, _last_error()
    assert torch.equal(out_seq, out) and torch.equal(pad_seq, pad)
    _check_all(x, lut, out_seq, pad_seq, f"sequence-major K {family} {pv} P.V")


def test_topk_limits_follow_the_shared_memory_layout():
    for (family, d), t in TOPK_LIMIT.items():
        assert _largest_topk(d, *FAMILIES[family]) == t, (family, d)
    for family, t in TOPK_LIMIT_FP8.items():
        assert _largest_topk(128, *FAMILIES[family], fp8v=True) == t, family


def _limit_inputs(family, d, topk, lq_blocks, seed):
    """h = 1, lk ragged with exactly `topk` key blocks, every query block's LUT all of them (ascending)."""
    blkq, blkk = FAMILIES[family]
    lk = topk * blkk - 17
    lq = (lq_blocks - 1) * blkq + 37
    q, k, v = _qkv(1, lq, lk, 1, d, seed, torch.device("cuda"), family)
    return q, k, v


@pytest.mark.parametrize("d,pv", D_PV)
@pytest.mark.parametrize("family", sorted(FAMILIES))
def test_largest_topk_and_one_more(cuda, family, d, pv):
    topk = TOPK_LIMIT_FP8[family] if pv == "fp8" else TOPK_LIMIT[(family, d)]
    q, k, v = _limit_inputs(family, d, topk, 2 if d == 128 else 3, 800 if pv == "fp8" else 700 + d)
    x = _prepare(q, k, v, family, torch.bfloat16, pv=pv)
    assert x.nblk == topk
    lut = torch.arange(topk, dtype=torch.int32, device=cuda).expand(1, 1, x.mblk, topk).contiguous()
    rc, out, pad = _run(x, lut)
    assert rc == 0, _last_error()
    _check_all(x, lut, out, pad, f"topk={topk} {family} d={d} {pv} P.V")
    # topk + 1 with lk long enough for it: refused before any launch, the buffer untouched
    blkk = FAMILIES[family][1]
    lut1 = torch.arange(topk + 1, dtype=torch.int32, device=cuda).expand(1, 1, x.mblk, topk + 1).contiguous()
    rc, out, pad = _run(x, lut1, lk=(topk + 1) * blkk)
    assert rc == ERR_UNSUPPORTED, rc
    assert f"topk={topk + 1}" in _last_error(), _last_error()
    assert (out == SENTINEL).all() and (pad == SENTINEL).all()


def _key_of_position(n):
    pos = torch.arange(n)
    return (pos & ~15) | (((pos >> 1) & 1) << 3) | (((pos >> 2) & 3) << 1) | (pos & 1)


@pytest.mark.parametrize("family,pv", FAMILY_PV)
def test_largest_key_block_count(cuda, family, pv):
    """nblk = 65535 (the LUT is staged as uint16): ids 0, 2^15 - 1, 2^15 and 65534 (ragged) meet the bars; nblk = 65536 is
    refused before any launch (tdb200_sla_quant_qk refuses that length too, so the refused call gets small buffers of its
    own, which it never reads)."""
    from turbodiffusion_b200._lib import DTYPE_TAG, lib, ptr, stream_ptr
    blkq, blkk = FAMILIES[family]
    lk = 65535 * blkk - 5
    q, k, v = _qkv(1, blkq + 20, lk, 1, 128, 900, cuda, family)
    x = _prepare(q, k, v, family, torch.bfloat16, pv=pv)
    del q, k, v
    assert x.nblk == 65535
    entries = [0, 32767, 32768, 65534]
    lut = _hand_lut(x, entries)
    rc, out, pad = _run(x, lut)
    assert rc == 0, _last_error()
    _check_all(x, lut, out, pad, f"nblk=65535 {family} {pv} P.V")

    lk = 65536 * blkk - 3
    small = [torch.zeros(4096, dtype=t, device=cuda) for t in (torch.int8, torch.float32, torch.bfloat16)]
    i8, f32, b16 = (ptr(t) for t in small)
    lut_s = torch.tensor(entries, dtype=torch.int32, device=cuda)
    buf = torch.full((4096,), SENTINEL, dtype=torch.bfloat16, device=cuda)
    head = (i8, f32, i8, f32)
    tail = (b16, DTYPE_TAG[torch.bfloat16], ptr(lut_s), 4, b16, f32, f32, ptr(buf), 1, 1, lk, 1, 128, 128 ** -0.5, 0, blkq,
            blkk, 0, stream_ptr(cuda))
    if pv == "fp8":
        rc = lib().tdb200_sla_attn_fwd_fp8v(*head, i8, f32, *tail)
    else:
        rc = lib().tdb200_sla_attn_fwd(*head, b16, *tail)
    torch.cuda.synchronize()
    assert rc == ERR_UNSUPPORTED, (rc, _last_error())
    assert (buf == SENTINEL).all()


FULL_SHAPES = {   # l, h, d, top-k ratio
    "A": (32760, 12, 128, 0.1), "B": (75600, 40, 128, 0.1), "d64": (32760, 24, 64, 0.1), "C_ltx": (28672, 32, 128, 0.3),
}


FULL_CASES = [pytest.param(s, t, "bf16", id=f"{s}-{t}") for s, t in
              [("A", "bf16"), ("A", "fp16"), ("B", "bf16"), ("d64", "bf16"), ("C_ltx", "bf16")]]
FULL_CASES += [pytest.param(s, t, "fp8", id=f"{s}-{t}-fp8") for s, t in [("A", "bf16"), ("A", "fp16"), ("B", "bf16"),
                                                                         ("C_ltx", "bf16")]]


@pytest.mark.parametrize("shape,dtype,pv", FULL_CASES)
@pytest.mark.parametrize("family", sorted(FAMILIES))
def test_full_shapes_sampled_rows(cuda, family, shape, dtype, pv):
    """The first 16, 32 random and the last 16 rows of three heads, each group of rows held to the block bar."""
    l, h, d, ratio = FULL_SHAPES[shape]
    q, k, v = _qkv(1, l, l, h, d, 1000 + l + h, cuda, family)
    x = _prepare(q, k, v, family, DTYPES[dtype], pv=pv)
    del q, k, v
    lut = _block_map_lut(x, int(ratio * x.nblk))
    rc, out, pad = _run(x, lut)
    assert rc == 0, _last_error()
    assert torch.equal(pad, torch.full_like(pad, SENTINEL))
    lut_cpu = lut.cpu()
    g = torch.Generator().manual_seed(l + h)
    groups = {"first": torch.arange(16), "random": torch.randint(16, l - 16, (32,), generator=g),
              "last": torch.arange(l - 16, l)}
    for hi in (0, h // 2, h - 1):
        assert torch.isfinite(out[0, :, hi].float()).all()
        for gname, rows in groups.items():
            fp8 = (x.v_codes[0, hi], x.v_scale[0, hi]) if pv == "fp8" else None
            refs, rests, terms = [], [], []
            for r in rows.tolist():   # rows of different query blocks read different LUTs
                ref, rest, t = _references(x, 0, hi, torch.tensor([r]), lut_cpu[0, hi, r // x.blkq].tolist(), fp8=fp8)
                refs.append(ref)
                rests.append(rest)
                terms.append(t)
            got = out[0, rows.to(cuda), hi]
            terms = None if fp8 is None else {key: torch.cat([t[key] for t in terms]) for key in terms[0]}
            block_ok, rows_ok, faith_ok = _judge(got, torch.cat(refs), torch.cat(rests), x.dtype,
                                                 f"shape {shape} {family} {dtype} {pv} P.V head {hi} {gname} rows",
                                                 lut.shape[-1], x.blkk, terms)
            if faith_ok is not None:
                rows_ok = rows_ok & faith_ok
            assert block_ok and bool(rows_ok.all()), (shape, family, hi, gname, rows[~rows_ok.cpu()].tolist())


# ------------------------------------------------------------------------------------------------------------ sensitivity
@pytest.mark.parametrize("family", sorted(FAMILIES))
def test_bars_reject_a_wrong_scale_entry_or_key(cuda, family):
    """The kernel's output against float64 references built the way a wrong kernel would compute, in one query block: its
    second LUT entry scaled with the next key block's k_scale, the block given the next query block's q_scale, that entry
    dropped, the ragged block's last valid key masked.  Each must fail the block bar and the row bar on at least half the
    block's rows.  Random keys without block contrast, so neighbouring k_scale differ by a few percent, and l = 4000 with a
    LUT of every fourth key block: the printed cosine / rel-L2 of the same rows shows which of these the cosine >= 0.999 /
    rel-L2 <= 2e-2 bars of the other SageSLA tests would accept (a neighbour's k_scale at 128 x 64, the masked key)."""
    blkq, blkk = FAMILIES[family]
    q, k, v = _qkv(1, 4000, 4000, 2, 128, 1100, cuda, contrast=False)
    x = _prepare(q, k, v, family, torch.bfloat16)
    rag = x.nblk - 1
    entries = list(range(1, rag, 4)) + [rag]
    lut = _hand_lut(x, entries)
    rc, out, pad = _run(x, lut)
    assert rc == 0, _last_error()
    bi, hi, m = 0, 1, 2
    rows = torch.arange(m * blkq, (m + 1) * blkq)
    nbr_ks = x.prep.k_scale[bi, hi, entries].clone()
    nbr_ks[1] = x.prep.k_scale[bi, hi, entries[1] + 1]
    wrong = {
        "entry 1 scaled with its neighbour's k_scale": dict(entry_k_scale=nbr_ks),
        "query block given the next block's q_scale": dict(q_scale=x.prep.q_scale[bi, hi, m + 1]),
        "entry 1 dropped": dict(entries=entries[:1] + entries[2:]),
        "the ragged block's last valid key masked": dict(key_limit=x.lk - 1),
    }
    _check_group(x, out, bi, hi, rows, entries, f"sensitivity {family} unperturbed")
    for what, kw in wrong.items():
        kw = dict(kw)
        ent = kw.pop("entries", entries)
        ref, rest, _ = _references(x, bi, hi, rows, ent, **kw)
        got = out[bi, rows.to(cuda), hi]
        block_ok, rows_ok, _ = _judge(got, ref, rest, x.dtype, f"sensitivity {family}: {what}", len(ent), x.blkk)
        g, r = got.double().flatten(), ref.flatten()
        print(f"    the same rows at the cosine / rel-L2 bars: cos {float(g @ r / (g.norm() * r.norm())):.6f} "
              f"rel-L2 {float((g - r).norm() / r.norm()):.3e}")
        assert not block_ok, what
        assert (~rows_ok).float().mean() >= 0.5, (what, int((~rows_ok).sum()))


@pytest.mark.parametrize("family", sorted(FAMILIES))
def test_fp8_bars_reject_a_wrong_v_scale_code_order_p_rounding_entry_or_key(cuda, family):
    """The FP8 kernel's output against references built the way a wrong kernel would compute, in one query block: every
    channel's v_scale taken from its pair neighbour (c ^ 1, a slip of the column pair cq), the next head's v_scale, V codes
    read in plain key order instead of tdb200_sla_quant_v_fp8's fragment order, P rounded to T (the 16-bit path dispatched),
    a dropped entry, the ragged block's last valid key masked.  Each must fail bar (b) on at least half the block's rows.
    The LUT is two full key blocks and the ragged one (160 keys at 128 x 64, 288 at 64 x 128): the chain allowance grows
    with sum |p v| / l, a key's share of the row with 1 / l, so over the 1,000 keys of the 16-bit variant's LUT a masked key
    hides inside the allowance on most rows.  The print shows whether a kernel computing the fault would pass
    test_gpu_sla_fp8_pv's bar on the same rows, rel-L2 <= 1.25x the e4m3 restatement's + the 16-bit one's.  l summed from
    the rounded P is printed, not asserted."""
    blkq, blkk = FAMILIES[family]
    q, k, v = _qkv(1, 4000, 4000, 2, 128, 1100, cuda, contrast=False)
    x = _prepare(q, k, v, family, torch.bfloat16, pv="fp8")
    rag = x.nblk - 1
    entries = [1, rag // 2, rag]
    lut = _hand_lut(x, entries)
    rc, out, pad = _run(x, lut)
    assert rc == 0, _last_error()
    bi, hi, m = 0, 0, 2
    rows = torch.arange(m * blkq, (m + 1) * blkq)
    codes, vs = x.v_codes[bi, hi], x.v_scale[bi, hi]
    pair = torch.arange(x.d, device=cuda) ^ 1
    wrong = {
        "v_scale of each channel's pair neighbour": dict(fp8=(codes, vs[pair])),
        "v_scale of the next head": dict(fp8=(codes, x.v_scale[bi, hi + 1])),
        "V codes in plain key order": dict(fp8=(x.v_fp8[bi, hi], vs)),
        "P rounded to T instead of e4m3": dict(p_dtype=x.dtype),
        "entry 1 dropped": dict(entries=entries[:1] + entries[2:]),
        "the ragged block's last valid key masked": dict(key_limit=x.lk - 1),
        "l summed from the e4m3-rounded P (reported only)": dict(l_from_rounded_p=True),
    }
    _check_group(x, out, bi, hi, rows, entries, f"fp8 sensitivity {family} unperturbed")
    unperturbed = list(_WORST_FAITH)   # the test's report: the kernel against the right references only
    got = out[bi, rows.to(cuda), hi]
    ref, _, right = _references(x, bi, hi, rows, entries, fp8=(codes, vs))
    _, rest16, _ = _references(x, bi, hi, rows, entries)
    rel = lambda a: float((a - ref).norm() / ref.norm())
    for what, kw in wrong.items():
        kw = dict(kw)
        ent = kw.pop("entries", entries)
        kw.setdefault("fp8", (codes, vs))
        wref, wrest, wterms = _references(x, bi, hi, rows, ent, **kw)
        _, _, faith_ok = _judge(got, wref, wrest, x.dtype, f"fp8 sensitivity {family}: {what}", len(ent), x.blkk, wterms)
        # a kernel that computes the fault, T(R32) of the wrong restatement, at test_gpu_sla_fp8_pv's bar
        old = rel(wrest) <= 1.25 * rel(right["r32"]) + rel(rest16)
        print(f"    bar (b) rejects {int((~faith_ok).sum())}/{len(rows)} rows; test_gpu_sla_fp8_pv's bar "
              f"{'accepts' if old else 'rejects'} it (rel-L2 {rel(wrest):.3e} against {1.25 * rel(right['r32']):.3e} + "
              f"{rel(rest16):.3e})")
        if "reported only" not in what:
            assert (~faith_ok).float().mean() >= 0.5, (what, int((~faith_ok).sum()))
    _WORST_FAITH[:] = unperturbed


# ------------------------------------------------------------------------------------------------------------ e4m3 range
def _chain_probe(family, dtype, dev):
    """One query block, a one-entry LUT, every score 0 (q_i8 = 0), so P = 1 on all BK keys; the linear branch 0 (kvw = 0,
    proj_b = 0).  V per channel: +448, -448, then BK - 2 keys of one small e4m3 value s_c (2^-9..2^4, varying mantissas):
    v_scale = 1 and the codes are V.  Returns (inputs, out [BK... rows, 128], exact [128] = (BK - 2) s_c / BK,
    sum |p v| [128])."""
    blkq, blkk = FAMILIES[family]
    c = torch.arange(128, device=dev, dtype=torch.float32)
    s = (torch.exp2(4 - c % 14) * (1 + (c // 14) / 8)).to(E4M3).float()
    v = torch.empty(1, blkk, 1, 128, device=dev)
    v[0, 0, 0], v[0, 1, 0], v[0, 2:, 0] = 448.0, -448.0, s
    q, k, _ = _qkv(1, blkq, blkk, 1, 128, 1300, dev, contrast=False)
    x = _prepare(q, k, v, family, dtype, pv="fp8")
    x.prep.q_i8.zero_()
    x.kvw.zero_()
    x.proj_b.zero_()
    assert torch.equal(x.v_scale, torch.ones_like(x.v_scale)), "v_scale = 448 / 448"
    rc, out, pad = _run(x, _hand_lut(x, [0]))
    assert rc == 0, _last_error()
    assert torch.equal(pad, torch.full_like(pad, SENTINEL))
    exact = (blkk - 2) * s.double() / blkk
    return out[0, :, 0].double(), exact, 896.0 + (blkk - 2) * s.double()


def test_fp8_chain_accumulation_width(cuda):
    """The e4m3 wgmma chain's accumulation width, through the kernel: with +448 and -448 in the first K = 32 step, what the
    chain drops of each channel's small values shows after the cancellation.  fp16 stores (BK - 2) s_c / BK exactly, so
    every output bit that differs is the chain's: its relative error against sum |p v| = 896 + (BK - 2) s_c, over every
    channel and row, is the width 2^-W.  W must be at least CHAIN_BITS, what bar (b) assumes.  bf16 rounds the output, so
    there each channel is held to CHAIN_BITS plus one bf16 ulp."""
    widths = {}
    for family in sorted(FAMILIES):
        blkk = FAMILIES[family][1]
        for name, dtype in sorted(DTYPES.items()):
            got, exact, total = _chain_probe(family, dtype, cuda)
            err = (got - exact).abs() * blkk / total    # relative to sum |p v|, in the units of the chain's sum
            if dtype == torch.float16:
                worst = float(err.max())
                widths[family] = -math.log2(worst) if worst > 0 else math.inf
                lost = (got - exact)[0].abs() > 0
                print(f"chain width {family} fp16: W = {widths[family]:.2f} bits (worst relative error {worst:.3e}); "
                      f"channels with a loss: s_c = {sorted(set(((exact * blkk / (blkk - 2))[lost]).tolist()))}")
                assert widths[family] >= CHAIN_BITS, (family, widths[family])
            else:
                ulp = torch.exp2(torch.floor(torch.log2(exact.abs())) - 7)
                bound = 2.0 ** -CHAIN_BITS * total / blkk + ulp
                print(f"chain {family} bf16: worst |out - exact| / bound {float(((got - exact).abs() / bound).max()):.3f}")
                assert bool(((got - exact).abs() <= bound).all()), family
    print(f"measured e4m3 chain width: {widths}")


def _hand_int8(x, tops, scales, offsets, seed):
    """Hand-made INT8 codes and scales, through the ABI, for one query block of h = 1 and key blocks 0, 1, 2.  Every query
    row: q_i8[0] = 64, the rest uniform in [-8, 8].  Key block e: key 0 with k_i8[0] = tops[e] and nothing else, so its
    score is exactly 64 tops[e] sc_e, the block's maximum; the other keys k_i8[0] = tops[e] - offsets(n), the rest uniform
    in [-2, 2].  k_scale[e] is searched so that the kernel's sc = fl(qsc k_scale) is scales[e] exactly (q_scale = 1)."""
    import numpy as np
    g = torch.Generator().manual_seed(seed)
    bq, bk, dev = x.blkq, x.blkk, x.q.device
    qi = torch.randint(-8, 9, (min(bq, x.lq), x.d), generator=g)
    qi[:, 0] = 64
    x.prep.q_i8.zero_()
    x.prep.q_i8[0, 0, :qi.shape[0]] = qi.to(torch.int8).to(dev)
    x.prep.q_scale.fill_(1.0)
    qsc = np.float32(np.float32(np.float32(1.0) * np.float32(x.sm_scale)) * np.float32(LOG2E32.item()))
    for e, (top, sc) in enumerate(zip(tops, scales)):
        ki = torch.randint(-2, 3, (bk, x.d), generator=g)
        ki[:, 0] = top - offsets(bk, g)
        ki[0] = 0
        ki[0, 0] = top
        x.prep.k_i8[0, 0, e * bk:(e + 1) * bk] = ki.to(torch.int8).to(dev)
        ks, target = np.float32(np.float32(sc) / qsc), np.float32(sc)
        for _ in range(64):
            if np.float32(qsc * ks) == target:
                break
            ks = np.nextafter(ks, np.float32(np.inf) if np.float32(qsc * ks) < target else np.float32(-np.inf))
        assert np.float32(qsc * ks) == target
        x.prep.k_scale[0, 0, e] = float(ks)
    return x


def _entry_scores(x, e):
    """fl(float(acc) sc) of key block e for the query block's rows, as the kernel forms them (float32)."""
    acc = x.prep.q_i8[0, 0, :x.lq].double() @ x.prep.k_i8[0, 0, e * x.blkk:(e + 1) * x.blkk].double().t()
    sc = (torch.tensor(float(x.prep.q_scale[0, 0, 0]), dtype=torch.float32) * torch.tensor(x.sm_scale, dtype=torch.float32)
          * LOG2E32) * x.prep.k_scale[0, 0, e].cpu()
    return acc.float().cpu() * sc


@pytest.mark.parametrize("rise", ["exactly_2^8", "2^8_and_one_ulp"])
@pytest.mark.parametrize("dtype", sorted(DTYPES))
@pytest.mark.parametrize("family", sorted(FAMILIES))
def test_fp8_entry_maximum_2_8_above_the_running_one(cuda, family, dtype, rise):
    """LUT [0, 2, 1] (entries 0 and 2 in one warpgroup sequence in both kernels).  Block 0 sets the running maximum m;
    block 1's maximum is m + 8 exactly, so the lazy rescale keeps m and that key's P is 2^8 = 256, the largest P it lets
    through (e4m3 holds it exactly); or one fp32 ulp above m + 8, so the maximum moves and P = 1.  Built on hand-made INT8
    codes: scores k_i8[0] * 64 * sc with sc = 2^-7 (block 0 at 2^-7 - 2^-31 in the second case, which puts m one ulp
    below 50).  The other keys of each block spread P over e4m3's range."""
    blkq, blkk = FAMILIES[family]
    q, k, v = _qkv(1, blkq, 3 * blkk, 1, 128, 1400, cuda, contrast=False)
    x = _prepare(q, k, v, family, DTYPES[dtype], pv="fp8")
    sc0 = 2.0 ** -7 if rise == "exactly_2^8" else 2.0 ** -7 - 2.0 ** -31
    offsets = lambda n, g: 8 + torch.randint(0, 25, (n,), generator=g)
    _hand_int8(x, tops=(100, 116, 104), scales=(sc0, 2.0 ** -7, 2.0 ** -7), offsets=offsets, seed=1401)
    s0, s1 = _entry_scores(x, 0), _entry_scores(x, 1)
    m, m1 = s0.amax(-1), s1.amax(-1)
    assert torch.equal(s0[:, 0], m) and torch.equal(s1[:, 0], m1), "key 0 holds each block's maximum"
    assert bool((_entry_scores(x, 2).amax(-1) <= m + 8.0).all()), "block 2 does not move the maximum"
    if rise == "exactly_2^8":   # premise: fl(s - m) = 8 exactly, and no rescale (s > fl(m + 8) is false)
        assert bool(((m1 - m) == 8.0).all()) and not bool((m1 > m + 8.0).any())
    else:                       # premise: s = fl(m + 8) + one ulp, so the maximum moves
        assert bool((m1 == torch.nextafter(m + 8.0, torch.tensor(math.inf))).all())
    lut = _hand_lut(x, [0, 2, 1])
    rc, out, pad = _run(x, lut)
    assert rc == 0, _last_error()
    _check_all(x, lut, out, pad, f"P at 2^8 ({rise}) {family} {dtype}")


@pytest.mark.parametrize("dtype", sorted(DTYPES))
@pytest.mark.parametrize("family", sorted(FAMILIES))
def test_fp8_rows_of_subnormal_p(cuda, family, dtype):
    """Every block's other keys 12 to 17 below its maximum key in k_i8[0], scores (12..17) / 2 below it with sc = 2^-7:
    most nonzero e4m3 P codes of each row are subnormals, [2^-9, 2^-6) (premise)."""
    blkq, blkk = FAMILIES[family]
    q, k, v = _qkv(1, blkq, 3 * blkk, 1, 128, 1500, cuda, contrast=False)
    x = _prepare(q, k, v, family, DTYPES[dtype], pv="fp8")
    offsets = lambda n, g: 12 + torch.randint(0, 6, (n,), generator=g)
    _hand_int8(x, tops=(100, 100, 100), scales=(2.0 ** -7,) * 3, offsets=offsets, seed=1501)
    s = torch.cat([_entry_scores(x, e) for e in range(3)], -1)
    p = torch.exp2(s - s.amax(-1, keepdim=True)).to(E4M3).float()
    share = ((p > 0) & (p < 2.0 ** -6)).float().sum(-1) / (p > 0).float().sum(-1)
    assert bool((share > 0.5).all()), share.min()
    lut = _hand_lut(x, [0, 2, 1])
    rc, out, pad = _run(x, lut)
    assert rc == 0, _last_error()
    _check_all(x, lut, out, pad, f"subnormal P {family} {dtype}")


@pytest.mark.parametrize("dtype", sorted(DTYPES))
@pytest.mark.parametrize("family", sorted(FAMILIES))
def test_fp8_v_channel_with_an_outlier(cuda, family, dtype):
    """V channel 37 of head 1 with one value 2^15 times the channel's standard deviation (about 2^13 above its other values),
    in a key block outside the LUT: it sets v_scale, so most of the channel's codes are e4m3 subnormals or zero (premise),
    while the rows' output stays of V's ordinary size."""
    blkq, blkk = FAMILIES[family]
    q, k, v = _qkv(1, 600, 1500, 2, 128, 1600, cuda, family)
    out_key = 3 * blkk + 7
    v[0, out_key, 1, 37] = 2.0 ** 15
    x = _prepare(q, k, v, family, DTYPES[dtype], pv="fp8")
    lut = _hand_lut(x, [e for e in range(x.nblk) if e % 3 != 1 and e != 3])   # block 3 outside the LUT
    c = x.v_codes[0, 1, 37, :x.lk].view(E4M3).float().abs()
    assert float(((c < 2.0 ** -6)).float().mean()) > 0.5, "most of the channel's codes subnormal or zero"
    rc, out, pad = _run(x, lut)
    assert rc == 0, _last_error()
    _check_all(x, lut, out, pad, f"V outlier {family} {dtype}")


# ------------------------------------------------------------------------------------------------------------ the module
@pytest.mark.parametrize("family", sorted(FAMILIES))
def test_module_fp8_equals_the_direct_call(cuda, family):
    """SageSparseLinearAttention.forward_with_lut under set_sage_pv("fp8") is tdb200_sla_attn_fwd_fp8v on the module's own
    LUT and inputs, bit for bit, so test_gpu_sla_fp8_pv's module-level tests stand on the row-level ones here."""
    from turbodiffusion_b200.SLA import SageSparseLinearAttention
    from turbodiffusion_b200.SLA.utils import set_sage_pv, set_served_arch
    for name, dtype in sorted(DTYPES.items()):
        q, k, v = _qkv(1, 1100, 1100, 2, 128, 1700, cuda, family)
        mod = SageSparseLinearAttention(128, 0.3, use_bf16=dtype == torch.bfloat16).to(cuda)
        g = torch.Generator().manual_seed(1701)
        with torch.no_grad():
            mod.proj_l.weight.copy_(torch.randn(128, 128, generator=g) * 0.05)
            mod.proj_l.bias.copy_(torch.randn(128, generator=g) * 0.05)
        prev_pv, prev_arch = set_sage_pv("fp8"), set_served_arch(family)
        try:
            want, sel = mod.forward_with_lut(*(t.to(dtype) for t in (q, k, v)))
        finally:
            set_sage_pv(prev_pv)
            set_served_arch(prev_arch)
        x = _prepare(q, k, v, family, dtype, pv="fp8", proj=(mod.proj_l.weight.detach(), mod.proj_l.bias.detach()))
        rc, out, pad = _run(x, sel["lut"])
        assert rc == 0, _last_error()
        assert torch.equal(out, want), (name, int((out != want).sum()))
        _check_all(x, sel["lut"], out, pad, f"module fp8 {family} {name}")
