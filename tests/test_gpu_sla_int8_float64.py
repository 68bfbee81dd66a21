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
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

FAMILIES = {"sm100": (128, 64), "sm90": (64, 128)}   # (BLKQ, BLKK): sla_attn_fwd_kernel, sla_attn_fwd_q64_kernel
DTYPES = {"bf16": torch.bfloat16, "fp16": torch.float16}
FEATURES = {"softmax": 0, "elu": 1, "relu": 2}
LOG2E32 = torch.tensor(1.4426950408889634, dtype=torch.float32)   # kLog2e as the kernel holds it
PAD_ROWS = 37          # rows of the buffer after the output, which the kernel must leave alone
SENTINEL = -1234.0     # exact in bf16 and fp16
CHUNK = 1 << 16        # keys per float64 score tile of the references
ERR_UNSUPPORTED = -2   # TDB200_ERR_UNSUPPORTED

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


def _qkv(b, lq, lk, h, d, seed, dev, family=None, contrast=True):
    """Float32 q [b, lq, h, d], k, v [b, lk, h, d] on `dev`, keys with a channel mean; with `contrast`, per-block magnitudes
    that vary by 2^-2..2^2 over the family's query and key blocks."""
    g = torch.Generator(device=dev).manual_seed(seed)
    q = torch.randn(b, lq, h, d, generator=g, device=dev)
    k = torch.randn(b, lk, h, d, generator=g, device=dev) + torch.randn(1, 1, h, d, generator=g, device=dev) * 2.0
    v = torch.randn(b, lk, h, d, generator=g, device=dev)
    if contrast:
        blkq, blkk = FAMILIES[family]
        q, k = _contrast(q, blkq, 0), _contrast(k, blkk, 1)
    return q, k, v


class Inputs:
    """What tdb200_sla_attn_fwd is given (GPU tensors), and the call's sizes."""


def _prepare(q, k, v, family, dtype, feature=0, seed=9):
    from turbodiffusion_b200.SLA.core import linear_moments, project_moments
    from turbodiffusion_b200.SLA.utils import quant_qk
    x = Inputs()
    x.blkq, x.blkk = FAMILIES[family]
    x.family, x.dtype, x.feature = family, dtype, feature
    x.q, x.k, x.v = (t.to(dtype).contiguous() for t in (q, k, v))
    x.b, x.lq, x.h, x.d = x.q.shape
    x.lk = x.k.shape[1]
    x.prep = quant_qk(x.q, x.k, x.lk, x.blkq, x.blkk)
    x.mblk, x.nblk = x.prep.mblk, x.prep.nblk
    kv, x.ksum = linear_moments(x.k, x.v, feature)
    g = torch.Generator().manual_seed(seed)
    w = (torch.randn(x.d, x.d, generator=g) * 0.05).to(q.device)
    x.proj_b = (torch.randn(x.d, generator=g) * 0.05).float().to(q.device).contiguous()
    x.kvw = project_moments(w, kv, dtype)
    x.sm_scale = x.d ** -0.5
    return x


def _block_map_lut(x, topk):
    from turbodiffusion_b200.SLA.utils import block_map_from_pools
    return block_map_from_pools(x.prep.q_pool, x.prep.k_pool, min(topk, x.nblk))[1]


def _hand_lut(x, entries):
    return torch.tensor(entries, dtype=torch.int32, device=x.q.device).view(1, 1, 1, -1).expand(
        x.b, x.h, x.mblk, len(entries)).contiguous()


def _run(x, lut, k_seq_major=False, lk=None, topk=None):
    """One tdb200_sla_attn_fwd call into a buffer PAD_ROWS rows longer than the output, filled with SENTINEL.
    Returns (return code, out [b, lq, h, d], pad rows)."""
    from turbodiffusion_b200._lib import DTYPE_TAG, lib, ptr, stream_ptr
    lk = x.lk if lk is None else lk
    topk = lut.shape[-1] if topk is None else topk
    k_i8 = x.prep.k_i8.permute(0, 2, 1, 3).contiguous() if k_seq_major else x.prep.k_i8
    n = x.b * x.lq * x.h * x.d
    buf = torch.full((n + PAD_ROWS * x.h * x.d,), SENTINEL, dtype=x.dtype, device=x.q.device)
    rc = lib().tdb200_sla_attn_fwd(ptr(x.prep.q_i8), ptr(x.prep.q_scale), ptr(k_i8), ptr(x.prep.k_scale), ptr(x.v), ptr(x.q),
                                   DTYPE_TAG[x.dtype], ptr(lut), topk, ptr(x.kvw), ptr(x.ksum), ptr(x.proj_b), ptr(buf), x.b,
                                   x.lq, lk, x.h, x.d, x.sm_scale, x.feature, x.blkq, x.blkk, int(k_seq_major),
                                   stream_ptr(x.q.device))
    torch.cuda.synchronize()
    return rc, buf[:n].view(x.b, x.lq, x.h, x.d), buf[n:]


def _last_error():
    from turbodiffusion_b200._lib import lib
    msg = lib().tdb200_last_error()
    return msg.decode() if msg else ""


# ------------------------------------------------------------------------------------------------------------ references
def _phi(x, feature):
    if feature == 0:
        return torch.softmax(x, -1)
    if feature == 1:
        return torch.nn.functional.elu(x) + 1
    return torch.relu(x)


def _round_operand(a, dtype):
    """T(a) as the kernel forms the linear branch's MMA operand: in fp16 a row whose max lies outside [2^-6, 2^15) is rounded
    as a * 2^sc with sc = clamp(14 - floor(log2 max), -64, 64), and the power of two divided out again (sla_attn.cu)."""
    if dtype == torch.bfloat16:
        return a.to(dtype).double()
    amax = a.amax(-1, keepdim=True)
    e = torch.frexp(amax.clamp_min(1e-300)).exponent - 1          # floor(log2 amax)
    sc = (14 - e).clamp(-64, 64).double()
    sc = torch.where(((amax > 0) & (amax < 2.0 ** -6)) | (amax >= 2.0 ** 15), sc, torch.zeros_like(sc))
    return (a * torch.exp2(sc)).to(dtype).double() * torch.exp2(-sc)


def _running_max(ent_max, two_warpgroups):
    """The row maximum each entry's P is formed against in the kernel ([R, entries] float32, in LUT order): the first entry
    of a warpgroup sets it, and it moves only when an entry's maximum exceeds it by more than 2^8 (the lazy rescale).  The
    64-row kernel runs one such sequence per warpgroup, over alternate entries."""
    m = ent_max.clone()
    for j in range(2 if two_warpgroups else 1, ent_max.shape[1]):
        prev = m[:, j - 2] if two_warpgroups else m[:, j - 1]
        m[:, j] = torch.where(ent_max[:, j] > prev + 8.0, ent_max[:, j], prev)
    return m


def _references(x, bi, hi, rows, entries, q_scale=None, entry_k_scale=None, key_limit=None, fp8=None):
    """(float64 reference, float32 restatement) [len(rows), d] float64 of query rows `rows` (one query block) of batch bi,
    head hi over the key blocks `entries`.  The keyword arguments replace what the kernel would read (the sensitivity test):
    the row block's q_scale, each entry's k_scale, the number of keys.  fp8 = (v_fp8 in key order [d, lk_pad], v_scale [d]):
    the restatement rounds P and reads V as e4m3, as tdb200_sla_attn_fwd_fp8v does."""
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
    m_ent = _running_max(torch.cat(ent_max, 1).cpu(), x.blkq == 64).to(dev)
    m_top = m_ent[:, -2:].amax(-1, keepdim=True).double()   # the maximum after the last entry (and the warpgroups' merge)
    w_ent = torch.exp2(m_ent.double() - m_top)               # exact rescale factor of each entry's P into that maximum
    # pass 2: float64 softmax . V; P against the running maximum, rounded to T, weighted into the final maximum
    l64 = torch.zeros(len(rows), 1, dtype=torch.float64, device=dev)
    l32 = torch.zeros_like(l64)
    o64 = torch.zeros(len(rows), d, dtype=torch.float64, device=dev)
    o32 = torch.zeros_like(o64)
    for e0, kk, s64, s32 in tiles():
        v64 = x.v[bi, kk, hi].double()
        p64 = torch.exp(s64 - m64)
        l64 += p64.sum(-1, keepdim=True)
        o64 += p64 @ v64
        ne = s32.shape[1] // bk
        p32 = torch.exp2(s32 - m_ent[:, e0:e0 + ne].repeat_interleave(bk, 1))
        w = w_ent[:, e0:e0 + ne].repeat_interleave(bk, 1)
        l32 += (p32.double() * w).sum(-1, keepdim=True)
        if fp8 is None:
            o32 += (p32.to(x.dtype).double() * w) @ v64
        else:
            v_codes, v_scale = fp8
            v8 = v_codes[:, kk].view(torch.float8_e4m3fn).double() * v_scale.double()[:, None]
            o32 += (p32.to(torch.float8_e4m3fn).double() * w) @ v8.t()

    q16 = x.q[bi, rows, hi].double()
    phi = _phi(q16, x.feature)
    den = phi @ x.ksum[bi, hi].double() + 1e-5
    kvw = x.kvw[bi, hi].double()
    pb = x.proj_b.double()
    ref = o64 / l64 + (phi @ kvw.t()) / den[:, None] + pb
    a = _round_operand(phi * (l32 / den[:, None]), x.dtype)
    rest = ((o32 + a @ kvw.t()) / l32 + pb).to(x.dtype).double()
    return ref, rest


def _distances(got, ref, rest, dtype):
    got = got.double()
    err = lambda a: (a - ref).norm(dim=-1)
    nrm = ref.norm(dim=-1)
    return {"kernel": float(err(got).norm() / nrm.norm()), "restatement": float(err(rest).norm() / nrm.norm()),
            "row_kernel": err(got) / nrm, "row_restatement": err(rest) / nrm,
            "row_rounding": err(ref.to(dtype).double()) / nrm}


def _judge(got, ref, rest, dtype, what, entries=0, blkk=64):
    """The bars.  Returns (the group passes, per-row pass [R] bool) and prints both distances.  The restatement sums P.V
    exactly, where the kernel adds each of the entries * blkk / 16 MMA steps into its fp32 accumulator: the row bar counts
    one fp32 rounding (2^-24 relative) per step on top of the restatement's row error.  Below 100 entries that is < 3e-5;
    it matters at the top-k limits, where 26,920 entries (107,680 steps) put single rows 1.2x past the bar without it."""
    s = _distances(got, ref, rest, dtype)
    acc = entries * blkk // 16 * 2.0 ** -24
    row_bar = 2 * torch.maximum(s["row_restatement"] + acc, s["row_rounding"])
    rows_ok = s["row_kernel"] <= row_bar
    block_ok = s["kernel"] <= 1.5 * s["restatement"]
    worst = int(torch.argmax(s["row_kernel"] / row_bar))
    print(f"{what}: rel-L2 kernel {s['kernel']:.3e} restatement {s['restatement']:.3e}; worst row {worst}: kernel "
          f"{float(s['row_kernel'][worst]):.3e} bar {float(row_bar[worst]):.3e}; rows failing {int((~rows_ok).sum())}/"
          f"{rows_ok.numel()}")
    return block_ok, rows_ok


def _check_group(x, out, bi, hi, rows, entries, what, **kw):
    ref, rest = _references(x, bi, hi, rows, entries, **kw)
    got = out[bi, rows.to(out.device), hi]
    block_ok, rows_ok = _judge(got, ref, rest, x.dtype, what, len(entries), x.blkk)
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
@pytest.mark.parametrize("d", [128, 64])
@pytest.mark.parametrize("dtype", sorted(DTYPES))
@pytest.mark.parametrize("family", sorted(FAMILIES))
def test_block_map_lut_scale_contrast(cuda, family, dtype, d, feature):
    """b = 2, h = 3, l = 1000 (ragged last query and key blocks) on the block map's LUT (a third of the key blocks), with
    per-block magnitudes that differ by up to 16x between neighbours, so a scale read from the wrong block, head or batch
    entry moves the output far past the bars."""
    q, k, v = _qkv(2, 1000, 1000, 3, d, 100 + d + FEATURES[feature], cuda, family)
    if feature != "softmax":
        q = q * 0.5
    x = _prepare(q, k, v, family, DTYPES[dtype], FEATURES[feature])
    lut = _block_map_lut(x, max(1, x.nblk // 3))
    rc, out, pad = _run(x, lut)
    assert rc == 0, _last_error()
    _check_all(x, lut, out, pad, f"block map {family} {dtype} d={d} {feature}")


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


def _hand_inputs(name, family, d, dtype, seed, valid=None):
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
    return _prepare(q, k, v, family, dtype), entries


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


@pytest.mark.parametrize("d", [128, 64])
@pytest.mark.parametrize("dtype", sorted(DTYPES))
@pytest.mark.parametrize("family", sorted(FAMILIES))
@pytest.mark.parametrize("name", list(HAND_LUTS))
def test_hand_made_luts(cuda, name, family, dtype, d):
    x, entries = _hand_inputs(name, family, d, DTYPES[dtype], 300 + len(name) + d)
    _premise(x, name, entries)
    lut = _hand_lut(x, entries)
    rc, out, pad = _run(x, lut)
    assert rc == 0, _last_error()
    _check_all(x, lut, out, pad, f"hand LUT {name} {family} {dtype} d={d}")


@pytest.mark.parametrize("valid", ["1", "BK-1"])
@pytest.mark.parametrize("name", ["ragged_alone", "ragged_last_wg0", "ragged_first_wg1"])
@pytest.mark.parametrize("family", sorted(FAMILIES))
def test_ragged_block_one_or_all_but_one_key(cuda, family, name, valid):
    blkk = FAMILIES[family][1]
    n = 1 if valid == "1" else blkk - 1
    for dtype in DTYPES.values():
        x, entries = _hand_inputs(name, family, 128, dtype, 400 + n, valid=n)
        assert x.lk - R * blkk == n
        lut = _hand_lut(x, entries)
        rc, out, pad = _run(x, lut)
        assert rc == 0, _last_error()
        _check_all(x, lut, out, pad, f"ragged {name} valid={n} {family} {dtype}")


@pytest.mark.parametrize("lq,lk", [(200, 5000), (3000, 300)])
@pytest.mark.parametrize("family", sorted(FAMILIES))
def test_query_and_key_lengths_differ(cuda, family, lq, lk):
    for i, (dtype, d) in enumerate([(torch.bfloat16, 128), (torch.float16, 64)]):
        q, k, v = _qkv(1, lq, lk, 2, d, 500 + lq + d, cuda, family)
        x = _prepare(q, k, v, family, dtype)
        lut = _block_map_lut(x, max(1, x.nblk // 3) + i)
        rc, out, pad = _run(x, lut)
        assert rc == 0, _last_error()
        _check_all(x, lut, out, pad, f"lq={lq} lk={lk} {family} {dtype} d={d}")


@pytest.mark.parametrize("family", sorted(FAMILIES))
def test_sequence_major_keys_equal_head_major(cuda, family):
    """k_i8 in the [1, lk, h, d] layout sequence-parallel ranks gather: the same bits as head-major K, and the bars."""
    q, k, v = _qkv(1, 700, 1500, 3, 128, 600, cuda, family)
    x = _prepare(q, k, v, family, torch.bfloat16)
    lut = _block_map_lut(x, max(1, x.nblk // 3))
    rc, out, pad = _run(x, lut)
    assert rc == 0, _last_error()
    rc, out_seq, pad_seq = _run(x, lut, k_seq_major=True)
    assert rc == 0, _last_error()
    assert torch.equal(out_seq, out) and torch.equal(pad_seq, pad)
    _check_all(x, lut, out_seq, pad_seq, f"sequence-major K {family}")


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


@pytest.mark.parametrize("d", [128, 64])
@pytest.mark.parametrize("family", sorted(FAMILIES))
def test_largest_topk_and_one_more(cuda, family, d):
    topk = TOPK_LIMIT[(family, d)]
    q, k, v = _limit_inputs(family, d, topk, 2 if d == 128 else 3, 700 + d)
    x = _prepare(q, k, v, family, torch.bfloat16)
    assert x.nblk == topk
    lut = torch.arange(topk, dtype=torch.int32, device=cuda).expand(1, 1, x.mblk, topk).contiguous()
    rc, out, pad = _run(x, lut)
    assert rc == 0, _last_error()
    _check_all(x, lut, out, pad, f"topk={topk} {family} d={d}")
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


@pytest.mark.parametrize("family", sorted(FAMILIES))
def test_largest_topk_fp8_pv(cuda, family):
    """tdb200_sla_attn_fwd_fp8v at its limit: every query block within test_gpu_sla_fp8_pv's bar, 1.25x the rel-L2 of an
    e4m3 restatement plus that of the 16-bit one; topk + 1 refused."""
    from turbodiffusion_b200 import _ops
    from turbodiffusion_b200._lib import DTYPE_TAG, lib, ptr, stream_ptr
    topk = TOPK_LIMIT_FP8[family]
    q, k, v = _limit_inputs(family, 128, topk, 2, 800)
    x = _prepare(q, k, v, family, torch.bfloat16)
    v_fp8, v_scale = _ops.sla_quant_v_fp8(x.v, x.lk, x.blkk)
    lut = torch.arange(topk, dtype=torch.int32, device=cuda).expand(1, 1, x.mblk, topk).contiguous()
    n = x.lq * x.h * x.d

    def call(t, lk):
        buf = torch.full((n + PAD_ROWS * x.h * x.d,), SENTINEL, dtype=x.dtype, device=cuda)
        lt = torch.arange(t, dtype=torch.int32, device=cuda).expand(1, 1, x.mblk, t).contiguous()
        rc = lib().tdb200_sla_attn_fwd_fp8v(ptr(x.prep.q_i8), ptr(x.prep.q_scale), ptr(x.prep.k_i8), ptr(x.prep.k_scale),
                                            ptr(v_fp8), ptr(v_scale), ptr(x.q), DTYPE_TAG[x.dtype], ptr(lt), t, ptr(x.kvw),
                                            ptr(x.ksum), ptr(x.proj_b), ptr(buf), 1, x.lq, lk, 1, 128, x.sm_scale, 0, x.blkq,
                                            x.blkk, 0, stream_ptr(cuda))
        torch.cuda.synchronize()
        return rc, buf[:n].view(1, x.lq, 1, 128), buf[n:]

    rc, out, pad = call(topk, x.lk)
    assert rc == 0, _last_error()
    assert torch.equal(pad, torch.full_like(pad, SENTINEL)) and torch.isfinite(out.float()).all()
    inv = torch.argsort(_key_of_position(v_fp8.shape[-1])).to(cuda)
    codes = v_fp8[0, 0][:, inv]
    for m in range(x.mblk):
        rows = torch.arange(m * x.blkq, min(x.lq, (m + 1) * x.blkq))
        ref, rest16 = _references(x, 0, 0, rows, lut[0, 0, m].tolist())
        _, emu = _references(x, 0, 0, rows, lut[0, 0, m].tolist(), fp8=(codes, v_scale[0, 0]))
        got = out[0, rows.to(cuda), 0].double()
        rel = lambda a: float((a - ref).norm() / ref.norm())
        print(f"fp8 topk={topk} {family} m{m}: rel-L2 kernel {rel(got):.3e} e4m3 restatement {rel(emu):.3e} "
              f"16-bit restatement {rel(rest16):.3e}")
        assert rel(got) <= 1.25 * rel(emu) + rel(rest16), m
    rc, out, pad = call(topk + 1, (topk + 1) * x.blkk)
    assert rc == ERR_UNSUPPORTED and f"topk={topk + 1}" in _last_error(), (rc, _last_error())
    assert (out == SENTINEL).all() and (pad == SENTINEL).all()


@pytest.mark.parametrize("family", sorted(FAMILIES))
def test_largest_key_block_count(cuda, family):
    """nblk = 65535 (the LUT is staged as uint16): ids 0, 2^15 - 1, 2^15 and 65534 (ragged) meet the bars; nblk = 65536 is
    refused before any launch (tdb200_sla_quant_qk refuses that length too, so the refused call gets small buffers of its
    own, which it never reads)."""
    from turbodiffusion_b200._lib import DTYPE_TAG, lib, ptr, stream_ptr
    blkq, blkk = FAMILIES[family]
    lk = 65535 * blkk - 5
    q, k, v = _qkv(1, blkq + 20, lk, 1, 128, 900, cuda, family)
    x = _prepare(q, k, v, family, torch.bfloat16)
    del q, k, v
    assert x.nblk == 65535
    entries = [0, 32767, 32768, 65534]
    lut = _hand_lut(x, entries)
    rc, out, pad = _run(x, lut)
    assert rc == 0, _last_error()
    _check_all(x, lut, out, pad, f"nblk=65535 {family}")

    lk = 65536 * blkk - 3
    small = [torch.zeros(4096, dtype=t, device=cuda) for t in (torch.int8, torch.float32, torch.bfloat16)]
    i8, f32, b16 = (ptr(t) for t in small)
    lut_s = torch.tensor(entries, dtype=torch.int32, device=cuda)
    buf = torch.full((4096,), SENTINEL, dtype=torch.bfloat16, device=cuda)
    rc = lib().tdb200_sla_attn_fwd(i8, f32, i8, f32, b16, b16, DTYPE_TAG[torch.bfloat16], ptr(lut_s), 4, b16, f32, f32,
                                   ptr(buf), 1, 1, lk, 1, 128, 128 ** -0.5, 0, blkq, blkk, 0, stream_ptr(cuda))
    torch.cuda.synchronize()
    assert rc == ERR_UNSUPPORTED, (rc, _last_error())
    assert (buf == SENTINEL).all()


FULL_SHAPES = {   # l, h, d, top-k ratio
    "A": (32760, 12, 128, 0.1), "B": (75600, 40, 128, 0.1), "d64": (32760, 24, 64, 0.1), "C_ltx": (28672, 32, 128, 0.3),
}


@pytest.mark.parametrize("shape,dtype", [("A", "bf16"), ("A", "fp16"), ("B", "bf16"), ("d64", "bf16"), ("C_ltx", "bf16")])
@pytest.mark.parametrize("family", sorted(FAMILIES))
def test_full_shapes_sampled_rows(cuda, family, shape, dtype):
    """The first 16, 32 random and the last 16 rows of three heads, each group of rows held to the block bar."""
    l, h, d, ratio = FULL_SHAPES[shape]
    q, k, v = _qkv(1, l, l, h, d, 1000 + l + h, cuda, family)
    x = _prepare(q, k, v, family, DTYPES[dtype])
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
            refs, rests = [], []
            for r in rows.tolist():   # rows of different query blocks read different LUTs
                ref, rest = _references(x, 0, hi, torch.tensor([r]), lut_cpu[0, hi, r // x.blkq].tolist())
                refs.append(ref)
                rests.append(rest)
            got = out[0, rows.to(cuda), hi]
            block_ok, rows_ok = _judge(got, torch.cat(refs), torch.cat(rests), x.dtype,
                                       f"shape {shape} {family} {dtype} head {hi} {gname} rows", lut.shape[-1], x.blkk)
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
        ref, rest = _references(x, bi, hi, rows, ent, **kw)
        got = out[bi, rows.to(cuda), hi]
        block_ok, rows_ok = _judge(got, ref, rest, x.dtype, f"sensitivity {family}: {what}", len(ent), x.blkk)
        g, r = got.double().flatten(), ref.flatten()
        print(f"    the same rows at the cosine / rel-L2 bars: cos {float(g @ r / (g.norm() * r.norm())):.6f} "
              f"rel-L2 {float((g - r).norm() / r.norm()):.3e}")
        assert not block_ok, what
        assert (~rows_ok).float().mean() >= 0.5, (what, int((~rows_ok).sum()))
