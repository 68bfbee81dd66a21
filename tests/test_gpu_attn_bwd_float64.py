"""The 16-bit attention backward kernels (csrc/sla_attn_bwd.cu: the delta kernel, the key-major index, the dQ kernels at 128 and
64 query rows, the dK / dV kernel at both heights, and their kDense instantiations behind tdb200_attn_dense_bwd) against
float64 on the kernel's own inputs, query block by query block, key block by key block and row by row.

Inputs are what the backward is given: the 16-bit q, k, v and dO, the forward's o_s and fp32 lse, and the LUT.  Two
references are built from them:
  * R64, the float64 closed form: P = 2^(S sm log2e - lse), delta = sum T(o_s) T(dO), dS = P o (dP - delta),
    dQ = sm dS K, dK = sm dS^T Q, dV = P^T dO.
  * R32, the restatement at the kernel's rounding points: S and dP in fp32, P = exp2(fl(S sc - lse)) in fp32 with
    sc = fl(sm log2e), delta in fp32, dS = P (dP - delta) in fp32; P rounded to T only as dV's operand and dS as the dQ / dK
    operand; the products summed exactly, then one fp32 rounding, the scale, and one rounding to T.  In fp16 R32 rounds dS
    to fp16's significand without its exponent limits: dS below fp16's normal range (small dO, as in loss-scaled training)
    must not cost the kernel more than fp16 precision, and the bar does not widen by what underflow would cost.
Bars: per (batch, head, block) rel-L2 against R64 <= 1.5x R32's; per row of dq, dk and dv
|kernel - R64| <= 2 max(|R32 - R64| + acc, |T(R64) - R64|) + sqrt(d) sub, sub one subnormal step of T (rows whose exact
gradient is ~0).  acc covers the fp32 sums R32 takes exactly: 2^-24 per 16-key (dQ) or 16-row (dK, dV) MMA step times the
row's |terms| sum (it matters only at the long lists of the limit tests), plus 2^-20 of the |terms| sums of each S, dP and
delta carried through P and dS (it matters where dP - delta cancels: a row with one key, or one dominant key, has an exact
dQ of ~0, and the kernel's dQ there is the fp32 noise of dP - delta).  Every output finite,
key blocks with an empty list exactly zero, and rows past l (past lq / lk for dense) of sentinel-filled buffers untouched.
The kernel's delta (the workspace's first array) and its key-major CSR index are also read back and checked, the index
exactly.  Every test prints its worst row as a fraction of its bar.

test_bars_reject_kernel_faults shows what these bars catch that cos >= 0.999 / rel-L2 <= 2e-2 and 1.5x SDPA let through.
"""
import math
import time
from types import SimpleNamespace

import pytest
import torch
import torch.nn.functional as F

import sla_backward_oracle as B

pytestmark = pytest.mark.gpu
D, BK = 128, 64
SM = D ** -0.5
F64, F32 = torch.float64, torch.float32
BF16, FP16 = torch.bfloat16, torch.float16
DTYPES = [pytest.param(BF16, id="bf16"), pytest.param(FP16, id="fp16")]
GEOMS = [pytest.param(128, id="q128"), pytest.param(64, id="q64")]
SM32 = torch.tensor(SM, dtype=F32)
SC32 = float(SM32 * torch.tensor(1.4426950408889634, dtype=F32))     # sc = p.sm_scale * kLog2e, in fp32
SUB = {BF16: 2.0 ** -133, FP16: 2.0 ** -24}                            # one subnormal step of T
PAD_ROWS = 37          # rows of each gradient buffer after the gradient, which the kernels must leave alone
SENTINEL = -1234.0     # exact in bf16 and fp16
FP32_SUM = 2.0 ** -20  # relative error of the kernel's fp32 S, dP (MMA chains over d) and delta, against their |terms| sums
CHUNK = 1 << 15        # keys (dQ) or query rows (dK, dV) per float64 tile of the references
# The backward's top-k limits (derived in tests/test_sla_q64_16bit_host.py beside the validation table): 33,664 on 128-row
# blocks, where the dQ kernel's on-chip uint16 LUT binds; 46,340 on 64-row blocks, where b*h*mblk*topk <= 2^31 - 1 binds
# (mblk >= topk there) before the LUT could.
BWD_TOPK_LIMIT = {128: 33664, 64: 46340}

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


def _buffers(dtype, dev, *shapes):
    """Sentinel-filled flat buffers PAD_ROWS rows longer than each [b, l, h, d] shape: (views, pads)."""
    return B.sentinel_buffers(dtype, dev, PAD_ROWS, SENTINEL, *shapes)


def _sla_forward(q, k, v, lut, blkq):
    from turbodiffusion_b200.SLA.core import attn_fwd_qk16_lse
    return attn_fwd_qk16_lse(q, k, v, lut, lut.shape[-1], SM, blkq=blkq)


def _sla_bwd(x):
    """tdb200_sla_attn16_bwd on x's tensors.  Sets x.dq, x.dk, x.dv, x.pads, x.ws (the workspace, read back afterwards)."""
    L = _lib()
    b, l, h, d = x.q.shape
    topk = x.lut.shape[-1]
    (x.dq, x.dk, x.dv), x.pads = _buffers(x.dtype, x.q.device, *[x.q.shape] * 3)
    nbytes = L.lib().tdb200_sla_attn16_bwd_workspace_bytes(b, h, l, topk, x.blkq)
    assert nbytes > 0, _last_error()
    x.ws = torch.empty(nbytes, dtype=torch.uint8, device=x.q.device)
    p = L.ptr
    t0 = time.perf_counter()
    rc = L.lib().tdb200_sla_attn16_bwd(p(x.q), p(x.k), p(x.v), p(x.o_s), p(x.do), p(x.lse), L.DTYPE_TAG[x.dtype], p(x.lut), topk,
                                       p(x.dq), p(x.dk), p(x.dv), p(x.ws), nbytes, b, l, h, d, SM, x.blkq, BK,
                                       L.stream_ptr(x.q.device))
    torch.cuda.synchronize()
    x.seconds = time.perf_counter() - t0
    assert rc == 0, _last_error()
    return x


def _dense_bwd(x):
    """tdb200_attn_dense_bwd (after tdb200_attn_dense_fwd_lse for o_s and lse unless x has them)."""
    L = _lib()
    p = L.ptr
    b, lq, h, d = x.q.shape
    lk = x.k.shape[1]
    if getattr(x, "o_s", None) is None:
        x.o_s = torch.empty_like(x.q)
        x.lse = torch.empty(b, h, lq, dtype=F32, device=x.q.device)
        rc = L.lib().tdb200_attn_dense_fwd_lse(p(x.q), p(x.k), p(x.v), L.DTYPE_TAG[x.dtype], p(x.o_s), p(x.lse), b, lq, lk, h, d, SM,
                                               L.stream_ptr(x.q.device))
        assert rc == 0, _last_error()
    (x.dq, x.dk, x.dv), x.pads = _buffers(x.dtype, x.q.device, x.q.shape, x.k.shape, x.k.shape)
    nbytes = L.lib().tdb200_attn_dense_bwd_workspace_bytes(b, h, lq)
    x.ws = torch.empty(nbytes, dtype=torch.uint8, device=x.q.device)
    rc = L.lib().tdb200_attn_dense_bwd(p(x.q), p(x.k), p(x.v), p(x.o_s), p(x.do), p(x.lse), L.DTYPE_TAG[x.dtype], p(x.dq), p(x.dk),
                                       p(x.dv), p(x.ws), nbytes, b, lq, lk, h, d, SM, L.stream_ptr(x.q.device))
    torch.cuda.synchronize()
    assert rc == 0, _last_error()
    return x


def _case(q, k, v, do, lut, blkq, o_s=None, lse=None):
    """The backward's inputs on the GPU (q, k, v, dO in one 16-bit type; lut None for dense attention), with the forward's o_s
    and lse unless given, and delta in float64 and fp32 from T(o_s) and T(dO)."""
    x = SimpleNamespace(q=q, k=k, v=v, do=do, lut=lut, blkq=blkq, dtype=q.dtype, o_s=o_s, lse=lse)
    x.b, x.lq, x.h, _ = q.shape
    x.lk = k.shape[1]
    x.mblk, x.nblk = B.cdiv(x.lq, blkq), B.cdiv(x.lk, BK)
    if lut is not None and o_s is None:
        x.o_s, x.lse = _sla_forward(q, k, v, lut, blkq)
    return x


def _finish(x):
    x.delta64 = (x.o_s.double() * x.do.double()).sum(-1).permute(0, 2, 1).contiguous()     # [b, h, lq]
    x.delta32 = x.delta64.float()
    return x


def _run(x):
    return _finish(_sla_bwd(x) if x.lut is not None else _dense_bwd(x))


_randn = B.randn


# ------------------------------------------------------------------------------------------------------------ references
def _query_keys(x, bi, hi, m, lut_row=None):
    """The key columns query block m reads (LUT order, keys >= lk dropped); dense: every key."""
    if x.lut is None:
        return torch.arange(x.lk, device=x.q.device)
    ids = (x.lut[bi, hi, m] if lut_row is None else lut_row).long().to(x.q.device)
    cols = (ids[:, None] * BK + torch.arange(BK, device=x.q.device)).flatten()
    return cols[cols < x.lk]


def _key_rows(x, bi, hi, n):
    """The query rows whose block lists key block n, once per listing; dense: every query row."""
    if x.lut is None:
        return torch.arange(x.lq, device=x.q.device)
    times = (x.lut[bi, hi] == n).sum(-1)                          # [mblk]
    blocks = torch.repeat_interleave(torch.arange(x.mblk, device=x.q.device), times.to(x.q.device))
    rows = (blocks[:, None] * x.blkq + torch.arange(x.blkq, device=x.q.device)).flatten()
    return rows[rows < x.lq]


def _round_ds(ds32, dtype):
    """T(dS) as the dQ / dK operand: bf16 plainly; fp16 with its 11-bit significand but no exponent limits, so that precision
    the kernel loses to fp16's subnormals is not part of the bar."""
    if dtype == BF16:
        return ds32.to(dtype).double()
    m, e = torch.frexp(ds32.double())
    return torch.ldexp(torch.round(m * 2048.0) / 2048.0, e)


def _tile(x, bi, hi, rows, keys, lse_rows=None, dlt_rows=None, raw=False):
    """(P64, dS64, T(P32), T(dS32), (eP, edS)) of the rows x keys tile, float64 (raw: P32 and dS32 before their rounding to
    T).  eP and edS bound what R32's exact-then-rounded S, dP and delta do not model: the kernel's fp32 sums for them, each
    within FP32_SUM of its |terms| sum, and ex2.approx's 2 ulp.  lse_rows / dlt_rows: the rows whose lse / delta each row
    uses (a faulty kernel's, for the sensitivity test)."""
    lse_rows = rows if lse_rows is None else lse_rows
    dlt_rows = rows if dlt_rows is None else dlt_rows
    qr, gr = x.q[bi, rows, hi].double(), x.do[bi, rows, hi].double()
    kc, vc = x.k[bi, keys, hi].double(), x.v[bi, keys, hi].double()
    s = qr @ kc.t()
    dp = gr @ vc.t()
    lse = x.lse[bi, hi, lse_rows].double()[:, None]
    p64 = torch.exp2(s * (SM / math.log(2.0)) - lse)
    ds64 = p64 * (dp - x.delta64[bi, hi, dlt_rows][:, None])
    p32 = torch.exp2((s.float().double() * SC32 - lse).float())
    ds32 = p32 * (dp.float() - x.delta32[bi, hi, dlt_rows][:, None])
    if raw:
        return p64, ds64, p32, ds32
    pd = p32.double()
    e_p = pd * (FP32_SUM * SC32 * math.log(2.0) * (qr.abs() @ kc.abs().t()) + 2.0 ** -22)
    e_dlt = FP32_SUM * (x.o_s[bi, dlt_rows, hi].double() * x.do[bi, dlt_rows, hi].double()).abs().sum(-1)
    e_ds = e_p * (dp - x.delta64[bi, hi, dlt_rows][:, None]).abs() + pd * FP32_SUM * (gr.abs() @ vc.abs().t() + e_dlt[:, None])
    return p64, ds64, p32.to(x.dtype).double(), _round_ds(ds32, x.dtype), (e_p, e_ds)


def _round_out(acc, scale, dtype):
    return (acc.float() * scale).to(dtype).double()


def _ref_dq(x, bi, hi, rows, keys, **kw):
    """(R64, R32, |terms| sum, MMA steps) of dQ at `rows` over `keys`."""
    r64 = torch.zeros(len(rows), D, dtype=F64, device=x.q.device)
    acc, mag, allow = torch.zeros_like(r64), torch.zeros_like(r64), torch.zeros_like(r64)
    for c0 in range(0, len(keys), CHUNK):
        kk = keys[c0:c0 + CHUNK]
        _, ds64, _, dst, (_, e_ds) = _tile(x, bi, hi, rows, kk, **kw)
        kc = x.k[bi, kk, hi].double()
        r64 += SM * (ds64 @ kc)
        acc += dst @ kc
        mag += dst.abs() @ kc.abs()
        allow += e_ds @ kc.abs()
    return r64, _round_out(acc, SM32, x.dtype), SM * mag, B.cdiv(len(keys), 16), SM * allow


def _ref_dkdv(x, bi, hi, keys, rows, **kw):
    """((R64, R32, |terms|, steps) of dK, the same of dV) at key rows `keys` over query rows `rows`."""
    z = lambda: torch.zeros(len(keys), D, dtype=F64, device=x.q.device)
    k64, kacc, kmag, kal, v64, vacc, vmag, val = z(), z(), z(), z(), z(), z(), z(), z()
    for r0 in range(0, len(rows), CHUNK):
        rr = rows[r0:r0 + CHUNK]
        p64, ds64, pt, dst, (e_p, e_ds) = _tile(x, bi, hi, rr, keys, **kw)
        qr, gr = x.q[bi, rr, hi].double(), x.do[bi, rr, hi].double()
        k64 += SM * (ds64.t() @ qr)
        kacc += dst.t() @ qr
        kmag += dst.t().abs() @ qr.abs()
        v64 += p64.t() @ gr
        vacc += pt.t() @ gr
        vmag += pt.t().abs() @ gr.abs()
        kal += e_ds.t() @ qr.abs()
        val += e_p.t() @ gr.abs()
    steps = B.cdiv(len(rows), 16)
    return ((k64, _round_out(kacc, SM32, x.dtype), SM * kmag, steps, SM * kal),
            (v64, _round_out(vacc, 1.0, x.dtype), vmag, steps, val))


def _judge(got, ref, dtype, what, record=True):
    """The bars on one block.  Returns (block passes, per-row pass) and prints the distances."""
    r64, r32, mag, steps, allow = ref
    got = got.double()
    e_k = (got - r64).norm(dim=-1)
    e_32 = (r32 - r64).norm(dim=-1)
    e_t = (r64.to(dtype).double() - r64).norm(dim=-1)
    acc = steps * 2.0 ** -24 * mag.norm(dim=-1) + allow.norm(dim=-1)
    floor = SUB[dtype] * math.sqrt(D)
    bar = 2 * torch.maximum(e_32 + acc, e_t) + floor
    rows_ok = e_k <= bar
    block_ok = e_k.norm() <= 1.5 * e_32.norm() + acc.norm() + floor * math.sqrt(len(e_k))
    ratio = e_k / bar
    worst = int(torch.argmax(ratio))
    if record:
        _WORST.append(float(ratio[worst]))
    nrm = r64.norm().clamp_min(1e-300)
    if not (block_ok and rows_ok.all()) or record is None:
        print(f"{what}: rel-L2 kernel {float(e_k.norm() / nrm):.3e} R32 {float(e_32.norm() / nrm):.3e}; worst row {worst} at "
              f"{float(ratio[worst]):.3f} of its bar; rows failing {int((~rows_ok).sum())}/{len(rows_ok)}")
    return bool(block_ok), rows_ok


def _assert_block(got, ref, dtype, what):
    block_ok, rows_ok = _judge(got, ref, dtype, what)
    assert block_ok and bool(rows_ok.all()), (what, "rows failing", (~rows_ok).nonzero().flatten().tolist()[:16])


def _check_index(x):
    """The key-major CSR index in the workspace against the LUT's transposition: offsets, and each list ascending."""
    b, h, mblk, topk = x.lut.shape
    nblk, l = x.nblk, x.lq
    a = lambda n: (n + 255) // 256 * 256
    off0 = a(4 * b * h * l)
    idx0 = off0 + a(4 * b * h * (nblk + 1)) + a(4 * b * h * nblk)
    kv_off = x.ws[off0:off0 + 4 * b * h * (nblk + 1)].view(torch.int32).view(b * h, nblk + 1).long()
    kv_idx = x.ws[idx0:idx0 + 4 * b * h * mblk * topk].view(torch.int32).view(b * h, mblk * topk).long()
    lut = x.lut.view(b * h, mblk * topk).long()
    blocks = torch.arange(mblk, device=lut.device).repeat_interleave(topk)[None].expand_as(lut)
    counts = torch.zeros(b * h, nblk, dtype=torch.long, device=lut.device).scatter_add_(1, lut, torch.ones_like(lut))
    want_off = F.pad(counts.cumsum(1), (1, 0))
    order = torch.argsort(lut * mblk + blocks, dim=1, stable=True)
    assert torch.equal(kv_off, want_off), "key-major offsets"
    assert torch.equal(kv_idx, blocks.gather(1, order)), "key-major lists"


def _check_delta(x):
    """The delta kernel's fp32 rows (the workspace's first array) against float64: 2^-20 of sum |T(o_s) T(dO)| each."""
    n = x.b * x.h * x.lq
    got = x.ws[:4 * n].view(F32).view(x.b, x.h, x.lq).double()
    mag = (x.o_s.double() * x.do.double()).abs().sum(-1).permute(0, 2, 1)
    assert bool(((got - x.delta64).abs() <= 2.0 ** -20 * mag + 1e-30).all()), "delta"


def _check_common(x, what):
    for name, pad in zip(("dq", "dk", "dv"), x.pads):
        assert torch.equal(pad, torch.full_like(pad, SENTINEL)), f"{what}: {name} written past its last row"
    for name, g in (("dq", x.dq), ("dk", x.dk), ("dv", x.dv)):
        assert torch.isfinite(g.float()).all(), (what, name)
    _check_delta(x)
    if x.lut is not None and x.lut.numel() < (1 << 26):
        _check_index(x)


def _check(x, what, q_blocks=None, k_blocks=None, bh=None):
    """All bars on every (or the sampled) query and key blocks of every (or the sampled) (batch, head)."""
    _check_common(x, what)
    bh = [(bi, hi) for bi in range(x.b) for hi in range(x.h)] if bh is None else bh
    q_blocks = range(x.mblk) if q_blocks is None else q_blocks
    k_blocks = range(x.nblk) if k_blocks is None else k_blocks
    for bi, hi in bh:
        for m in q_blocks:
            rows = torch.arange(m * x.blkq, min(x.lq, (m + 1) * x.blkq), device=x.q.device)
            _assert_block(x.dq[bi, rows, hi], _ref_dq(x, bi, hi, rows, _query_keys(x, bi, hi, m)), x.dtype,
                          f"{what} dq b{bi} h{hi} m{m}")
        for n in k_blocks:
            keys = torch.arange(n * BK, min(x.lk, (n + 1) * BK), device=x.q.device)
            rows = _key_rows(x, bi, hi, n)
            if len(rows) == 0:
                assert not x.dk[bi, keys, hi].any() and not x.dv[bi, keys, hi].any(), (what, "empty list not zero", n)
                continue
            rk, rv = _ref_dkdv(x, bi, hi, keys, rows)
            _assert_block(x.dk[bi, keys, hi], rk, x.dtype, f"{what} dk b{bi} h{hi} n{n}")
            _assert_block(x.dv[bi, keys, hi], rv, x.dtype, f"{what} dv b{bi} h{hi} n{n}")


# ------------------------------------------------------------------------------------------------------------ inputs
_block_map_lut = B.block_map_lut


def _inputs(b, l, h, dtype, seed, lk=None):
    lk = l if lk is None else lk
    return (_randn((b, l, h, D), dtype, seed), _randn((b, lk, h, D), dtype, seed + 1), _randn((b, lk, h, D), dtype, seed + 2),
            _randn((b, l, h, D), dtype, seed + 3))


def _hand_lut(b, h, mblk, rows):
    """[b, h, mblk, topk] int32 on the GPU from rows(bi, hi, m) -> list of key blocks."""
    return torch.tensor([[[rows(bi, hi, m) for m in range(mblk)] for hi in range(h)] for bi in range(b)], dtype=torch.int32,
                        device="cuda")


# ------------------------------------------------------------------------------------------------------------ 2. cases
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("blkq", GEOMS)
def test_block_map_luts(cuda, blkq, dtype):
    """The module's own selection at b = 2, h = 3, L = 1000: ragged last query block (104 or 40 rows) and last key block (40
    keys), 5 of 16 key blocks per row.  Every block of every head."""
    q, k, v, do = _inputs(2, 1000, 3, dtype, 11)
    lut = _block_map_lut(q, k, blkq, 5)
    _check(_run(_case(q, k, v, do, lut, blkq)), f"block map q{blkq}")


HAND = {
    # name: (L, topk, rows(bi, hi, m, mblk, nblk) -> LUT row)
    "topk1": (1000, 1, lambda bi, hi, m, mb, nb: [(7 * m + 3 * hi) % nb]),
    "ragged_block_1_key": (64 * 9 + 1, 1, lambda bi, hi, m, mb, nb: [nb - 1]),
    "ragged_block_63_keys": (64 * 9 + 63, 1, lambda bi, hi, m, mb, nb: [nb - 1]),
    "block_in_every_list": (1000, 3, lambda bi, hi, m, mb, nb: sorted({5, (m + hi) % 5, 6 + (2 * m + hi) % 10})),
    "blocks_in_no_list": (1000, 4, lambda bi, hi, m, mb, nb: sorted({1 + (m + hi + j * 3) % 14 for j in range(4)})),
    "list_len_2": (1000, 2, lambda bi, hi, m, mb, nb: [(m + hi) % 8, 8 + (m + 2 * hi) % (nb - 8)]),
    "list_len_3": (1000, 3, lambda bi, hi, m, mb, nb: [(m + hi) % 5, 5 + (m % 5), nb - 1 - (m % 5)]),
    "permuted_rows": (1000, 6, None),
    "descending_rows": (1000, 6, None),
}


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("blkq", GEOMS)
@pytest.mark.parametrize("name", sorted(HAND))
def test_hand_made_luts(cuda, name, blkq, dtype):
    """topk = 1; the ragged key block alone with 1 and 63 valid keys; a key block in every list; key blocks (the first and the
    ragged last) in no list; lists of 2 and 3 entries (on 64-row blocks warpgroup 1 takes entry 1 and nothing more; topk = 1
    leaves it no entry); LUT rows permuted and descending.  b = 1, h = 2."""
    l, topk, rows = HAND[name]
    q, k, v, do = _inputs(1, l, 2, dtype, 100 + l + topk)
    mblk, nblk = B.cdiv(l, blkq), B.cdiv(l, BK)
    if rows is None:
        lut = _block_map_lut(q, k, blkq, topk)
        if name == "descending_rows":
            lut = lut.flip(-1).contiguous()
        else:
            g = torch.Generator().manual_seed(blkq)
            lut = lut.gather(-1, torch.argsort(torch.rand(lut.shape, generator=g), -1).cuda()).contiguous()
    else:
        lut = _hand_lut(1, 2, mblk, lambda bi, hi, m: rows(bi, hi, m, mblk, nblk))
    assert lut.shape[-1] == topk
    assert bool((lut.sort(-1).values.diff(dim=-1) != 0).all()), "a LUT row lists a key block twice"
    if name == "blocks_in_no_list":
        assert not bool((lut == 0).any()) and not bool((lut == nblk - 1).any())
    if name == "block_in_every_list":
        assert bool((lut == 5).any(-1).all())
    _check(_run(_case(q, k, v, do, lut, blkq)), f"{name} q{blkq}")


LARGE = [pytest.param(n, id=n) for n in ("all_x8", "ragged_last", "split_dominant")]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("blkq", GEOMS)
@pytest.mark.parametrize("name", LARGE)
def test_large_score_and_entry_split_inputs(cuda, name, blkq, dtype):
    """The large-score (q scaled by 8 or 12, the maximum in the ragged last key block) and entry-split (row maxima in
    warpgroup 1's entries, 140+ log2 units above warpgroup 0's) inputs of the large-score tests, under the row bars.  In fp16,
    ragged_last has key rows whose dS lies below fp16's normal range (peaked softmax: small P) while their dk is a normal
    value; rounding that dS into fp16's subnormals put one of them past its bar, which the kernel's per-row dS scale fixes."""
    if name in B.SPLIT:
        q, k, v, lut = B.split_case(name, blkq)
        lut = lut.cuda()
        q, k, v = (t.to(dtype).cuda() for t in (q, k, v))
    else:
        q, k, v, ratio = B.scaled_case(name, blkq)
        q, k, v = (t.to(dtype).cuda() for t in (q, k, v))
        nblk = B.cdiv(q.shape[1], BK)
        lut = _block_map_lut(q, k, blkq, max(1, min(nblk, int(ratio * nblk))))
    do = _randn(q.shape, dtype, 1)
    _check(_run(_case(q, k, v, do, lut, blkq)), f"{name} q{blkq}")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("blkq", GEOMS)
def test_shape_a_sampled(cuda, blkq, dtype):
    """Shape A (Wan2.1-1.3B at 480p): L = 32760, 12 heads, top-k 0.1 of 512 key blocks by the module's selection.  First,
    middle and last query and key blocks of heads 0, 5 and 11; the index and delta of every head."""
    l, h = 32760, 12
    q, k, v, do = _inputs(1, l, h, dtype, 32760)
    lut = _block_map_lut(q, k, blkq, 51)
    x = _run(_case(q, k, v, do, lut, blkq))
    mblk, nblk = B.cdiv(l, blkq), B.cdiv(l, BK)
    _check(x, f"shape A q{blkq}", q_blocks=(0, mblk // 2, mblk - 1), k_blocks=(0, nblk // 2, nblk - 1),
           bh=[(0, 0), (0, 5), (0, 11)])


DENSE = [pytest.param(1, 333, 77, id="333x77"), pytest.param(2, 1000, 512, id="1000x512"),
         pytest.param(1, 128, 130, id="128x130"), pytest.param(1, 1, 226, id="1x226")]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("b,lq,lk", DENSE)
def test_dense_lengths_differ(cuda, b, lq, lk, dtype):
    """The dense backward (the kDense dQ and 128-row dK / dV kernels) at lq != lk, every block of every head, sentinel rows
    past lq (dq) and lk (dk, dv)."""
    q, k, v, do = _inputs(b, lq, 2, dtype, 500 + lq + lk, lk=lk)
    _check(_run(_case(q, k, v, do, None, 128)), f"dense {lq}x{lk}")


@pytest.mark.parametrize("dtype", DTYPES)
def test_dense_shape_a_cross_attention(cuda, dtype):
    """Shape A cross-attention: 32760 queries over 512 text keys, 12 heads.  First, middle and last query blocks and every key
    block of heads 0, 5 and 11."""
    q, k, v, do = _inputs(1, 32760, 12, dtype, 77, lk=512)
    x = _run(_case(q, k, v, do, None, 128))
    _check(x, "dense shape A cross", q_blocks=(0, x.mblk // 2, x.mblk - 1), bh=[(0, 0), (0, 5), (0, 11)])


# ------------------------------------------------------------------------------------------------------------ 3. exact properties
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("blkq", GEOMS)
def test_index_readout_through_dv(cuda, blkq, dtype):
    """q = 0 and lse = log2(N) passed in, N = 64 topk keys a power of two: P = 1/N exactly.  dO rows of query block i one-hot
    in channel i mod 128, so dV[key, c] = (blkq / N) #{i = c mod 128 : key block in LUT[i]}, a small integer times a power of
    two, exact in T: it reads every key block's list, with its multiplicity per channel, out of the kernel.  dK = 0 exactly.
    b = 2, h = 3, L = 19,200: mblk = 150 or 300, so channels carry up to two or three query blocks; random LUT rows in
    random order."""
    b, h, topk = 2, 3, 4
    nblk = 300
    l = 64 * nblk                                      # full key blocks
    mblk = B.cdiv(l, blkq)
    assert mblk > D
    n = 64 * topk
    g = torch.Generator().manual_seed(blkq)
    lut = torch.stack([torch.randperm(nblk, generator=g)[:topk] for _ in range(b * h * mblk)]).view(b, h, mblk, topk)
    lut = lut.int().cuda()
    q = torch.zeros(b, l, h, D, dtype=dtype, device="cuda")
    k, v = _randn((b, l, h, D), dtype, 3), _randn((b, l, h, D), dtype, 4)
    do = torch.zeros_like(q)
    rows = torch.arange(l, device="cuda")
    do[:, rows, :, (rows // blkq) % D] = 1
    lse = torch.full((b, h, l), math.log2(n), dtype=F32, device="cuda")
    x = _run(_case(q, k, v, do, lut, blkq, o_s=torch.zeros_like(q), lse=lse))
    _check_index(x)
    member = B.block_mask(lut, nblk).permute(0, 1, 3, 2).float()                   # [b, h, nblk, mblk]
    member = F.pad(member, (0, B.cdiv(mblk, D) * D - mblk))
    counts_c = member.view(b, h, nblk, -1, D).sum(-2)                               # [b, h, nblk, channel]
    assert counts_c.max() >= 2
    want = (counts_c * (blkq / n)).repeat_interleave(BK, 2).permute(0, 2, 1, 3)     # [b, l, h, D]
    assert torch.equal(x.dv.float(), want), ("dV read-out", int((x.dv.float() != want).sum()))
    assert not x.dk.any()
    counts = (x.dv.float() * (n / blkq)).sum(-1)[:, ::BK].permute(0, 2, 1)         # list length of every key block
    assert torch.equal(counts, B.block_mask(lut, nblk).sum(2).float())
    print(f"q{blkq} {dtype}: dV = (blkq / N) x per-channel counts (up to {int(counts_c.max())}) exactly, "
          f"ex2.approx(-log2 {n}) exact")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("blkq", GEOMS)
def test_lut_row_order_leaves_dk_dv_bits(cuda, blkq, dtype):
    """The key-major lists are ascending whatever the order of a LUT row, so permuting every row must leave dK and dV bit for
    bit the same; dQ (whose sum follows the LUT order) only has to meet the row bars.  b = 2, h = 3, L = 1000."""
    q, k, v, do = _inputs(2, 1000, 3, dtype, 21)
    lut = _block_map_lut(q, k, blkq, 6)
    g = torch.Generator().manual_seed(7 + blkq)
    plut = lut.gather(-1, torch.argsort(torch.rand(lut.shape, generator=g), -1).cuda()).contiguous()
    assert not torch.equal(plut, lut)
    a = _run(_case(q, k, v, do, lut, blkq))
    x = _run(_case(q, k, v, do, plut, blkq, o_s=a.o_s, lse=a.lse))
    assert torch.equal(x.dk, a.dk) and torch.equal(x.dv, a.dv)
    _check(x, f"permuted q{blkq}", k_blocks=())


def _equivariance_inputs(dtype):
    """Inputs whose rounded operands and outputs stay away from zero by construction (no cancellation): q, |k| positive and
    small, so P is near 1/N; v zero but for channel 0 = s_j = +-1, with k_j = s_j |k_j|; dO positive, channel 0 = 1.  Then
    dP - delta = s_j - delta with |delta| < 1, dS_ij s_j > 0, and every dq, dk, dv element is a sum of one sign."""
    b, l, h = 1, 640, 2
    g = torch.Generator(device="cuda").manual_seed(5)
    u = lambda *s: torch.rand(*s, generator=g, device="cuda")
    sgn = torch.where(u(b, l, h, 1) < 0.5, -1.0, 1.0)
    q = 0.02 * (1 + u(b, l, h, D))
    k = sgn * (1 + u(b, l, h, D))
    v = torch.zeros(b, l, h, D, device="cuda")
    v[..., :1] = sgn
    do = 1 + u(b, l, h, D)
    do[..., 0] = 1
    return [t.to(dtype) for t in (q, k, v, do)]


def _scaled_run(x, s, exact=True):
    """The backward on 2^s dO (exact in T unless exact=False: dO itself in T's subnormals)."""
    y = _case(x.q, x.k, x.v, (x.do.double() * 2.0 ** s).to(x.dtype), x.lut, x.blkq, o_s=x.o_s, lse=x.lse)
    assert not exact or torch.equal(y.do.double(), x.do.double() * 2.0 ** s)
    return _run(y)


def _bits_scale(y, x, s):
    return all(torch.equal(a.double(), b.double() * 2.0 ** s) for a, b in ((y.dq, x.dq), (y.dk, x.dk), (y.dv, x.dv)))


@pytest.mark.parametrize("blkq", GEOMS)
def test_power_of_two_dO_bf16(cuda, blkq):
    """bwd(2^s dO) = 2^s bwd(dO) bit for bit in bf16 (fp32's exponent range) for s from -40 to 40, on randn inputs and the
    module's selection."""
    q, k, v, do = _inputs(1, 1000, 2, BF16, 31)
    x = _run(_case(q, k, v, do, _block_map_lut(q, k, blkq, 5), blkq))
    for s in (-40, -24, -9, -1, 1, 7, 23, 40):
        assert _bits_scale(_scaled_run(x, s), x, s), s


def _normal_or_zero(t, dtype):
    a = t.abs()
    return bool(((a == 0) | ((a >= torch.finfo(dtype).tiny) & (a <= torch.finfo(dtype).max))).all())


@pytest.mark.parametrize("blkq", GEOMS)
def test_power_of_two_dO_fp16(cuda, blkq):
    """fp16: bwd(2^s dO) = 2^s bwd(dO) bit for bit at every s where dO and every output stay in fp16's normal range or at zero,
    on inputs without cancellation (_equivariance_inputs)."""
    q, k, v, do = _equivariance_inputs(FP16)
    nblk = B.cdiv(q.shape[1], BK)
    lut = _hand_lut(1, 2, B.cdiv(q.shape[1], blkq), lambda bi, hi, m: [(m + hi) % nblk, (m + hi + 3) % nblk])
    x = _run(_case(q, k, v, do, lut, blkq))
    tiny, big = torch.finfo(FP16).tiny, torch.finfo(FP16).max
    lo, hi_ = -1000, 1000                     # s with tiny <= |a| 2^s <= max / 2 for every nonzero a that scales with dO
    for a in (x.do, x.dq, x.dk, x.dv):
        a = a.double().abs()
        a = a[a != 0]
        lo = max(lo, math.ceil(math.log2(tiny / float(a.min()))))
        hi_ = min(hi_, math.floor(math.log2(big / 2 / float(a.max()))))
    print(f"q{blkq} fp16: dO and the outputs are normal or zero for s in [{lo}, {hi_}]")
    assert lo <= -3 and hi_ >= 3, (lo, hi_)
    for s in sorted({lo, lo + 1, lo // 2, -1, 1, hi_ - 1, hi_}):
        assert _bits_scale(_scaled_run(x, s), x, s), s


@pytest.mark.parametrize("blkq", GEOMS)
@pytest.mark.parametrize("shift", [6, 8, 10])
def test_fp16_small_dO(cuda, shift, blkq):
    """fp16 at the gradient magnitudes of loss-scaled training: randn q, k, v, dO = randn 2^-shift, the module's selection.
    dS then lies mostly below fp16's normal range while most dq and dk rows are still normal fp16 values; every row must meet
    the bars of an R32 that keeps fp16's significand for dS without its underflow."""
    q, k, v, _ = _inputs(1, 1000, 2, FP16, 61)
    do = _randn(q.shape, FP16, 62, scale=2.0 ** -shift)
    x = _run(_case(q, k, v, do, _block_map_lut(q, k, blkq, 5), blkq))
    normal = lambda t: float((t.double().pow(2).mean(-1).sqrt() >= torch.finfo(FP16).tiny).float().mean())
    print(f"q{blkq} dO 2^-{shift}: rows of normal size: dq {normal(x.dq):.2f}, dk {normal(x.dk):.2f}, dv {normal(x.dv):.2f}")
    assert normal(x.dq) > 0.9 and normal(x.dk) > 0.6
    _check(x, f"fp16 dO 2^-{shift} q{blkq}")


# ------------------------------------------------------------------------------------------------------------ 4. limits
@pytest.mark.parametrize("blkq", GEOMS)
def test_largest_key_block_count(cuda, blkq):
    """nblk = 65,535 (L = 4,194,240, h = 1, bf16; about 9 GB), every LUT row {0, 32767, 32768, 65534}: ids past 32767 through
    the dQ kernels' uint16 LUT staging, and key-major lists mblk long.  Sampled query blocks, the four key blocks and two
    empty ones."""
    l, nblk = 64 * 65535, 65535
    ids = [0, 32767, 32768, 65534]
    q, k, v, do = _inputs(1, l, 1, BF16, 65535)
    mblk = B.cdiv(l, blkq)
    lut = torch.tensor(ids, dtype=torch.int32, device="cuda").expand(1, 1, mblk, 4).contiguous()
    x = _run(_case(q, k, v, do, lut, blkq))
    print(f"nblk 65535 q{blkq}: backward {x.seconds:.2f} s")
    _check(x, f"nblk 65535 q{blkq}", q_blocks=(0, 1, mblk // 2, mblk - 1), k_blocks=(*ids, 1, 40000))


def test_largest_topk_128_row_blocks(cuda):
    """topk = 33,664 on 128-row blocks, every key block selected (L = 2,154,496): the dQ kernel's LUT fills its shared memory
    to the byte.  The forward with lse refuses a top-k that large, so lse is an upper bound (P <= 1: |q| max|k| sm log2e + 1
    per row) and o_s = 0, both inputs of the backward and of R64 alike.  bf16; sampled rows.  At 2.15M keys per dQ row and
    2.15M query rows per key block the fp32 accumulation allowance (2^-24 per MMA step of the |terms| sum) dominates the row
    bar, so here the bars catch gross errors (wrong blocks, garbage, unwritten rows), not a single missing entry."""
    topk = BWD_TOPK_LIMIT[128]
    l = 64 * topk
    q, k, v, do = _inputs(1, l, 1, BF16, 33664)
    q = (q.float() * 0.1).to(BF16)
    kmax = k.float().norm(dim=-1).max()
    lse = (q.float().norm(dim=-1) * kmax * (SM / math.log(2.0)) + 1).permute(0, 2, 1).contiguous()
    lut = torch.arange(topk, dtype=torch.int32, device="cuda").expand(1, 1, B.cdiv(l, 128), topk).contiguous()
    x = _run(_case(q, k, v, do, lut, 128, o_s=torch.zeros_like(q), lse=lse))
    print(f"topk {topk} q128: backward {x.seconds:.2f} s")
    mblk = x.mblk
    _check(x, f"topk {topk} q128", q_blocks=(0, mblk - 1), k_blocks=(0, topk // 2, topk - 1))


# ------------------------------------------------------------------------------------------------------------ 5. sensitivity
def _old_block_bar(got, want):
    a, b = got.double().flatten(), want.flatten()
    rel = float((a - b).norm() / b.norm())
    cos = float(torch.dot(a, b) / (a.norm() * b.norm()))
    return cos >= 0.999 and rel <= 2e-2


@pytest.mark.parametrize("blkq", GEOMS)
def test_bars_reject_kernel_faults(cuda, blkq):
    """R64 as six faulty kernels would compute it (rounded to T as their output would be), judged by the row bars: each must
    fail on at least half of the rows it changes.  Prints which faults the old block bars (cos >= 0.999, rel-L2 <= 2e-2 on
    the block) and the dense tests' whole-tensor bar (rel-L2 <= 1.5x SDPA's) accept.  Dense selection (every key block in
    every list), L = 1000, bf16, so that SDPA computes the same gradients."""
    l, h = 1000, 2
    q, k, v, do = _inputs(1, l, h, BF16, 41)
    mblk, nblk = B.cdiv(l, blkq), B.cdiv(l, BK)
    lut = torch.arange(nblk, dtype=torch.int32, device="cuda").expand(1, h, mblk, nblk).contiguous()
    x = _run(_case(q, k, v, do, lut, blkq))
    leaves = [t.detach().clone().requires_grad_() for t in (q, k, v)]
    F.scaled_dot_product_attention(*(t.transpose(1, 2) for t in leaves), scale=SM).transpose(1, 2).backward(do)
    sdpa = {"dq": leaves[0].grad, "dk": leaves[1].grad, "dv": leaves[2].grad}
    exact = {n: torch.zeros(1, l, h, D, dtype=F64, device="cuda") for n in ("dq", "dk", "dv")}
    for hi in range(h):
        for m in range(mblk):
            rows = torch.arange(m * blkq, min(l, (m + 1) * blkq), device="cuda")
            exact["dq"][0, rows, hi] = _ref_dq(x, 0, hi, rows, _query_keys(x, 0, hi, m))[0]
        for n in range(nblk):
            keys = torch.arange(n * BK, min(l, (n + 1) * BK), device="cuda")
            rk, rv = _ref_dkdv(x, 0, hi, keys, _key_rows(x, 0, hi, n))
            exact["dk"][0, keys, hi], exact["dv"][0, keys, hi] = rk[0], rv[0]

    m, n, hi = 2, 3, 1
    rows = torch.arange(m * blkq, (m + 1) * blkq, device="cuda")
    keys = torch.arange(n * BK, (n + 1) * BK, device="cuda")
    last = torch.arange((nblk - 1) * BK, l, device="cuda")
    partner = m * blkq + ((rows - m * blkq) ^ 8)
    neighbour = m * blkq + ((rows - m * blkq) ^ 1)
    listed = _key_rows(x, 0, hi, n)
    missing = listed[listed // blkq != m]                           # query block m dropped from key block n's list
    twice = torch.cat([listed, rows])                               # query block m listed twice
    entries = lut[0, hi, m].tolist()
    faults = {  # name: (output, rows or keys, (R64 of the faulty kernel, ref of the right one))
        "lse of the fragment partner (r ^ 8)": ("dq", rows, lambda: _ref_dq(x, 0, hi, rows, _query_keys(x, 0, hi, m),
                                                                            lse_rows=partner)),
        "delta of the neighbouring row": ("dq", rows, lambda: _ref_dq(x, 0, hi, rows, _query_keys(x, 0, hi, m),
                                                                      dlt_rows=neighbour)),
        "query block missing from a key list": ("dv", keys, lambda: _ref_dkdv(x, 0, hi, keys, missing)[1]),
        "query block counted twice in a list": ("dk", keys, lambda: _ref_dkdv(x, 0, hi, keys, twice)[0]),
        "ragged block's last key masked in dQ": ("dq", rows, lambda: _ref_dq(x, 0, hi, rows, _query_keys(x, 0, hi, m)[:-1])),
    }
    if blkq == 64:
        odd = [j for j in range(len(entries)) if j % 2 == 1][-1]
        kept = torch.tensor([e for j, e in enumerate(entries) if j != odd], dtype=torch.int32, device="cuda")
        faults["warpgroup 1's last entry dropped from dQ"] = ("dq", rows, lambda: _ref_dq(x, 0, hi, rows, _query_keys(x, 0, hi, m, kept)))
    accepted_old = []
    for name, (out, idx, faulty) in faults.items():
        bad = faulty()[0].to(BF16)
        if out == "dq":
            ref = _ref_dq(x, 0, hi, idx, _query_keys(x, 0, hi, m))
        else:
            rk, rv = _ref_dkdv(x, 0, hi, idx, _key_rows(x, 0, hi, n))
            ref = rk if out == "dk" else rv
        changed = (bad.double() != ref[0].to(BF16).double()).any(-1)
        block_ok, rows_ok = _judge(bad, ref, BF16, f"fault: {name}", record=None)
        rejected = int((~rows_ok & changed).sum())
        assert rejected >= 0.5 * int(changed.sum()) and int(changed.sum()) > 0, (name, rejected, int(changed.sum()))
        whole = getattr(x, out).clone()
        whole[0, idx, hi] = bad
        e_bad = float((whole.double() - exact[out]).norm() / exact[out].norm())
        e_sdpa = float((sdpa[out].double() - exact[out]).norm() / exact[out].norm())
        old = [nm for nm, ok in (("block cos/rel-L2", _old_block_bar(bad, ref[0])), ("1.5x SDPA", e_bad <= 1.5 * e_sdpa)) if ok]
        print(f"q{blkq} {name}: new bars reject {rejected}/{int(changed.sum())} changed rows; accepted by: {', '.join(old) or '-'}")
        if old:
            accepted_old.append(name)
    print(f"q{blkq}: faults the old bars accept: {accepted_old}")
