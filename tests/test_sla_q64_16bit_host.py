"""CPU checks of SparseLinearAttention's (BLKQ, BLKK) = (64, 64) path: argument validation of the general 16-bit entry points,
the workspace size at blkq = 64, the closed-form backward (tests/sla_backward_oracle.py) at blkq = 64 against torch.autograd
through the oracle's forward, and which constructor arguments warn."""
import ctypes
import warnings

import pytest
import torch

from oracle import td_oracle as O

import sla_backward_oracle as B

INVALID, UNSUPPORTED, WORKSPACE = -1, -2, -5
BQ, BK = 64, 64


def _p(v=4096):
    return ctypes.c_void_p(v)


@pytest.fixture(scope="module")
def lib():
    from turbodiffusion_b200 import _build, _lib
    _build.build()
    return _lib.lib()


def _fwd(lib, q=True, topk=4, d=128, dtype=0, l=256, blkq=BQ, blkk=BK, feature=0, b=1):
    return lib.tdb200_sla_attn16_fwd(_p() if q else None, _p(), _p(), dtype, _p(), topk, _p(), _p(), _p(), _p(), b, l, l, 2, d, 0.088,
                                     feature, blkq, blkk, None)


def _fwd_lse(lib, q=True, topk=4, d=128, dtype=0, l=256, blkq=BQ, blkk=BK, b=1):
    return lib.tdb200_sla_attn16_fwd_lse(_p() if q else None, _p(), _p(), dtype, _p(), topk, _p(), _p(), b, l, 2, d, 0.088, blkq, blkk,
                                         None)


def _bwd(lib, ws=_p(), ws_bytes=1 << 30, topk=4, d=128, dtype=0, l=256, lse=True, blkq=BQ, blkk=BK, b=1, h=2):
    return lib.tdb200_sla_attn16_bwd(_p(), _p(), _p(), _p(), _p(), _p() if lse else None, dtype, _p(), topk, _p(), _p(), _p(), ws,
                                     ws_bytes, b, l, h, d, 0.088, blkq, blkk, None)


# The backward's own limits (tdb200_sla_attn16_bwd; the dQ kernels stage a LUT row on chip as uint16 ids):
#   nblk <= 65535 (grid.x of the dK / dV kernel; the uint16 ids), and b * h * mblk * topk <= 2^31 - 1 (the key-major index);
#   1024 (alignment) + kOffLut + round16(2 topk) <= 227 KB, kOffLut the dQ kernel's shared memory before its LUT:
#     (128, 64)  sla_bwd_dq_kernel      Q 32768 | dO 32768 | 3 K + 3 V stages of 16384 | 256 barriers = 164096
#                232448 - 1024 - 164096 = 67328 = 2 * 33664: topk 33664 fits, 33665 is refused for its LUT.  topk <= nblk
#                puts L >= 64 topk and mblk = L / 128 ~ topk / 2, so at b = h = 1 the index bound (topk^2 / 2) is far away.
#     (64, 64)   sla_bwd_dq_q64_kernel  Q 16384 | dO 16384 | 3 K + 3 V stages of 16384 | 256 barriers = 131328
#                the LUT would allow topk <= (232448 - 1024 - 131328) / 2 = 50048, but mblk = L / 64 >= nblk >= topk, so
#                b * h * mblk * topk >= topk^2 and the index bound refuses first: 46340^2 <= 2^31 - 1 < 46341^2.  The LUT
#                refusal cannot be reached on 64-row blocks.
BWD_TOPK_LIMIT = {128: 33664, 64: 46340}
BWD_MAX_NBLK = 65535
# The 16-bit forwards' limit (tdb200_sla_attn16_fwd and _fwd_lse, sla_attn.cu launch()): 1024 (alignment) + Lay::kOffLut +
# round16(2 topk) (uint16 ids) + 4 topk (a k_scale copy the 16-bit kernels do not read) <= 227 KB = 232448.
# Lay<128, true, BQ, 64>: Q BQ*256 | 3 K + 3 V stages of 16384 | KVW 32768 | 256 B of barriers (the lse forward reserves KVW too).
#   (128, 64)  32768 + 98304 + 32768 + 256 = 164096;  232448 - 1024 - 164096 = 67328 = round16(22440) + 44880
#              = 22448 + 44880: topk 11220 fits exactly; 11221 needs round16(22442) + 44884 = 67332 > 67328.
#   (64, 64)   16384 + 98304 + 32768 + 256 = 147712;  232448 - 1024 - 147712 = 83712 = round16(27904) + 55808
#              = 27904 + 55808: topk 13952 fits exactly; 13953 needs round16(27906) + 55812 = 83732 > 83712.
FWD_TOPK_LIMIT = {128: 11220, 64: 13952}


def _fwd_at(lib, fn, blkq, topk):
    """A forward call (fn: _fwd or _fwd_lse) at b = 1, L = 64 topk: every key block selected."""
    return fn(lib, topk=topk, l=64 * topk, blkq=blkq)


def _bwd_at(lib, blkq, topk, nblk=None, ws_bytes=None):
    """A backward call at b = h = 1 with L = 64 * nblk (default: topk key blocks, every one selected)."""
    l = 64 * (topk if nblk is None else nblk)
    if ws_bytes is None:
        ws_bytes = lib.tdb200_sla_attn16_bwd_workspace_bytes(1, 1, l, topk, blkq)
    return _bwd(lib, ws_bytes=ws_bytes, topk=topk, l=l, blkq=blkq, b=1, h=1)


def test_argument_validation(lib):
    ws_need = lib.tdb200_sla_attn16_bwd_workspace_bytes(1, 2, 256, 4, BQ)
    cases = [("fwd null", lambda: _fwd(lib, q=False), INVALID, b"null"),
             ("fwd bad shape", lambda: _fwd(lib, b=0), INVALID, b"shape"),
             ("fwd topk 0", lambda: _fwd(lib, topk=0), INVALID, b"topk"),
             ("fwd topk > nblk", lambda: _fwd(lib, topk=5), INVALID, b"topk"),
             ("fwd head dim", lambda: _fwd(lib, d=64), UNSUPPORTED, b"head dim"),
             ("fwd dtype", lambda: _fwd(lib, dtype=7), UNSUPPORTED, b"dtype"),
             ("fwd feature", lambda: _fwd(lib, feature=3), INVALID, b"feature"),
             ("lse null", lambda: _fwd_lse(lib, q=False), INVALID, b"null"),
             ("lse bad shape", lambda: _fwd_lse(lib, b=0), INVALID, b"shape"),
             ("lse topk 0", lambda: _fwd_lse(lib, topk=0), INVALID, b"topk"),
             ("lse topk > nblk", lambda: _fwd_lse(lib, topk=5), INVALID, b"topk"),
             ("lse head dim", lambda: _fwd_lse(lib, d=64), UNSUPPORTED, b"head dim"),
             ("lse dtype", lambda: _fwd_lse(lib, dtype=7), UNSUPPORTED, b"dtype"),
             ("bwd null lse", lambda: _bwd(lib, lse=False), INVALID, b"null"),
             ("bwd null workspace", lambda: _bwd(lib, ws=None), INVALID, b"null"),
             ("bwd bad shape", lambda: _bwd(lib, b=0), INVALID, b"shape"),
             ("bwd topk 0", lambda: _bwd(lib, topk=0), INVALID, b"topk"),
             ("bwd topk > nblk", lambda: _bwd(lib, topk=5), INVALID, b"topk"),
             ("bwd head dim", lambda: _bwd(lib, d=64), UNSUPPORTED, b"head dim"),
             ("bwd dtype", lambda: _bwd(lib, dtype=3), UNSUPPORTED, b"dtype"),
             ("bwd workspace", lambda: _bwd(lib, ws_bytes=ws_need - 1), WORKSPACE, b"workspace"),
             ("workspace bad shape", lambda: lib.tdb200_sla_attn16_bwd_workspace_bytes(0, 2, 256, 4, BQ), INVALID, b"shape")]
    for blkq, blkk in [(32, 64), (64, 128), (128, 128)]:
        cases += [(f"fwd blocks {blkq}x{blkk}", lambda q=blkq, k=blkk: _fwd(lib, blkq=q, blkk=k), UNSUPPORTED, b"block"),
                  (f"lse blocks {blkq}x{blkk}", lambda q=blkq, k=blkk: _fwd_lse(lib, blkq=q, blkk=k), UNSUPPORTED, b"block"),
                  (f"bwd blocks {blkq}x{blkk}", lambda q=blkq, k=blkk: _bwd(lib, blkq=q, blkk=k), UNSUPPORTED, b"block")]
    cases.append(("workspace blkq 32", lambda: lib.tdb200_sla_attn16_bwd_workspace_bytes(1, 2, 256, 4, 32), UNSUPPORTED, b"block"))
    cases += [("bwd q128 topk limit + 1", lambda: _bwd_at(lib, 128, BWD_TOPK_LIMIT[128] + 1), UNSUPPORTED, b"LUT"),
              ("bwd q64 topk limit + 1", lambda: _bwd_at(lib, 64, BWD_TOPK_LIMIT[64] + 1), UNSUPPORTED, b"dimension too large"),
              ("bwd q64 LUT bound + 1", lambda: _bwd_at(lib, 64, 50049), UNSUPPORTED, b"dimension too large")]
    for blkq in (128, 64):
        cases += [(f"fwd q{blkq} topk limit + 1", lambda q=blkq: _fwd_at(lib, _fwd, q, FWD_TOPK_LIMIT[q] + 1), UNSUPPORTED,
                   b"on-chip LUT"),
                  (f"lse q{blkq} topk limit + 1", lambda q=blkq: _fwd_at(lib, _fwd_lse, q, FWD_TOPK_LIMIT[q] + 1), UNSUPPORTED,
                   b"on-chip LUT")]
        cases.append((f"bwd q{blkq} nblk 65536", lambda q=blkq: _bwd_at(lib, q, 4, nblk=BWD_MAX_NBLK + 1, ws_bytes=1 << 40),
                      UNSUPPORTED, b"dimension too large"))
    for name, call, code, needle in cases:
        rc = call()
        msg = lib.tdb200_last_error() or b""
        assert rc == code, (name, rc, msg)
        assert needle in msg, (name, msg)


def test_valid_calls_pass_validation(lib):
    """Well-formed (64, 64) calls, with exactly the queried workspace, and the forwards at their largest top-k on both block
    heights, get past validation: on a host without a GPU they stop at the device check."""
    if torch.cuda.is_available():
        pytest.skip("this check is for hosts without a GPU")
    calls = [lambda: _fwd(lib, feature=2), lambda: _fwd_lse(lib),
             lambda: _bwd(lib, ws_bytes=lib.tdb200_sla_attn16_bwd_workspace_bytes(1, 2, 256, 4, BQ))]
    for blkq, topk in FWD_TOPK_LIMIT.items():     # the forwards' largest top-k (one more is refused, test_argument_validation)
        calls += [lambda q=blkq, t=topk: _fwd_at(lib, _fwd, q, t), lambda q=blkq, t=topk: _fwd_at(lib, _fwd_lse, q, t)]
    for call in calls:
        assert call() in (-3, -4) and lib.tdb200_last_error()


def test_backward_limits_pass_validation(lib):
    """Each of the backward's limits is accepted by validation (one more is refused, test_argument_validation): the largest
    top-k of both block heights with every key block selected, and 65,535 key blocks at both heights.  On a host without a
    GPU the calls stop at the device check."""
    if torch.cuda.is_available():
        pytest.skip("this check is for hosts without a GPU")
    for blkq in (128, 64):
        for name, call in ((f"q{blkq} topk {BWD_TOPK_LIMIT[blkq]}", lambda: _bwd_at(lib, blkq, BWD_TOPK_LIMIT[blkq])),
                           (f"q{blkq} nblk {BWD_MAX_NBLK}", lambda: _bwd_at(lib, blkq, 4, nblk=BWD_MAX_NBLK))):
            rc = call()
            msg = lib.tdb200_last_error() or b""
            assert rc in (-3, -4) and msg, (name, rc, msg)


@pytest.mark.parametrize("b,h,l,topk", [(1, 2, 256, 4), (2, 3, 1000, 7), (1, 40, 75600, 118), (1, 12, 32760, 51)])
def test_workspace_size_formula(lib, b, h, l, topk):
    def a(x):
        return (x + 255) // 256 * 256
    nblk = (l + 63) // 64
    for blkq in (128, 64):
        mblk = (l + blkq - 1) // blkq
        want = a(4 * b * h * l) + a(4 * b * h * (nblk + 1)) + a(4 * b * h * nblk) + a(4 * b * h * mblk * topk)
        assert lib.tdb200_sla_attn16_bwd_workspace_bytes(b, h, l, topk, blkq) == want
    assert lib.tdb200_sla_attn16_bwd_workspace_bytes(b, h, l, topk, 128) == lib.tdb200_sla_attn_bwd_workspace_bytes(b, h, l, topk)


def _lut(b, h, l, topk, seed, unselected=()):
    """Random distinct key blocks per 64-row query block; the blocks in `unselected` are never chosen."""
    g = torch.Generator().manual_seed(seed)
    mblk, nblk = (l + BQ - 1) // BQ, (l + BK - 1) // BK
    allowed = torch.tensor([n for n in range(nblk) if n not in unselected])
    lut = torch.empty(b, h, mblk, topk, dtype=torch.int32)
    for bi in range(b):
        for hi in range(h):
            for mi in range(mblk):
                lut[bi, hi, mi] = allowed[torch.randperm(len(allowed), generator=g)[:topk]].sort().values.int()
    return lut


@pytest.mark.parametrize("b,h,l,topk,unselected", [(1, 1, 1000, 3, (4,)), (2, 1, 256, 2, ()), (1, 2, 300, 2, (0,))])
def test_closed_form_backward_matches_autograd(b, h, l, topk, unselected):
    """B.sparse_attention_bwd_dq / _dkdv at blkq = 64 (float64, given lse and delta) against torch.autograd through
    O.sparse_attention(blkq=64, blkk=64); ragged tails (1000 = 15*64 + 40, 300 = 4*64 + 44) and a key block that no query
    block selects are included."""
    g = torch.Generator().manual_seed(17 + l)
    q, k, v, d_o = (torch.randn(b, h, l, 128, generator=g, dtype=torch.float64) for _ in range(4))
    lut = _lut(b, h, l, topk, 3 + l, unselected)
    qf, kf, vf = (t.float().requires_grad_() for t in (q, k, v))
    O.sparse_attention(qf, kf, vf, lut, BQ, BK).backward(d_o.float())
    lse = B.sparse_attention_lse(q, k, lut, BQ, BK)
    delta = (O.sparse_attention(q, k, v, lut, BQ, BK).double() * d_o).sum(-1)
    for bi in range(b):
        for hi in range(h):
            for mi in range((l + BQ - 1) // BQ):
                got = B.sparse_attention_bwd_dq(q, k, v, d_o, lut, lse, delta, bi, hi, mi, BQ, BK)
                torch.testing.assert_close(got, qf.grad[bi, hi, mi * BQ:(mi + 1) * BQ].double(), rtol=1e-4, atol=1e-4)
            for ni in range((l + BK - 1) // BK):
                dk, dv = B.sparse_attention_bwd_dkdv(q, k, v, d_o, lut, lse, delta, bi, hi, ni, BQ, BK)
                torch.testing.assert_close(dk, kf.grad[bi, hi, ni * BK:(ni + 1) * BK].double(), rtol=1e-4, atol=1e-4)
                torch.testing.assert_close(dv, vf.grad[bi, hi, ni * BK:(ni + 1) * BK].double(), rtol=1e-4, atol=1e-4)
                if ni in unselected:
                    assert not dk.any() and not dv.any()


def _warnings(*args, **kw):
    from turbodiffusion_b200.SLA import SparseLinearAttention
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        mod = SparseLinearAttention(*args, **kw)
    return mod, [w for w in rec if "block selection differs" in str(w.message)]


def test_constructor_warns_only_for_unserved_block_sizes():
    mod, rec = _warnings(128, 0.1)
    assert not rec and mod.block_sizes(0) == (64, 64)
    mod, rec = _warnings(128, 0.1, BLKQ=128, BLKK=64)
    assert not rec and mod.block_sizes(0) == (128, 64)
    for args, kw in [((128, 0.1), {"BLKQ": 32, "BLKK": 64}), ((64, 0.1), {}), ((64, 0.1), {"BLKQ": 64, "BLKK": 64})]:
        mod, rec = _warnings(*args, **kw)
        assert len(rec) == 1 and mod.block_sizes(0) == (128, 64), (args, kw)
