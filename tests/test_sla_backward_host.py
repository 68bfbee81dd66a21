"""CPU checks of the SparseLinearAttention backward: argument validation of its C entry points, the workspace size, the
closed-form sparse-attention backward (tests/sla_backward_oracle.py) against torch.autograd through the oracle's forward, and the d = 64 refusal of the training path."""
import ctypes

import pytest
import torch

from oracle import td_oracle as O

import sla_backward_oracle as B

INVALID, UNSUPPORTED, WORKSPACE = -1, -2, -5


def _p(v=4096):
    return ctypes.c_void_p(v)


@pytest.fixture(scope="module")
def lib():
    from turbodiffusion_b200 import _build, _lib
    _build.build()
    return _lib.lib()


def _fwd_lse(lib, q=True, topk=4, d=128, dtype=0, l=256):
    return lib.tdb200_sla_attn_fwd_qk16_lse(_p() if q else None, _p(), _p(), dtype, _p(), topk, _p(), _p(), 1, l, 2, d, 0.088, None)


def _bwd(lib, ws=_p(), ws_bytes=1 << 30, topk=4, d=128, dtype=0, l=256, lse=True):
    return lib.tdb200_sla_attn_bwd_qk16(_p(), _p(), _p(), _p(), _p(), _p() if lse else None, dtype, _p(), topk, _p(), _p(), _p(), ws,
                                        ws_bytes, 1, l, 2, d, 0.088, None)


def test_argument_validation(lib):
    cases = [
        ("fwd null", lambda: _fwd_lse(lib, q=False), INVALID, b"null"),
        ("fwd topk 0", lambda: _fwd_lse(lib, topk=0), INVALID, b"topk"),
        ("fwd topk > nblk", lambda: _fwd_lse(lib, topk=5), INVALID, b"topk"),
        ("fwd head dim", lambda: _fwd_lse(lib, d=64), UNSUPPORTED, b"head dim"),
        ("fwd dtype", lambda: _fwd_lse(lib, dtype=7), UNSUPPORTED, b"dtype"),
        ("bwd null lse", lambda: _bwd(lib, lse=False), INVALID, b"null"),
        ("bwd null workspace", lambda: _bwd(lib, ws=None), INVALID, b"null"),
        ("bwd topk 0", lambda: _bwd(lib, topk=0), INVALID, b"topk"),
        ("bwd topk > nblk", lambda: _bwd(lib, topk=5), INVALID, b"topk"),
        ("bwd head dim", lambda: _bwd(lib, d=64), UNSUPPORTED, b"head dim"),
        ("bwd dtype", lambda: _bwd(lib, dtype=3), UNSUPPORTED, b"dtype"),
        ("bwd workspace", lambda: _bwd(lib, ws_bytes=lib.tdb200_sla_attn_bwd_workspace_bytes(1, 2, 256, 4) - 1), WORKSPACE,
         b"workspace"),
    ]
    for name, call, code, needle in cases:
        rc = call()
        msg = lib.tdb200_last_error() or b""
        assert rc == code, (name, rc, msg)
        assert needle in msg, (name, msg)


def test_exact_workspace_passes_validation(lib):
    """With exactly the queried workspace the call gets past validation: on a host without a GPU it stops at the device check."""
    if torch.cuda.is_available():
        pytest.skip("this check is for hosts without a GPU")
    rc = _bwd(lib, ws_bytes=lib.tdb200_sla_attn_bwd_workspace_bytes(1, 2, 256, 4))
    assert rc in (-3, -4) and lib.tdb200_last_error()


@pytest.mark.parametrize("b,h,l,topk", [(1, 2, 256, 4), (2, 3, 1000, 7), (1, 40, 75600, 118), (1, 12, 32760, 51)])
def test_workspace_size_formula(lib, b, h, l, topk):
    def a(x):
        return (x + 255) // 256 * 256
    mblk, nblk = (l + 127) // 128, (l + 63) // 64
    want = a(4 * b * h * l) + a(4 * b * h * (nblk + 1)) + a(4 * b * h * nblk) + a(4 * b * h * mblk * topk)
    assert lib.tdb200_sla_attn_bwd_workspace_bytes(b, h, l, topk) == want
    assert lib.tdb200_sla_attn_bwd_workspace_bytes(0, h, l, topk) == INVALID


def _case(b, h, l, d, seed):
    g = torch.Generator().manual_seed(seed)
    q, k, v, d_o = (torch.randn(b, h, l, d, generator=g, dtype=torch.float64) for _ in range(4))
    return q, k, v, d_o


def _lut(b, h, l, topk, seed, unselected=()):
    """Random distinct key blocks per query row; the blocks in `unselected` are never chosen."""
    g = torch.Generator().manual_seed(seed)
    mblk, nblk = (l + 127) // 128, (l + 63) // 64
    allowed = torch.tensor([n for n in range(nblk) if n not in unselected])
    lut = torch.empty(b, h, mblk, topk, dtype=torch.int32)
    for bi in range(b):
        for hi in range(h):
            for mi in range(mblk):
                lut[bi, hi, mi] = allowed[torch.randperm(len(allowed), generator=g)[:topk]].sort().values.int()
    return lut


@pytest.mark.parametrize("b,h,l,topk,unselected", [(1, 2, 300, 2, (1,)), (2, 1, 256, 4, ()), (1, 1, 200, 3, (0,))])
def test_closed_form_backward_matches_autograd(b, h, l, topk, unselected):
    """B.sparse_attention_bwd_dq / _dkdv (float64, given lse and delta) against torch.autograd through O.sparse_attention,
    which evaluates the forward in fp32; ragged tails (300 = 2*128 + 44 query rows, 4*64 + 44 keys) and a key block that no
    query block selects are included."""
    q, k, v, d_o = _case(b, h, l, 128, 17 + l)
    lut = _lut(b, h, l, topk, 3 + l, unselected)
    qf, kf, vf = (t.float().requires_grad_() for t in (q, k, v))
    o = O.sparse_attention(qf, kf, vf, lut)
    o.backward(d_o.float())
    lse = B.sparse_attention_lse(q, k, lut)
    delta = (O.sparse_attention(q, k, v, lut).double() * d_o).sum(-1)
    for bi in range(b):
        for hi in range(h):
            for mi in range((l + 127) // 128):
                got = B.sparse_attention_bwd_dq(q, k, v, d_o, lut, lse, delta, bi, hi, mi)
                want = qf.grad[bi, hi, mi * 128:(mi + 1) * 128].double()
                torch.testing.assert_close(got, want, rtol=1e-4, atol=1e-4)
            for ni in range((l + 63) // 64):
                dk, dv = B.sparse_attention_bwd_dkdv(q, k, v, d_o, lut, lse, delta, bi, hi, ni)
                torch.testing.assert_close(dk, kf.grad[bi, hi, ni * 64:(ni + 1) * 64].double(), rtol=1e-4, atol=1e-4)
                torch.testing.assert_close(dv, vf.grad[bi, hi, ni * 64:(ni + 1) * 64].double(), rtol=1e-4, atol=1e-4)
                if ni in unselected:
                    assert not dk.any() and not dv.any()


def test_lse_is_the_log2_normaliser():
    q, k, v, _ = _case(1, 1, 200, 128, 5)
    lut = _lut(1, 1, 200, 2, 6)
    lse = B.sparse_attention_lse(q, k, lut)
    row, mi = 150, 1
    cols = (lut[0, 0, mi].long()[:, None] * 64 + torch.arange(64)).reshape(-1)
    cols = cols[cols < 200]
    s = (q[0, 0, row] @ k[0, 0, cols].t()) * 128 ** -0.5
    assert abs(torch.logsumexp(s, 0).item() / torch.log(torch.tensor(2.0, dtype=torch.float64)).item() - lse[0, 0, row].item()) < 1e-12


def test_training_path_refuses_head_dim_64_before_any_cuda_call():
    from turbodiffusion_b200.SLA import SparseLinearAttention
    mod = SparseLinearAttention(64, 0.25, BLKQ=128, BLKK=64)
    q = torch.randn(1, 256, 2, 64, requires_grad=True)
    with pytest.raises(NotImplementedError, match="d = 128"):
        mod(q, q.detach(), q.detach())
