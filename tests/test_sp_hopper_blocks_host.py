"""CPU checks of sequence parallelism on the Hopper SageSLA block family (BLKQ=64, BLKK=128): argument validation of the
sequence-major entry points with a block size, the binding of the hooks to the family they were built for, and `gloo` runs of
the dist.py plumbing at (64, 128) with the CPU oracle injected as the per-rank primitives."""
import ctypes
import os
import socket
import sys
from types import SimpleNamespace

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from turbodiffusion_b200.dist import (SequenceParallel, SPAttention, UlyssesAttention, UnevenUlyssesAttention,  # noqa: E402
                                      cdiv)
from turbodiffusion_b200.SLA import utils as sla_utils  # noqa: E402

BQ, BK = 64, 128
INVALID, UNSUPPORTED = -1, -2


def _p(v=4096):
    return ctypes.c_void_p(v)          # non-null, 16-byte aligned, never dereferenced: validation runs before any CUDA call


@pytest.fixture(scope="module")
def lib():
    from turbodiffusion_b200 import _build, _lib
    _build.build()
    return _lib.lib()


def _quant(lib, blkk=128, d=128, kmean=None):
    return lib.tdb200_sla_quant_k_seq_blocks(_p(), _p() if kmean is None else kmean, 0, 1, 256, 2, d, _p(), _p(), _p(), blkk,
                                             None)


def _attn(lib, blkq=BQ, blkk=BK, b=1, d=128, topk=1, q_i8=None, dtype=0):
    return lib.tdb200_sla_attn_fwd_kseq_blocks(_p() if q_i8 is None else q_i8, _p(), _p(), _p(), _p(), _p(), dtype, _p(), topk,
                                               _p(), _p(), _p(), _p(), b, 256, 256, 2, d, 0.088, blkq, blkk, None)


def test_argument_validation_of_the_sequence_major_block_entry_points(lib):
    cases = [
        ("quant block 32", lambda: _quant(lib, blkk=32), UNSUPPORTED, b"block"),
        ("quant block 256", lambda: _quant(lib, blkk=256), UNSUPPORTED, b"block"),
        ("quant head dim", lambda: _quant(lib, d=96), UNSUPPORTED, b"head dim"),
        ("quant null", lambda: _quant(lib, kmean=ctypes.c_void_p(0)), INVALID, b"null"),
        ("quant null 64", lambda: _quant(lib, blkk=64, kmean=ctypes.c_void_p(0)), INVALID, b"null"),
        ("attn block pair 64x64", lambda: _attn(lib, blkq=64, blkk=64), UNSUPPORTED, b"block"),
        ("attn block pair 128x128", lambda: _attn(lib, blkq=128, blkk=128), UNSUPPORTED, b"block"),
        ("attn batch", lambda: _attn(lib, b=2), UNSUPPORTED, b"batch"),
        ("attn batch 128x64", lambda: _attn(lib, b=2, blkq=128, blkk=64), UNSUPPORTED, b"batch"),
        ("attn head dim", lambda: _attn(lib, d=64), UNSUPPORTED, b"head dim"),
        ("attn head dim 128x64", lambda: _attn(lib, d=64, blkq=128, blkk=64), UNSUPPORTED, b"head dim"),
        ("attn null", lambda: _attn(lib, q_i8=ctypes.c_void_p(0)), INVALID, b"null"),
        # lk = 256: nblk = 2 for 128-row key blocks, so topk = 3 is out of range ...
        ("attn topk follows blkk", lambda: _attn(lib, topk=3), INVALID, b"topk"),
        # ... but not for 64-row key blocks (nblk = 4): that call gets past the topk check and stops at the dtype tag
        ("attn topk 128x64", lambda: _attn(lib, topk=3, blkq=128, blkk=64, dtype=7), UNSUPPORTED, b"dtype"),
        ("attn topk 2 of 2", lambda: _attn(lib, topk=2, dtype=7), UNSUPPORTED, b"dtype"),
    ]
    for name, call, code, needle in cases:
        rc = call()
        msg = lib.tdb200_last_error() or b""
        assert rc == code, (name, rc, msg)
        assert needle in msg, (name, msg)


@pytest.fixture
def served():
    """Restores the served arch after a test that changes it."""
    prev = sla_utils.SERVED_ARCH
    yield sla_utils.set_served_arch
    sla_utils.set_served_arch(prev)


def _model(heads_per_block):
    sla = SimpleNamespace(dtype=torch.bfloat16, quantised_qk=True, feature=0, topk=0.1)
    return SimpleNamespace(blocks=[SimpleNamespace(heads=h, sla=sla, attn_hook=None) for h in heads_per_block])


@pytest.mark.parametrize("mode,heads,hook_type", [("allgather", 2, SPAttention), ("ulysses", 2, UlyssesAttention),
                                                  ("ulysses", 3, UnevenUlyssesAttention)])
def test_install_builds_hooks_for_the_hopper_family(served, mode, heads, hook_type):
    served("sm90")
    sp = SequenceParallel(1024, world=2, rank=0)
    model = _model([heads, heads])
    assert sp.install(model, mode, sage_arch="sm90") == mode
    for blk in model.blocks:
        hook = blk.attn_hook
        assert type(hook) is hook_type
        assert hook.sage_arch == "sm90" and hook.blocks == (BQ, BK)
        assert hook.prims.sage_arch == "sm90" and (hook.prims.blkq, hook.prims.blkk) == (BQ, BK)


def test_install_refuses_a_family_mismatch_before_touching_the_model(served):
    sp = SequenceParallel(1024, world=2, rank=0)
    for served_arch, built_for in (("sm90", "sm100"), ("sm100", "sm90")):
        served(served_arch)
        model = _model([2])
        with pytest.raises(NotImplementedError, match=f"{built_for}.*{served_arch}"):
            sp.install(model, "allgather", sage_arch=built_for)
        assert model.blocks[0].attn_hook is None
    with pytest.raises(ValueError, match="sage_arch"):
        sp.install(_model([2]), "allgather", sage_arch="sm86")


def test_hooks_built_for_the_hopper_family_refuse_a_later_switch(served):
    served("sm90")
    sp = SequenceParallel(1024, world=2, rank=0)
    hooks = [SPAttention(sp, None, "sm90"), UlyssesAttention(sp, None, sage_arch="sm90"),
             UnevenUlyssesAttention(sp, None, heads=3, sage_arch="sm90")]
    served("sm100")
    for hook in hooks:
        with pytest.raises(NotImplementedError, match="sm90.*sm100"):
            hook(None, None, None)


# ---- gloo runs at (64, 128) ----------------------------------------------------------------------------------------------
class OraclePrims:
    """CPU per-rank primitives built from the oracle on (blkq, blkk) blocks: the 16-bit K exchange, and with `int8_k` the
    INT8-K exchange (128-row partial sums, global mean, per-rank smoothing / Sage INT8 / pooling per blkk rows)."""

    def __init__(self, O, proj_w, proj_b, topk, blkq, blkk, int8_k):
        self.O, self.w, self.b, self.topk, self.blkq, self.blkk, self.int8_k = O, proj_w, proj_b, topk, blkq, blkk, int8_k

    def moments(self, k, v):
        phi = torch.softmax(k.transpose(1, 2).float(), -1).to(k.dtype).float()   # [1,H,rows,D]
        kv, ksum = v.transpose(1, 2).float().transpose(-1, -2) @ phi, phi.sum(-2)
        buf = torch.cat([kv.reshape(-1), ksum.reshape(-1)]).contiguous()         # one buffer, like SLA.core.linear_moments
        return buf[: kv.numel()].view(kv.shape), buf[kv.numel():].view(ksum.shape)

    def _linear(self, qh, kv, ksum):
        pq = torch.softmax(qh.float(), -1).to(qh.dtype).float()
        num = pq @ kv.transpose(-1, -2)
        den = 1e-5 + (pq * ksum[:, :, None, :]).sum(-1, keepdim=True)
        return (num / den) @ self.w.float().t() + self.b.float()

    def attention(self, q, k_full, v_full, lk, kv, ksum, qprep=None):
        O = self.O
        qh = q.transpose(1, 2).contiguous()
        kh = k_full[:, :lk].transpose(1, 2).contiguous()
        vh = v_full[:, :lk].transpose(1, 2).contiguous()
        _, lut, _ = O.get_block_map(qh, kh, self.topk, self.blkq, self.blkk)
        o_s = O.sparse_attention(qh, kh, vh, lut, self.blkq, self.blkk)
        return (o_s + self._linear(qh, kv, ksum)).to(q.dtype).transpose(1, 2).contiguous()

    def prepare_q(self, q):
        return None

    def k_partials(self, k):
        _, rows, h, d = k.shape
        kf = torch.nn.functional.pad(k[0].float(), (0, 0, 0, 0, 0, (-rows) % 128))       # [rows_p, H, D]
        return kf.view(-1, 128, h, d).sum(1).permute(1, 0, 2).contiguous().unsqueeze(0)   # [1, H, chunks, D]

    def k_mean(self, partials, l_total):
        return partials.sum(2) / l_total

    def k_quant(self, k, kmean, out=None):
        O = self.O
        arg = k.transpose(1, 2) - kmean.to(k.dtype)[:, :, None, :]                    # T(k - T(mean)), utils.py:56
        k_i8, k_s = O.sage_quant_blocks(arg, self.blkk)
        assert k_s.shape[-1] == cdiv(k.shape[1], self.blkk)
        return k_i8.transpose(1, 2).contiguous(), k_s, O.mean_pool(arg, self.blkk)

    def attention_i8(self, q, qprep, k_i8_full, k_scale, k_pool, kmean, v_full, lk, kv, ksum):
        O = self.O
        assert k_scale.shape[-1] == k_pool.shape[2] == cdiv(lk, self.blkk)    # SPAttention reassembled BLKK-row key blocks
        qh = q.transpose(1, 2).contiguous()
        vh = v_full[:, :lk].transpose(1, 2).contiguous()
        k8 = k_i8_full[:, :lk].transpose(1, 2).contiguous()
        scores = (O.mean_pool(qh, self.blkq).float() @ k_pool.float().transpose(-1, -2)).to(q.dtype)
        nblk = scores.shape[-1]
        _, lut = O.select_topk(scores, min(nblk, int(self.topk * nblk)))
        q_i8, q_s = O.sage_quant_blocks(qh, self.blkq)
        o_s = O.sparse_attention(qh, k8, vh, lut, self.blkq, self.blkk, p_dtype=q.dtype, q_i8=q_i8, q_s=q_s, k_i8=k8,
                                 k_s=k_scale)
        return (o_s + self._linear(qh, kv, ksum)).to(q.dtype).transpose(1, 2).contiguous()


def _worker(rank, world, port, l, h, d, topk, out_path, mode):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from oracle import td_oracle as O
    sla_utils.set_served_arch("sm90")
    g = torch.Generator().manual_seed(123)
    q = torch.randn(1, l, h, d, generator=g).bfloat16()
    k = (torch.randn(1, l, h, d, generator=g) + torch.randn(1, 1, h, d, generator=g) * 2).bfloat16()
    v = torch.randn(1, l, h, d, generator=g).bfloat16()
    w, b = torch.randn(d, d, generator=g) * 0.05, torch.randn(d, generator=g) * 0.05
    sp = SequenceParallel(l, world, rank)
    if mode == "ulysses":
        class Prims:
            @staticmethod
            def attend(get_q, get_k, get_v):
                kf, qf, vf = get_k(), get_q(), get_v()     # the order the GPU primitives consume them in
                return O.sla_forward(qf, kf, vf, w, b, topk, BQ, BK, mode="exact")
        attn = (UlyssesAttention(sp, Prims, sage_arch="sm90") if h % world == 0
                else UnevenUlyssesAttention(sp, Prims, h, sage_arch="sm90"))
    else:
        attn = SPAttention(sp, OraclePrims(O, w, b, topk, BQ, BK, int8_k=mode == "allgather_i8"), "sm90")
        assert attn._use_int8(k) == (mode == "allgather_i8")
    sl = slice(sp.row_begin, sp.row_end)
    out_local = attn(q[:, sl].contiguous(), k[:, sl].contiguous(), v[:, sl].contiguous())
    full = sp.gather_rows(out_local[0].reshape(sp.local_rows, h * d))
    if rank == 0:
        ref = O.sla_forward(q, k, v, w, b, topk, BQ, BK, mode="sage" if mode == "allgather_i8" else "exact")
        torch.save({"stats": O.stats(full, ref[0].reshape(l, h * d))}, out_path)
    dist.barrier()
    dist.destroy_process_group()


def _spawn(tmp_path, world, l, h, d, mode):
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    out = str(tmp_path / "sp.pt")
    mp.spawn(_worker, args=(world, port, l, h, d, 0.3, out, mode), nprocs=world, join=True)
    return torch.load(out)["stats"]


@pytest.mark.parametrize("l,world", [(600, 2), (1000, 3)])
def test_int8_k_exchange_hopper_blocks_gloo(tmp_path, l, world):
    """INT8-K mode on 128-row key blocks (short last ranks: 600 = 384 + 216, 1000 = 384 + 384 + 232) equals the
    single-process Sage emulation at (64, 128) up to the summation order of the key mean."""
    assert _spawn(tmp_path, world, l, 2, 128, "allgather_i8")["rel_l2"] < 5e-3


@pytest.mark.parametrize("l", [600, 1000])
def test_bf16_k_exchange_hopper_blocks_gloo(tmp_path, l):
    """d = 64 keeps the 16-bit K exchange; every rank prepares the whole key sequence on 128-row key blocks."""
    assert _spawn(tmp_path, 2, l, 2, 64, "allgather")["rel_l2"] < 5e-3   # only bf16 output rounding differs


@pytest.mark.parametrize("l,h", [(600, 2), (1000, 3)])
def test_ulysses_hopper_blocks_gloo(tmp_path, l, h):
    """Head<->sequence mode with even (2 over 2) and uneven (3 over 2) heads, the per-rank forward on (64, 128) blocks."""
    assert _spawn(tmp_path, 2, l, h, 64, "ulysses")["rel_l2"] < 1e-4
