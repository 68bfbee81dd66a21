"""N>1 host logic on CPU: world_size=2 `gloo` run of the sequence-parallel attention plumbing
(turbodiffusion_b200/dist.py) with the CPU oracle injected as the per-rank primitives.  Checks that sharding +
K/V all-gather + moment all-reduce reproduce the single-process result."""
import os
import socket
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from turbodiffusion_b200.dist import (SequenceParallel, SPAttention, UlyssesAttention, UnevenUlyssesAttention,  # noqa: E402
                                      shard_rows, split_heads)


def test_shard_rows_are_128_aligned_and_cover_everything():
    for total, world in ((32760, 8), (75600, 8), (32760, 2), (600, 2), (1000, 4), (128, 1)):
        covered = 0
        for r in range(world):
            b, e, pad = shard_rows(total, world, r)
            assert b % 128 == 0 and pad % 128 == 0 and e - b <= pad
            assert b == covered
            covered = e
        assert covered == total
    b, e, _ = shard_rows(32760, 8, 7)
    assert (b, e) == (7 * 4096, 32760)          # only the last rank is short (4088 rows)
    b, e, pad = shard_rows(75600, 8, 7)
    assert pad == 74 * 128 and e - b == 75600 - 7 * 74 * 128


class OraclePrims:
    """CPU implementations of the two per-rank primitives, built from the oracle."""

    def __init__(self, O, proj_w, proj_b, topk):
        self.O, self.w, self.b, self.topk = O, proj_w, proj_b, topk

    def moments(self, k, v):
        phi = torch.softmax(k.transpose(1, 2).float(), -1).to(k.dtype).float()   # [1,H,rows,D]
        vh = v.transpose(1, 2).float()
        return vh.transpose(-1, -2) @ phi, phi.sum(-2)                            # kv [1,H,dv,dk], ksum [1,H,D]

    def attention(self, q, k_full, v_full, lk, kv, ksum, qprep=None):
        O = self.O
        qh = q.transpose(1, 2).contiguous()
        kh = k_full[:, :lk].transpose(1, 2).contiguous()
        vh = v_full[:, :lk].transpose(1, 2).contiguous()
        _, lut, _ = O.get_block_map(qh, kh, self.topk, 128, 64)
        o_s = O.sparse_attention(qh, kh, vh, lut, 128, 64)
        pq = torch.softmax(qh.float(), -1).to(q.dtype).float()
        num = pq @ kv.transpose(-1, -2)                                            # [1,H,rows,dv]
        den = 1e-5 + (pq * ksum[:, :, None, :]).sum(-1, keepdim=True)
        o_l = (num / den) @ self.w.float().t() + self.b.float()
        return (o_s + o_l).to(q.dtype).transpose(1, 2).contiguous()


class OraclePrimsI8(OraclePrims):
    """The INT8-K exchange primitives from the oracle: 128-row partial sums, global mean, per-rank smoothing / Sage INT8 /
    pooling of the rank's own key rows, and the Sage-emulation attention over the gathered INT8 K."""
    int8_k = True

    def prepare_q(self, q):
        return None

    def moments(self, k, v):
        """Both accumulators as views of ONE buffer, like turbodiffusion_b200.SLA.core.linear_moments: SPAttention then reduces
        them with a single collective."""
        kv, ksum = super().moments(k, v)
        buf = torch.cat([kv.reshape(-1), ksum.reshape(-1)]).contiguous()
        return buf[: kv.numel()].view(kv.shape), buf[kv.numel():].view(ksum.shape)

    def k_partials(self, k):
        _, rows, h, d = k.shape
        pad = (-rows) % 128
        kf = torch.nn.functional.pad(k[0].float(), (0, 0, 0, 0, 0, pad))               # [rows_p, H, D]
        return kf.view(-1, 128, h, d).sum(1).permute(1, 0, 2).contiguous().unsqueeze(0)   # [1, H, chunks, D]

    def k_mean(self, partials, l_total):
        return partials.sum(2) / l_total

    def k_quant(self, k, kmean, out=None):
        O = self.O
        kh = k.transpose(1, 2)
        arg = kh - kmean.to(k.dtype)[:, :, None, :]                                   # T(k - T(mean)), utils.py:56
        k_i8, k_s = O.sage_quant_blocks(arg, 64)
        return k_i8.transpose(1, 2).contiguous(), k_s, O.mean_pool(arg, 64)

    def attention_i8(self, q, qprep, k_i8_full, k_scale, k_pool, kmean, v_full, lk, kv, ksum):
        O = self.O
        qh = q.transpose(1, 2).contiguous()
        vh = v_full[:, :lk].transpose(1, 2).contiguous()
        k8 = k_i8_full[:, :lk].transpose(1, 2).contiguous()
        scores = (O.mean_pool(qh, 128).float() @ k_pool.float().transpose(-1, -2)).to(q.dtype)
        nblk = scores.shape[-1]
        _, lut = O.select_topk(scores, min(nblk, int(self.topk * nblk)))
        q_i8, q_s = O.sage_quant_blocks(qh, 128)
        o_s = O.sparse_attention(qh, k8, vh, lut, 128, 64, p_dtype=q.dtype, q_i8=q_i8, q_s=q_s, k_i8=k8, k_s=k_scale)
        pq = torch.softmax(qh.float(), -1).to(q.dtype).float()
        num = pq @ kv.transpose(-1, -2)
        den = 1e-5 + (pq * ksum[:, :, None, :]).sum(-1, keepdim=True)
        o_l = (num / den) @ self.w.float().t() + self.b.float()
        return (o_s + o_l).to(q.dtype).transpose(1, 2).contiguous()


def _worker(rank, world, port, l, h, d, topk, out_path, mode="allgather"):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from oracle import td_oracle as O
    g = torch.Generator().manual_seed(123)
    q = torch.randn(1, l, h, d, generator=g).bfloat16()
    k = (torch.randn(1, l, h, d, generator=g) + torch.randn(1, 1, h, d, generator=g) * 2).bfloat16()
    v = torch.randn(1, l, h, d, generator=g).bfloat16()
    w, b = torch.randn(d, d, generator=g) * 0.05, torch.randn(d, generator=g) * 0.05
    sp = SequenceParallel(l, world, rank)
    if mode == "ulysses":
        assert sp.pick_mode(h, "ulysses") == "ulysses"
        class Prims:
            @staticmethod
            def attend(get_q, get_k, get_v):
                kf, qf, vf = get_k(), get_q(), get_v()     # the order the GPU primitives consume them in
                return O.sla_forward(qf, kf, vf, w, b, topk, mode="exact")
        attn = UlyssesAttention(sp, Prims) if h % world == 0 else UnevenUlyssesAttention(sp, Prims, h)
        assert attn.q_first
    elif mode == "allgather_i8":
        attn = SPAttention(sp, OraclePrimsI8(O, w, b, topk))
        assert attn._use_int8(k)
    else:
        attn = SPAttention(sp, OraclePrims(O, w, b, topk))
    sl = slice(sp.row_begin, sp.row_end)
    out_local = attn(q[:, sl].contiguous(), k[:, sl].contiguous(), v[:, sl].contiguous())
    full = sp.gather_rows(out_local[0].reshape(sp.local_rows, h * d))
    if rank == 0:
        ref = O.sla_forward(q, k, v, w, b, topk, mode="sage" if mode == "allgather_i8" else "exact")[0].reshape(l, h * d)
        torch.save({"stats": O.stats(full, ref), "rows": [sp.row_begin, sp.row_end]}, out_path)
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("l", [600, 1000])
def test_sequence_parallel_attention_gloo_world2(tmp_path, l):
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    out = str(tmp_path / "sp.pt")
    mp.spawn(_worker, args=(2, port, l, 2, 64, 0.3, out), nprocs=2, join=True)
    res = torch.load(out)
    assert res["stats"]["rel_l2"] < 5e-3, res  # only bf16 output rounding differs from the single-process oracle


@pytest.mark.parametrize("l,world", [(600, 2), (1000, 3)])
def test_int8_k_exchange_gloo(tmp_path, l, world):
    """INT8-K mode: partial-sum all-gather -> global key mean -> per-rank Sage quantisation -> gathered INT8 K / scales / pooled
    means reassembled in global block order (uneven last rank; 3 ranks: rows_pad = 384, last rank 232 rows) equals the
    single-process Sage emulation up to the summation order of the key mean."""
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    out = str(tmp_path / "sp8.pt")
    mp.spawn(_worker, args=(world, port, l, 2, 128, 0.3, out, "allgather_i8"), nprocs=world, join=True)
    res = torch.load(out)
    assert res["stats"]["rel_l2"] < 5e-3, res


@pytest.mark.parametrize("l", [600, 1000])
def test_ulysses_attention_gloo_world2(tmp_path, l):
    """Head<->sequence all-to-all mode (uneven row shards, 2 heads over 2 ranks): every head sees the whole sequence, so the
    result is the single-process oracle's up to the CPU matmul's batch-shape-dependent summation order."""
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    out = str(tmp_path / "ul.pt")
    mp.spawn(_worker, args=(2, port, l, 2, 64, 0.3, out, "ulysses"), nprocs=2, join=True)
    res = torch.load(out)
    assert res["stats"]["rel_l2"] < 1e-4, res


@pytest.mark.parametrize("l,h", [(600, 3), (1000, 5)])
def test_uneven_ulysses_attention_gloo_world2(tmp_path, l, h):
    """heads % world != 0: rank 0 takes the extra head (3 heads -> 2+1, 5 -> 3+2), uneven row shards at the same time."""
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    out = str(tmp_path / "ul.pt")
    mp.spawn(_worker, args=(2, port, l, h, 64, 0.3, out, "ulysses"), nprocs=2, join=True)
    res = torch.load(out)
    assert res["stats"]["rel_l2"] < 1e-4, res


def test_uneven_ulysses_attention_gloo_world8_twelve_heads(tmp_path):
    """The N = 8 default for Wan-1.3B: 12 heads over 8 ranks (2,2,2,2,1,1,1,1), sixteen 128-row blocks over 8 ranks (the last rank
    holds the ragged tail), the gather-kernel reordering on both sides of the exchange."""
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    out = str(tmp_path / "ul8.pt")
    mp.spawn(_worker, args=(8, port, 2000, 12, 64, 0.3, out, "ulysses"), nprocs=8, join=True)
    res = torch.load(out)
    assert res["stats"]["rel_l2"] < 1e-4, res


def test_split_heads():
    assert split_heads(12, 8) == ([2, 2, 2, 2, 1, 1, 1, 1], [0, 2, 4, 6, 8, 9, 10, 11])
    assert split_heads(40, 8) == ([5] * 8, list(range(0, 40, 5)))
    assert split_heads(3, 2) == ([2, 1], [0, 2])


def test_pick_mode():
    sp = SequenceParallel(32760, world=8, rank=0)
    assert sp.pick_mode(12) == "ulysses" and sp.pick_mode(40) == "ulysses" and sp.pick_mode(40, "allgather") == "allgather"
    assert sp.pick_mode(4) == "allgather"                    # fewer heads than ranks: only the all-gather mode applies
    assert sp.pick_mode(12, "ulysses") == "ulysses"          # uneven head split
    with pytest.raises(ValueError):
        sp.pick_mode(4, "ulysses")                             # fewer heads than ranks
    assert SequenceParallel(32760, world=1, rank=0).pick_mode(12) == "allgather"
    assert SequenceParallel(32760, world=2, rank=0).pick_mode(12) == "allgather"   # N = 2: all-gather
    assert SequenceParallel(32760, world=4, rank=0).pick_mode(12) == "ulysses"     # from N = 4 up: all-to-all
    assert SequenceParallel(32760, world=2, rank=0).pick_mode(12, "ulysses") == "ulysses"
