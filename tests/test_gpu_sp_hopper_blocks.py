"""GPU checks of sequence parallelism on the Hopper SageSLA block family (BLKQ=64, BLKK=128; SLA.utils.set_served_arch("sm90")):
  * the split key prep on 128-row key blocks and the attention over sequence-major INT8 K are bit-identical to the
    single-GPU calls;
  * the per-rank primitives, composed in one process with the collectives replaced by concatenation, reproduce the single-GPU
    attention bit for bit when fed the same summed moments, and the module within test_gpu_dist.py's bound;
  * the real hooks in a one-rank NCCL group, eager and captured in a CUDA graph, and in a two-rank group (skipped below two
    GPUs), reproduce the single-GPU step within that bound.
"""
import os
import socket
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BQ, BK = 64, 128


def _within_dist_bound(got, ref):
    """test_gpu_dist.py's bound: only the fp32 summation order of the linear-attention moments differs, which moves the
    16-bit kvw operand and through it many outputs by one unit in the last place."""
    diff = got.float() - ref.float()
    rel_l2, max_abs = (diff.norm() / ref.float().norm()).item(), diff.abs().max().item()
    assert rel_l2 < 4e-3 and max_abs <= 0.0625, (rel_l2, max_abs)


@pytest.fixture
def sm90(cuda):
    from turbodiffusion_b200.SLA.utils import set_served_arch
    prev = set_served_arch("sm90")
    yield cuda
    set_served_arch(prev)


def _qkv(b, l, h, d, seed, kbias=2.0, dtype=torch.bfloat16):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(b, l, h, d, generator=g)
    k = torch.randn(b, l, h, d, generator=g) + torch.randn(1, 1, h, d, generator=g) * kbias
    v = torch.randn(b, l, h, d, generator=g)
    return q.to(dtype), k.to(dtype), v.to(dtype)


def _module(d, ratio, cuda, seed=5):
    from turbodiffusion_b200.SLA import SageSparseLinearAttention
    g = torch.Generator().manual_seed(seed)
    mod = SageSparseLinearAttention(d, ratio).to(cuda)
    with torch.no_grad():
        mod.proj_l.weight.copy_(torch.randn(d, d, generator=g) * 0.05)
        mod.proj_l.bias.copy_(torch.randn(d, generator=g) * 0.05)
    return mod


@pytest.mark.parametrize("l,h,d,shards", [(1000, 3, 128, (384, 384, 232)), (690, 2, 128, (384, 306)),
                                          (1000, 2, 64, (512, 488))])
def test_split_key_prep_on_128_row_key_blocks(sm90, l, h, d, shards):
    """Per-shard 128-row partial sums -> concatenated -> kmean_final, then quant_k_seq(blkk=128) per shard: the key mean, codes,
    scales and pooled means of quant_k_into(blkk=128), bit for bit (shard boundaries are multiples of 128 rows)."""
    from turbodiffusion_b200.SLA.utils import QKPrep, kmean_from_partials, kmean_partials, quant_k_into, quant_k_seq
    assert sum(shards) == l
    k = _qkv(1, l, h, d, seed=31)[1].to(sm90)
    ref = quant_k_into(QKPrep(), k, l, BK)
    bounds = [sum(shards[:i]) for i in range(len(shards) + 1)]
    partials = torch.cat([kmean_partials(k[:, a:e].contiguous()) for a, e in zip(bounds, bounds[1:])], dim=2).contiguous()
    kmean = kmean_from_partials(partials, l)
    assert torch.equal(kmean, ref.kmean)
    codes, scales, pools = [], [], []
    for a, e in zip(bounds, bounds[1:]):
        c, s, p = quant_k_seq(k[:, a:e].contiguous(), kmean, blkk=BK)
        assert c.shape == (1, e - a, h, d) and s.shape == (1, h, (e - a + BK - 1) // BK)
        codes.append(c), scales.append(s), pools.append(p)
    assert torch.equal(torch.cat(codes, 1).transpose(1, 2), ref.k_i8)
    assert torch.equal(torch.cat(scales, 2), ref.k_scale)
    assert torch.equal(torch.cat(pools, 2), ref.k_pool)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_hopper_attention_reads_sequence_major_int8_keys(sm90, dtype):
    """attn_fwd at (64, 128) on INT8 K in the gathered [1, Lk, H, D] layout, zero rows padded past lk, equals the head-major
    call bit for bit.  l = 1000: the last key block has 104 rows, the last query block 40."""
    from turbodiffusion_b200.SLA.core import attn_fwd, linear_moments, project_moments
    from turbodiffusion_b200.SLA.utils import block_map_from_pools, quant_qk
    b, l, h, d = 1, 1000, 3, 128
    q, k, v = (t.to(sm90) for t in _qkv(b, l, h, d, seed=32, dtype=dtype))
    prep = quant_qk(q, k, blkq=BQ, blkk=BK)
    topk = 3
    _, lut = block_map_from_pools(prep.q_pool, prep.k_pool, topk)
    kv, ksum = linear_moments(k, v)
    g = torch.Generator().manual_seed(3)
    kvw = project_moments((torch.randn(d, d, generator=g) * 0.05).to(sm90), kv, dtype)
    pb = (torch.randn(d, generator=g) * 0.05).to(sm90)
    ref = attn_fwd(prep, v, q, lut, topk, kvw, ksum, pb, d ** -0.5, blkq=BQ, blkk=BK)
    pad = 152                                                  # the gathered slab carries zero rows past lk
    k_seq = torch.zeros(b, l + pad, h, d, dtype=torch.int8, device=sm90)
    k_seq[:, :l] = prep.k_i8.transpose(1, 2)
    v_pad = torch.zeros(b, l + pad, h, d, dtype=dtype, device=sm90)
    v_pad[:, :l] = v
    prep.k_i8, prep.k_seq_major = k_seq, True
    got = attn_fwd(prep, v_pad, q, lut, topk, kvw, ksum, pb, d ** -0.5, lk=l, blkq=BQ, blkk=BK)
    assert torch.equal(got, ref)


def _compose_allgather(prims, q, k, v, world):
    """SPAttention's INT8-K exchange for `world` ranks in one process: the real per-rank primitives, the all-gathers replaced by
    concatenation of zero-padded per-rank buffers (the layout SPAttention gathers into), the moment all-reduce by a sum in
    rank order.  Returns (output [1, L, H, D], summed kv, summed ksum)."""
    from turbodiffusion_b200.dist import SequenceParallel, cdiv
    from turbodiffusion_b200.SLA.core import linear_moments
    _, l, h, d = q.shape
    sps = [SequenceParallel(l, world, r) for r in range(world)]
    rows_pad, cp, nbp = sps[0].rows_pad, sps[0].rows_pad // 128, sps[0].rows_pad // BK
    shard = [(sp.row_begin, sp.row_end) for sp in sps]

    def gather(parts, pad_rows):       # [rows_r, ...] per rank -> [world * pad_rows, ...], each slot zero past its rows
        out = torch.zeros(world * pad_rows, *parts[0].shape[1:], dtype=parts[0].dtype, device=parts[0].device)
        for r, t in enumerate(parts):
            out[r * pad_rows: r * pad_rows + t.shape[0]] = t
        return out

    ks = [k[:, a:e].contiguous() for a, e in shard]
    partials = gather([prims.k_partials(kr)[0].transpose(0, 1) for kr in ks], cp)
    partials = partials[: cdiv(l, 128)].transpose(0, 1).contiguous().unsqueeze(0)
    kmean = prims.k_mean(partials, l)
    quant = [prims.k_quant(kr, kmean) for kr in ks]
    nblk = cdiv(l, BK)
    k8_full = gather([c[0] for c, _, _ in quant], rows_pad).unsqueeze(0)
    k_scale = gather([s[0].transpose(0, 1) for _, s, _ in quant], nbp)[:nblk].transpose(0, 1).contiguous().unsqueeze(0)
    k_pool = gather([p[0].transpose(0, 1) for _, _, p in quant], nbp)[:nblk].transpose(0, 1).contiguous().unsqueeze(0)
    v_full = gather([v[0, a:e] for a, e in shard], rows_pad).unsqueeze(0)
    moments = [linear_moments(kr, v[:, a:e].contiguous()) for kr, (a, e) in zip(ks, shard)]
    kv, ksum = moments[0]
    for kv_r, ksum_r in moments[1:]:
        kv, ksum = kv + kv_r, ksum + ksum_r
    outs = []
    for a, e in shard:
        qr = q[:, a:e].contiguous()
        outs.append(prims.attention_i8(qr, prims.prepare_q(qr), k8_full, k_scale, k_pool, kmean, v_full, l, kv, ksum))
    return torch.cat(outs, 1), kv, ksum


@pytest.mark.parametrize("l,h,world", [(1000, 2, 2), (1000, 3, 3), (2000, 2, 8)])
def test_per_rank_composition_equals_single_gpu(sm90, l, h, world):
    """world 8 at l = 2000: rows_pad 256, the last rank 208 rows (four 64-row query blocks, the last of 16 rows)."""
    from turbodiffusion_b200.dist import GpuPrimitives
    from turbodiffusion_b200.SLA.core import attn_fwd, project_moments
    from turbodiffusion_b200.SLA.utils import block_map_from_pools, quant_qk
    d = 128
    q, k, v = (t.to(sm90) for t in _qkv(1, l, h, d, seed=40 + world))
    mod = _module(d, 0.3, sm90)
    prims = GpuPrimitives(mod, "sm90")
    assert prims.int8_k and (prims.blkq, prims.blkk) == (BQ, BK)
    got, kv, ksum = _compose_allgather(prims, q, k, v, world)
    prep = quant_qk(q, k, blkq=BQ, blkk=BK)
    topk = min(prep.nblk, int(mod.topk * prep.nblk))
    _, lut = block_map_from_pools(prep.q_pool, prep.k_pool, topk)
    kvw = project_moments(mod.proj_l.weight, kv, q.dtype)
    ref = attn_fwd(prep, v, q, lut, topk, kvw, ksum, mod.proj_l.bias.float().contiguous(), d ** -0.5, blkq=BQ, blkk=BK)
    assert torch.equal(got, ref)
    _within_dist_bound(got, mod(q, k, v))


@pytest.mark.parametrize("heads", [slice(0, 2), slice(2, 3)])
def test_ulysses_prims_on_a_head_subset_match_the_module(sm90, heads):
    from turbodiffusion_b200.dist import UlyssesGpuPrims
    l, h, d = 1000, 3, 128
    q, k, v = (t.to(sm90)[:, :, heads].contiguous() for t in _qkv(1, l, h, d, seed=50))
    mod = _module(d, 0.3, sm90)
    prims = UlyssesGpuPrims(mod, "sm90")
    got = prims.attend(lambda: q, lambda: k, lambda: v)
    _within_dist_bound(got, mod(q, k, v))


# ---- the installed hooks on WanHotPath ------------------------------------------------------------------------------------
def _stage(msg):
    print(f"[worker] {msg}", file=sys.stderr, flush=True)


def _worker(rank, world, port, out_path, mode, dim, heads, graph):
    sys.path.insert(0, ROOT)
    import threading
    import torch.distributed as dist
    # a rank that has not finished in 240 s exits with code 3, so mp.spawn reports a failure instead of waiting for ever
    watchdog = threading.Timer(240.0, lambda: (_stage("timed out"), os._exit(3)))
    watchdog.daemon = True
    watchdog.start()
    from turbodiffusion_b200.block import WanHotPath
    from turbodiffusion_b200.dist import SequenceParallel, SPAttention
    from turbodiffusion_b200.ops import wan_rope_angles
    from turbodiffusion_b200.SLA.utils import set_served_arch
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    set_served_arch("sm90")
    ffn, thw = 512, (3, 10, 23)  # L = 690 -> 6 blocks of 128: at world 2 ranks get 384 and 306 rows
    l = thw[0] * thw[1] * thw[2]
    g = torch.Generator().manual_seed(11)
    x = torch.randn(l, dim, generator=g).bfloat16().to(dev)
    e0 = (torch.randn(6, dim, generator=g) * 0.1).to(dev)
    ctx = torch.randn(64, dim, generator=g).bfloat16().to(dev)
    ang = wan_rope_angles(*thw, dim // heads, dev)
    model = WanHotPath(dim, ffn, heads, 2, dev, topk=0.4, seed=5)
    ref = model.step(x, e0, ang, ctx) if rank == 0 else None      # single-GPU result on 64/128 blocks (no hook installed yet)
    sp = SequenceParallel(l, world, rank)
    assert sp.install(model, mode, sage_arch="sm90") == mode
    hook = model.blocks[0].attn_hook
    int8 = isinstance(hook, SPAttention) and hook.prims.int8_k and dim // heads == 128
    xs, angs = sp.scatter(x), sp.scatter(ang)
    y_local = model.step(xs, e0, angs, ctx)
    y = sp.gather_rows(y_local)
    torch.cuda.synchronize()
    _stage("eager step done")
    res = {"y": y.cpu(), "ref": ref.cpu() if ref is not None else None, "int8": int8}
    if graph:
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            model.step(xs, e0, angs, ctx)
        torch.cuda.current_stream().wait_stream(s)
        cg = torch.cuda.CUDAGraph()
        with torch.cuda.graph(cg):
            y_graph = model.step(xs, e0, angs, ctx)
        _stage("captured")
        cg.replay()
        torch.cuda.synchronize()
        _stage("replayed")
        res["graph_vs_eager"] = (y_graph.cpu(), y_local.cpu())
    if rank == 0:
        torch.save(res, out_path)
    if graph:
        # as in bench.py: the communicator's teardown can block after graph-captured collectives, so a one-rank run leaves
        # without it once its GPU work is drained
        torch.cuda.synchronize()
        _stage("leaving")
        os._exit(0)
    dist.barrier()
    dist.destroy_process_group()


def _spawn(tmp_path, world, mode, dim, heads, graph=False):
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    out = str(tmp_path / "sp.pt")
    mp.spawn(_worker, args=(world, port, out, mode, dim, heads, graph), nprocs=world, join=True)
    return torch.load(out)


@pytest.mark.parametrize("mode", ["allgather", "ulysses"])
def test_hooks_in_a_one_rank_group_match_single_gpu_and_replay_in_a_graph(cuda, tmp_path, mode):
    """At world 1 the all-gather mode still runs the INT8-K exchange: quant_k_seq into the padded send slab and the attention
    over sequence-major K."""
    res = _spawn(tmp_path, 1, mode, 256, 2, graph=True)
    assert res["int8"] == (mode == "allgather")
    _within_dist_bound(res["y"], res["ref"])
    _within_dist_bound(*res["graph_vs_eager"])


@pytest.mark.parametrize("mode,dim,heads", [("allgather", 256, 2), ("ulysses", 256, 2), ("allgather", 384, 3),
                                            ("ulysses", 384, 3)])     # 3 heads over 2 ranks: the uneven head split
def test_two_gpu_hooks_on_hopper_blocks_match_single_gpu(tmp_path, mode, dim, heads):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    res = _spawn(tmp_path, 2, mode, dim, heads)
    assert res["int8"] == (mode == "allgather")
    _within_dist_bound(res["y"], res["ref"])
