"""Compare the two SageSLA block families on one GPU: BLKQ=128 / BLKK=64 (the Sage2++ family, served as "sm100") and
BLKQ=64 / BLKK=128 (SpargeAttn's Hopper family, served as "sm90").

    python tools/sla_block_families.py [--shape A|B|both] [--iters 50] [--warmup 10] [--topk 0.1]

Both families run in the same process and are timed with CUDA events, call by call, in an order that rotates every
iteration (so no timing always follows the same predecessor): the whole SageSparseLinearAttention forward, the fused
attention launch alone (on that family's own prep, LUT and moments), and the work the forward does before the attention
(prep: quantisation, block map, moments, projection); forward ~ prep + attention is a consistency check of the run.  The SM
clock and the active throttle reasons are read before and after each shape's timed window.
Reported per family: median times, the attention's TFLOP/s with FLOPs = H*Mblk*topk*4*BLKQ*BLKK*D (the count bench.py uses;
BLKQ*BLKK = 8192 in both families), and the fraction of keys each query attends to (topk*BLKK/L).  One JSON line per
(shape, family), preceded by one line with the device name and power limit read in the same run.

    python tools/sla_block_families.py --ranks 1,2,4,8 [--shape ...]

times instead, for each world size N, rank 0's share of one sequence-parallel attention layer (dist.py) on this one GPU, both
families in the same rotating order: in the all-gather mode its own key prep (128-row partial sums, key mean, INT8 and
pooling of its rows), its Q prep and block map and the fused attention of its query rows over the whole gathered slab
("allgather"; the fused attention alone is "allgather_attn"); in the Ulysses mode the single-GPU pipeline on its H/N heads
(rank 0 takes the extra head of an uneven split).  The collectives and their overlap with compute are not timed.  One JSON
line per (shape, N, family).
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SHAPES = {"A": (32760, 12, 128), "B": (75600, 40, 128)}   # (L, heads, head dim): Wan2.1-1.3B and Wan2.1-14B at 480p / 720p
FAMILIES = ("sm100", "sm90")


def device_info():
    name = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError) as e:
        power = f"unavailable ({e})"
    return {"device": name, "power_limit_and_max_sm_clock": power}


def clock_state():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks_throttle_reasons.active", "--format=csv,noheader",
                               "-i", "0"], capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError) as e:
        return f"unavailable ({e})"


def _timed(fn):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end)


def _module(d, ratio, device):
    from turbodiffusion_b200.SLA import SageSparseLinearAttention
    mod = SageSparseLinearAttention(d, ratio).to(device)
    with torch.no_grad():
        mod.proj_l.weight.normal_(0, 0.05)
        mod.proj_l.bias.normal_(0, 0.05)
    return mod


def setup(arch, q, k, v, ratio):
    """The module and one family's attention inputs, built by the same calls its forward makes."""
    from turbodiffusion_b200.SLA.core import attn_fwd, linear_moments, project_moments
    from turbodiffusion_b200.SLA.utils import block_map_from_pools, quant_qk, set_served_arch
    set_served_arch(arch)
    d = q.shape[-1]
    mod = _module(d, ratio, q.device)
    blkq, blkk = mod.block_sizes(q.device.index)
    prep = quant_qk(q, k, blkq=blkq, blkk=blkk)
    topk = max(1, min(prep.nblk, int(ratio * prep.nblk)))
    _, lut = block_map_from_pools(prep.q_pool, prep.k_pool, topk)
    kv, ksum = linear_moments(k, v)
    kvw = project_moments(mod.proj_l.weight, kv, q.dtype)
    pb = mod.proj_l.bias.float().contiguous()

    def attn():
        attn_fwd(prep, v, q, lut, topk, kvw, ksum, pb, d ** -0.5, blkq=blkq, blkk=blkk)

    def forward():
        mod(q, k, v)

    def prep_only():   # what forward() runs before the fused attention
        p = quant_qk(q, k, blkq=blkq, blkk=blkk)
        block_map_from_pools(p.q_pool, p.k_pool, topk)
        project_moments(mod.proj_l.weight, linear_moments(k, v)[0], q.dtype)

    return {"blkq": blkq, "blkk": blkk, "mblk": prep.mblk, "topk": topk, "attn": attn, "forward": forward, "prep": prep_only}


def run_shape(name, ratio, iters, warmup):
    from turbodiffusion_b200.SLA.utils import set_served_arch
    l, h, d = SHAPES[name]
    g = torch.Generator(device="cuda").manual_seed(0)
    q, k, v = (torch.randn(1, l, h, d, generator=g, device="cuda").bfloat16() for _ in range(3))
    k += torch.randn(1, 1, h, d, generator=g, device="cuda").bfloat16() * 2
    prev = set_served_arch("sm100")
    try:
        fams = {arch: setup(arch, q, k, v, ratio) for arch in FAMILIES}
        kinds = ("attn", "forward", "prep")
        times = {arch: {what: [] for what in kinds} for arch in FAMILIES}
        calls = [(arch, what) for arch in FAMILIES for what in kinds]
        clocks = {}
        for i in range(warmup + iters):
            if i == warmup:
                clocks["sm_clock_throttle_before"] = clock_state()
            r = i % len(calls)
            for arch, what in calls[r:] + calls[:r]:
                set_served_arch(arch)
                t = _timed(fams[arch][what])
                if i >= warmup:
                    times[arch][what].append(t)
        clocks["sm_clock_throttle_after"] = clock_state()
    finally:
        set_served_arch(prev)
    rows = []
    for arch in FAMILIES:
        f = fams[arch]
        attn_ms = statistics.median(times[arch]["attn"])
        flops = h * f["mblk"] * f["topk"] * 4 * f["blkq"] * f["blkk"] * d
        rows.append({"shape": name, "L": l, "heads": h, "head_dim": d, "family": arch, "blkq": f["blkq"], "blkk": f["blkk"],
                     "topk": f["topk"], "keys_per_query": round(f["topk"] * f["blkk"] / l, 4),
                     "attn_ms_median": round(attn_ms, 4), "attn_tflops": round(flops / attn_ms / 1e9, 1),
                     "forward_ms_median": round(statistics.median(times[arch]["forward"]), 4),
                     "prep_ms_median": round(statistics.median(times[arch]["prep"]), 4), "calls": iters, **clocks})
    base, hop = rows
    hop["attn_tflops_vs_sm100"] = round(hop["attn_tflops"] / base["attn_tflops"], 3)
    return rows


def setup_rank0(arch, q, k, v, ratio, world):
    """Rank 0's share of one sequence-parallel layer on `world` GPUs (dist.py), on one family's blocks, built from the real
    per-rank primitives.  The gathered slab rank 0 attends over is made here from the whole sequence; the split key prep
    reproduces it bit for bit (tests/test_gpu_sp_hopper_blocks.py)."""
    from turbodiffusion_b200.dist import GpuPrimitives, UlyssesGpuPrims, shard_rows, split_heads
    from turbodiffusion_b200.SLA.core import attn_fwd, linear_moments, project_moments
    from turbodiffusion_b200.SLA.utils import block_map_from_pools, kmean_from_partials, kmean_partials, quant_k_seq, set_served_arch
    set_served_arch(arch)
    _, l, h, d = q.shape
    mod = _module(d, ratio, q.device)
    gp, up = GpuPrimitives(mod, arch), UlyssesGpuPrims(mod, arch)
    blkq, blkk = gp.blkq, gp.blkk
    begin, end, rows_pad = shard_rows(l, world, 0)
    q0, k0 = q[:, begin:end].contiguous(), k[:, begin:end].contiguous()
    partials = kmean_partials(k)                               # every rank's partials, as gathered
    kmean = kmean_from_partials(partials, l)
    k8 = torch.zeros(1, world * rows_pad, h, d, dtype=torch.int8, device=q.device)
    _, k_scale, k_pool = quant_k_seq(k, kmean, k8[:, :l], blkk=blkk)
    v_full = torch.zeros(1, world * rows_pad, h, d, dtype=v.dtype, device=v.device)
    v_full[:, :l] = v
    kv, ksum = linear_moments(k, v)
    pb = mod.proj_l.bias.float().contiguous()

    def allgather():     # own key prep (partials, mean, INT8 + pooling of its rows), Q prep + block map, fused attention
        gp.k_partials(k0)
        gp.k_quant(k0, gp.k_mean(partials, l))
        gp.attention_i8(q0, gp.prepare_q(q0), k8, k_scale, k_pool, kmean, v_full, l, kv, ksum)

    prep = gp.prepare_q(q0)
    prep.kmean, prep.k_i8, prep.k_scale, prep.k_pool, prep.nblk, prep.k_seq_major = kmean, k8, k_scale, k_pool, k_scale.shape[-1], True
    topk = min(prep.nblk, int(ratio * prep.nblk))
    _, lut = block_map_from_pools(prep.q_pool, prep.k_pool, topk)
    kvw = project_moments(mod.proj_l.weight, kv, q.dtype)

    def allgather_attn():
        attn_fwd(prep, v_full, q0, lut, topk, kvw, ksum, pb, d ** -0.5, lk=l, blkq=blkq, blkk=blkk)

    hl = split_heads(h, world)[0][0]                           # rank 0 holds the most heads
    qh, kh, vh = (t[:, :, :hl].contiguous() for t in (q, k, v))

    def ulysses():       # the single-GPU pipeline on rank 0's heads of the whole sequence
        up.attend(lambda: qh, lambda: kh, lambda: vh)

    return {"blkq": blkq, "blkk": blkk, "rows": end - begin, "heads": hl, "mblk": prep.mblk, "topk": topk,
            "allgather": allgather, "allgather_attn": allgather_attn, "ulysses": ulysses}


def run_ranks(name, ratio, iters, warmup, ranks):
    """Rank 0's share per family for each world size; collectives are not timed."""
    from turbodiffusion_b200.SLA.utils import set_served_arch
    l, h, d = SHAPES[name]
    g = torch.Generator(device="cuda").manual_seed(0)
    q, k, v = (torch.randn(1, l, h, d, generator=g, device="cuda").bfloat16() for _ in range(3))
    k += torch.randn(1, 1, h, d, generator=g, device="cuda").bfloat16() * 2
    rows = []
    prev = set_served_arch("sm100")
    try:
        for world in ranks:
            fams = {arch: setup_rank0(arch, q, k, v, ratio, world) for arch in FAMILIES}
            kinds = ("allgather", "allgather_attn", "ulysses")
            times = {arch: {what: [] for what in kinds} for arch in FAMILIES}
            calls = [(arch, what) for arch in FAMILIES for what in kinds]
            clocks = {}
            for i in range(warmup + iters):
                if i == warmup:
                    clocks["sm_clock_throttle_before"] = clock_state()
                r = i % len(calls)
                for arch, what in calls[r:] + calls[:r]:
                    set_served_arch(arch)
                    t = _timed(fams[arch][what])
                    if i >= warmup:
                        times[arch][what].append(t)
            clocks["sm_clock_throttle_after"] = clock_state()
            out = []
            for arch in FAMILIES:
                f = fams[arch]
                med = {what: statistics.median(times[arch][what]) for what in kinds}
                flops = h * f["mblk"] * f["topk"] * 4 * f["blkq"] * f["blkk"] * d
                out.append({"shape": name, "L": l, "heads": h, "head_dim": d, "world": world, "family": arch,
                            "blkq": f["blkq"], "blkk": f["blkk"], "rank0_rows": f["rows"], "rank0_query_blocks": f["mblk"],
                            "rank0_ulysses_heads": f["heads"], "topk": f["topk"],
                            "allgather_ms_median": round(med["allgather"], 4),
                            "allgather_attn_ms_median": round(med["allgather_attn"], 4),
                            "allgather_attn_tflops": round(flops / med["allgather_attn"] / 1e9, 1),
                            "ulysses_ms_median": round(med["ulysses"], 4), "calls": iters, **clocks})
            base, hop = out
            for what in kinds:
                hop[f"{what}_speedup_vs_sm100"] = round(base[f"{what}_ms_median"] / hop[f"{what}_ms_median"], 3)
            rows += out
            del fams
            torch.cuda.empty_cache()
    finally:
        set_served_arch(prev)
    return rows


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--shape", default="both", choices=["A", "B", "both"])
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--topk", type=float, default=0.1)
    ap.add_argument("--ranks", default=None,
                    help="comma-separated world sizes, e.g. 1,2,4,8: time rank 0's share of a sequence-parallel layer instead")
    args = ap.parse_args()
    ranks = None
    if args.ranks is not None:
        ranks = [int(n) for n in args.ranks.split(",")]
        if not ranks or min(ranks) < 1:
            raise SystemExit("--ranks: positive world sizes, e.g. 1,2,4,8")
    if not torch.cuda.is_available():
        raise SystemExit("sla_block_families.py measures on a CUDA device; none is available")
    if args.iters < 50:
        raise SystemExit("--iters: the medians are taken over at least 50 calls")
    print(json.dumps(device_info()), flush=True)
    for name in (["A", "B"] if args.shape == "both" else [args.shape]):
        rows = run_shape(name, args.topk, args.iters, args.warmup) if ranks is None else \
            run_ranks(name, args.topk, args.iters, args.warmup, ranks)
        for row in rows:
            print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
