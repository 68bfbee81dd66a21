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


def setup(arch, q, k, v, ratio):
    """The module and one family's attention inputs, built by the same calls its forward makes."""
    from turbodiffusion_b200.SLA import SageSparseLinearAttention
    from turbodiffusion_b200.SLA.core import attn_fwd, linear_moments, project_moments
    from turbodiffusion_b200.SLA.utils import block_map_from_pools, quant_qk, set_served_arch
    set_served_arch(arch)
    d = q.shape[-1]
    mod = SageSparseLinearAttention(d, ratio).to(q.device)
    with torch.no_grad():
        mod.proj_l.weight.normal_(0, 0.05)
        mod.proj_l.bias.normal_(0, 0.05)
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


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--shape", default="both", choices=["A", "B", "both"])
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--topk", type=float, default=0.1)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sla_block_families.py measures on a CUDA device; none is available")
    if args.iters < 50:
        raise SystemExit("--iters: the medians are taken over at least 50 calls")
    print(json.dumps(device_info()), flush=True)
    for name in (["A", "B"] if args.shape == "both" else [args.shape]):
        for row in run_shape(name, args.topk, args.iters, args.warmup):
            print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
