"""Time the dense attention operator (ops.dense_attention, the dense_attn_fwd_kernel) against F.scaled_dot_product_attention
on one GPU, bf16, at the shapes the models run it at.

    python tools/dense_attention.py [--iters 60] [--warmup 10] [--only NAME] [--out-dir DIR]

Shapes (queries x keys, heads x head dim):
  A-cross   32760 x 512,   12 x 128   Wan2.1-1.3B at 480p, cross-attention over the text tokens
  B-cross   75600 x 512,   40 x 128   Wan2.1-14B at 720p, cross-attention
  C-512     28672 x 512,   32 x 128   LTX shape C's video stream, text keys padded
  C-226     28672 x 226,   32 x 128   the same with the text trimmed to 226 keys
  A-self    32760 x 32760, 12 x 128   dense self-attention at shape A, the baseline SLA is compared with
Per shape, in one process: both legs warmed up, then --iters rounds of one CUDA-event-timed call of each leg, alternating
(ours, SDPA, ours, SDPA, ...); median, minimum, maximum and the 10th / 90th percentiles per leg.  SDPA is fed the
transposed views block.py feeds it.  Reported per leg: TFLOP/s from 4 * B * H * Lq * Lk * D, that rate as a share of the
H100 SXM data sheet's 989 TFLOP/s (dense bf16, a 700 W figure, not a rate reached here), and the HBM lower bound of the call
(q, k, v read once and out written once at the data sheet's 3.35 TB/s).  The rel-L2 distance between the two outputs is
printed with the times.  Which kernels each leg launches comes from a torch.profiler pass of its own after the timed
window (three calls per leg; the trace goes to --out-dir).  One JSON line with the device name, power limit and maximum SM
clock, then one per shape with the SM clock and throttle reasons read before and after its timed window.
There is no CPU timing: without a CUDA device the script exits with an error."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import tempfile

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from sla_block_families import _timed, clock_state, device_info  # noqa: E402

D = 128
SHAPES = {"A-cross": (32760, 512, 12), "B-cross": (75600, 512, 40), "C-512": (28672, 512, 32), "C-226": (28672, 226, 32),
          "A-self": (32760, 32760, 12)}      # (Lq, Lk, heads)
DATA_SHEET_BF16_TFLOPS, DATA_SHEET_HBM_TBS = 989.0, 3.35


def counts(lq, lk, h):
    """(FLOPs, HBM bytes) the algorithm needs for one call at batch 1, bf16."""
    return 4 * h * lq * lk * D, 2 * (2 * lq + 2 * lk) * h * D


def _spread(ms, flop):
    ms = sorted(ms)
    med = statistics.median(ms)
    pct = lambda f: ms[min(len(ms) - 1, int(f * len(ms)))]
    return {"median_ms": round(med, 4), "min_ms": round(ms[0], 4), "p10_ms": round(pct(0.1), 4), "p90_ms": round(pct(0.9), 4),
            "max_ms": round(ms[-1], 4), "tflops_at_median": round(flop / med / 1e9, 1),
            "share_of_data_sheet_989_tflops": round(flop / med / 1e9 / DATA_SHEET_BF16_TFLOPS, 3)}


def _kernels(fn, calls, trace_path):
    """Device kernels fn launches: name -> mean ms per call, from a profiler pass of its own."""
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    prof.export_chrome_trace(trace_path)
    return {ev.key[:160]: round(ev.device_time_total / 1e3 / calls, 4) for ev in prof.key_averages()
            if ev.device_time_total > 0}


def run_shape(name, iters, warmup, out_dir):
    from turbodiffusion_b200 import ops
    lq, lk, h = SHAPES[name]
    g = torch.Generator(device="cuda").manual_seed(0)
    q = torch.randn(1, lq, h, D, device="cuda", generator=g).bfloat16()
    k, v = (torch.randn(1, lk, h, D, device="cuda", generator=g).bfloat16() for _ in range(2))
    sm_scale = D ** -0.5
    legs = {"dense_attention": lambda: ops.dense_attention(q, k, v, sm_scale),
            "sdpa": lambda: F.scaled_dot_product_attention(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2),
                                                           scale=sm_scale).transpose(1, 2)}
    for _ in range(warmup):
        for fn in legs.values():
            fn()
    ours, lib_out = legs["dense_attention"]().double(), legs["sdpa"]().double()
    rel = ((ours - lib_out).norm() / lib_out.norm()).item()
    del ours, lib_out
    torch.cuda.synchronize()
    flop, nbytes = counts(lq, lk, h)
    row = {"shape": name, "Lq": lq, "Lk": lk, "heads": h, "head_dim": D, "dtype": "bf16", "flop": flop, "hbm_bytes": nbytes,
           "hbm_lower_bound_ms": round(nbytes / (DATA_SHEET_HBM_TBS * 1e12) * 1e3, 4),
           "rel_l2_between_the_outputs": float(f"{rel:.3e}"), "sm_clock_throttle_before": clock_state()}
    times = {n: [] for n in legs}
    for _ in range(iters):
        for n, fn in legs.items():
            times[n].append(_timed(fn))
    row["sm_clock_throttle_after"] = clock_state()
    for n in legs:
        row[n] = _spread(times[n], flop)
    row["sdpa_over_dense_attention_at_medians"] = round(row["sdpa"]["median_ms"] / row["dense_attention"]["median_ms"], 3)
    for n, fn in legs.items():
        row[n]["kernels_ms_per_call"] = _kernels(fn, 3, os.path.join(out_dir, f"{name}_{n}.trace.json"))
    row["calls_per_leg"] = iters
    return row


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--iters", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--only", choices=tuple(SHAPES), default=None)
    ap.add_argument("--out-dir", default=None, help="where the profiler traces go (default: a new temporary directory)")
    args = ap.parse_args()
    if args.iters < 50:
        ap.error("--iters: at least 50 timed calls per leg")
    if not torch.cuda.is_available():
        raise SystemExit("dense_attention.py measures on the GPU; no CUDA device found")
    out_dir = args.out_dir or tempfile.mkdtemp(prefix="dense_attention_")
    os.makedirs(out_dir, exist_ok=True)
    print(json.dumps({**device_info(), "torch": torch.__version__, "traces": out_dir}), flush=True)
    for name in ((args.only,) if args.only else SHAPES):
        print(json.dumps(run_shape(name, args.iters, args.warmup, out_dir)), flush=True)


if __name__ == "__main__":
    main()
