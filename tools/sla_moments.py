"""Time the linear-attention moments kernel (tdb200_sla_linear_moments: kv = phi(K)^T V and ksum = sum phi(K), bf16, softmax
feature map) per call with torch.profiler, optionally against a second build of the library.

    python tools/sla_moments.py [--baseline-lib PATH] [--rounds 6] [--calls 30]

Shapes: A (L = 32760, 12 x 128), B (L = 75600, 40 x 128), the Ulysses-rank slices of each (2 heads of A: 12 heads on 8 ranks;
5 heads of B: 40 heads on 8 ranks) and the 24 x 64 configuration (L = 32760, 24 heads of 64, run as 12 head pairs).
Each round profiles --calls launches per shape and build; the builds alternate, and their order flips every round, so that
neither build always runs first.  A call is the C entry point on a zeroed buffer; only the moments kernel's device time is
counted.  `--baseline-lib` is another libtdb200.so with the same C ABI (for example the parent commit's build): it is loaded
next to this tree's library and called through the same arguments.  Printed: one JSON line with the device name and power
limit read in this run, then one line per shape with each build's per-round mean kernel time (us) and its median, the
achieved HBM bandwidth of the K and V reads, and the SM clock / throttle reasons around the timed window.
"""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from sla_block_families import clock_state, device_info  # noqa: E402

SHAPES = {   # name: (L, heads, head dim)
    "A": (32760, 12, 128),
    "A_ulysses8_rank0": (32760, 2, 128),
    "B": (75600, 40, 128),
    "B_ulysses8_rank0": (75600, 5, 128),
    "24x64": (32760, 24, 64),
}


def _load(path):
    from turbodiffusion_b200 import _lib
    handle = ctypes.CDLL(path)
    fn = handle.tdb200_sla_linear_moments
    fn.argtypes = _lib._PROTOS["tdb200_sla_linear_moments"]
    fn.restype = ctypes.c_int
    return fn


def _launcher(fn, k, v):
    from turbodiffusion_b200._lib import DTYPE_TAG, ptr
    b, l, h, d = k.shape
    buf = torch.zeros(b * h * d * (d + 1), dtype=torch.float32, device=k.device)
    stream = torch.cuda.current_stream().cuda_stream

    def call():
        buf.zero_()
        rc = fn(ptr(k), ptr(v), DTYPE_TAG[k.dtype], b, l, h, d, 0, ptr(buf), ptr(buf) + 4 * b * h * d * d, stream)
        if rc != 0:
            raise RuntimeError(f"tdb200_sla_linear_moments returned {rc}")
    return call, buf


def _kernel_us(call, calls):
    """Mean device time (us) of the moments kernels the trace of `calls` launches holds, and how many it holds (the
    profiler can drop records of a long window)."""
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            call()
        torch.cuda.synchronize()
    total, count = 0.0, 0
    for ev in prof.key_averages():
        if "sla_moments_kernel" in ev.key:
            total += ev.device_time_total
            count += ev.count
    if count == 0:
        raise RuntimeError("no moments kernel in the trace")
    return total / count, count


def run_shape(name, builds, rounds, calls):
    l, h, d = SHAPES[name]
    g = torch.Generator(device="cuda").manual_seed(0)
    k = torch.randn(1, l, h, d, generator=g, device="cuda").bfloat16()
    v = torch.randn(1, l, h, d, generator=g, device="cuda").bfloat16()
    launch = {b: _launcher(fn, k, v) for b, fn in builds.items()}
    for call, _ in launch.values():   # warm-up: module load, first-launch attribute setting
        for _ in range(5):
            call()
    torch.cuda.synchronize()
    names = list(builds)
    times = {b: [] for b in names}
    traced = {b: 0 for b in names}
    before = clock_state()
    for r in range(rounds):
        for b in (names if r % 2 == 0 else names[::-1]):
            us, n = _kernel_us(launch[b][0], calls)
            times[b].append(round(us, 2))
            traced[b] += n
    after = clock_state()
    row = {"shape": name, "L": l, "heads": h, "head_dim": d, "tiles": -(-l // 128), "calls_per_round": calls,
           "sm_clock_throttle_before": before, "sm_clock_throttle_after": after}
    hbm_bytes = 2 * l * h * d * 2                         # K and V, 16-bit, each read once
    for b in names:
        med = statistics.median(times[b])
        row[b] = {"us_per_round": times[b], "us_median": med, "hbm_gbs": round(hbm_bytes / med / 1e3, 1),
                  "kernels_traced": traced[b]}
    if len(names) == 2:
        row["median_ratio_" + names[0] + "_over_" + names[1]] = round(row[names[0]]["us_median"] / row[names[1]]["us_median"], 3)
        # the two builds' kv and ksum, for information: equal only up to the fp32 summation order
        out0, out1 = (launch[b][1] for b in names)
        row["rel_l2_between_builds"] = float(((out0 - out1).norm() / out1.norm()).item())
    del launch, k, v
    torch.cuda.empty_cache()
    return row


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--baseline-lib", default=None, help="another libtdb200.so with the same C ABI, timed alternately")
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--calls", type=int, default=30)
    ap.add_argument("--shape", default="all", choices=["all"] + list(SHAPES))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sla_moments.py measures on a CUDA device; none is available")
    from turbodiffusion_b200 import _lib
    builds = {"this": _load(_lib.LIB_PATH)}
    if args.baseline_lib:
        builds["baseline"] = _load(os.path.abspath(args.baseline_lib))
    print(json.dumps({**device_info(), "builds": {"this": _lib.LIB_PATH, "baseline": args.baseline_lib}}), flush=True)
    for name in (SHAPES if args.shape == "all" else [args.shape]):
        print(json.dumps(run_shape(name, builds, args.rounds, args.calls)), flush=True)


if __name__ == "__main__":
    main()
