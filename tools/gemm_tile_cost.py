"""Measure what one 128x256 output tile of the W8A8 GEMM costs outside its K loop.

    python tools/gemm_tile_cost.py [--iters 50] [--warmup 5]

At M = 32760 (256 row tiles) and N in {1536, 4608, 8960} the depth is swept over 1, 2, 4, 8, 12, 24, 40 and 70 K-blocks of
128 through the entry points block.py uses: the 16-bit output with bias (gemm_cuda_swizzle_bias) for every N, and the
quantised-output GELU epilogue (gemm_cuda_quant_out, the FFN up GEMM) at N = 8960.  Each point is the median of --iters
launches timed with CUDA events after --warmup launches.  With one CTA per SM an SM works through ceil(tiles / SMs) tiles
one after the other, so

    per-tile time = time / ceil(tiles / SMs)

and a least-squares line  per-tile time = F + c * K-blocks  over the sweep gives F, the time a tile spends outside the
steady K loop (launch, ring fill, epilogue, retirement), and c, the time per K-block.  One JSON line per point and one per
fit, after a line with the device name, power limit, maximum SM clock and the library path (TDB200_LIB selects the build);
the SM clock and throttle reasons are read before and after each sweep.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from gemm_shapes import make_call  # noqa: E402
from sla_block_families import _timed, clock_state, device_info  # noqa: E402

M = 32760
K_BLOCKS = (1, 2, 4, 8, 12, 24, 40, 70)
# (n, entry point as gemm_shapes.make_call names it)
SWEEPS = ((1536, "bias"), (4608, "bias"), (8960, "bias"), (8960, "quant_gelu"))


def fit_line(xs, ys):
    """least-squares (intercept, slope) of ys over xs"""
    mx, my = statistics.fmean(xs), statistics.fmean(ys)
    slope = sum((x - mx) * (y - my) for x, y in zip(xs, ys)) / sum((x - mx) ** 2 for x in xs)
    return my - slope * mx, slope


def run_sweep(n, kind, iters, warmup, sms):
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(0)
    tiles = ((M + 127) // 128) * ((n + 255) // 256)
    waves = -(-tiles // sms)
    before = clock_state()
    rows = []
    for kb in K_BLOCKS:
        fn = make_call(M, n, 128 * kb, kind, 1, dev, g)
        for _ in range(warmup):
            fn()
        torch.cuda.synchronize()
        ms = statistics.median(_timed(fn) for _ in range(iters))
        rows.append({"n": n, "epilogue": kind, "k_blocks": kb, "tiles": tiles, "tiles_per_sm": waves, "ms": round(ms, 4),
                     "per_tile_us": round(1e3 * ms / waves, 3)})
        del fn
        torch.cuda.empty_cache()
    f, c = fit_line([r["k_blocks"] for r in rows], [r["per_tile_us"] for r in rows])
    rows.append({"n": n, "epilogue": kind, "fit_F_us": round(f, 3), "fit_c_us_per_k_block": round(c, 4), "calls": iters,
                 "sm_clock_throttle_before": before, "sm_clock_throttle_after": clock_state()})
    return rows


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gemm_tile_cost.py measures on the GPU; no CUDA device found")
    from turbodiffusion_b200 import _lib
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    print(json.dumps({**device_info(), "sms": sms, "library": _lib.LIB_PATH}), flush=True)
    for n, kind in SWEEPS:
        for row in run_sweep(n, kind, args.iters, args.warmup, sms):
            print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
