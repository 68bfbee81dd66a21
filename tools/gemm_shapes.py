"""Time the W8A8 GEMMs of one Wan DiT block at shapes A and B through the entry points block.py uses.

    python tools/gemm_shapes.py [--shape A|B|both] [--iters 100] [--warmup 10]

Per shape, one row per GEMM of a block (q/k/v as one split GEMM, o, cross q, cross o, cross k/v, FFN up with GELU and the
quantised output, FFN down): the median of --iters launches, each timed with CUDA events after --warmup launches of every
GEMM (the split and quantised-output entry points allocate their outputs from torch's caching allocator inside the
timed window, as block.py does), its TOPS (2 m n k / time) and the fraction of the H100 SXM data-sheet dense INT8 rate (1979 TOPS; a data-sheet
figure for a card allowed 700 W).  Then the block's GEMM total and the step's (times the layer count).  The library is
whatever turbodiffusion_b200._lib loads, so TDB200_LIB selects a build to time; its path is printed with the device name,
power limit and maximum SM clock, and the SM clock and throttle reasons are read before and after each shape.  One JSON line
per item.
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
from sla_block_families import _timed, clock_state, device_info  # noqa: E402

INT8_PEAK_TOPS = 1979.0
# name: (L, dim, ffn, layers, text tokens) as in bench.py
SHAPES = {"A": (32760, 1536, 8960, 30, 512), "B": (75600, 5120, 13824, 40, 512)}


def gemms(shape):
    """(name, m, n, k, entry point, parts) of one block"""
    l, dim, ffn, _, text = SHAPES[shape]
    return [("qkv", l, 3 * dim, dim, "split", 3), ("o", l, dim, dim, "bias", 1), ("cross_q", l, dim, dim, "bias", 1),
            ("cross_o", l, dim, dim, "bias", 1), ("cross_kv", text, 2 * dim, dim, "split", 2),
            ("ffn_up", l, ffn, dim, "quant_gelu", 1), ("ffn_down", l, dim, ffn, "bias", 1)]


def make_call(m, n, k, kind, parts, dev, g):
    from turbodiffusion_b200.turbo_diffusion_ops import gemm_cuda_quant_out, gemm_cuda_split, gemm_cuda_swizzle_bias
    a = torch.randint(-128, 128, (m, k), device=dev, dtype=torch.int8, generator=g)
    b = torch.randint(-128, 128, (n, k), device=dev, dtype=torch.int8, generator=g)
    a_s = torch.rand((m + 127) // 128, k // 128, device=dev, generator=g) * 1e-3
    b_s = torch.rand((n + 127) // 128, k // 128, device=dev, generator=g) * 1e-3
    bias = torch.randn(n, device=dev, generator=g).bfloat16()
    if kind == "split":
        return lambda: gemm_cuda_split(a, a_s, b, b_s, bias, torch.bfloat16, parts)
    if kind == "quant_gelu":
        return lambda: gemm_cuda_quant_out(a, a_s, b, b_s, bias, torch.bfloat16, gelu=True)
    c = torch.empty(m, n, device=dev, dtype=torch.bfloat16)
    return lambda: gemm_cuda_swizzle_bias(a, a_s, b, b_s, c, bias)


def run_shape(shape, iters, warmup):
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(0)
    rows = [(name, m, n, k, make_call(m, n, k, kind, parts, dev, g)) for name, m, n, k, kind, parts in gemms(shape)]
    for _ in range(warmup):
        for *_, fn in rows:
            fn()
    torch.cuda.synchronize()
    before = clock_state()
    out, total_ms, total_flop = [], 0.0, 0.0
    for name, m, n, k, fn in rows:
        ms = statistics.median(_timed(fn) for _ in range(iters))
        flop = 2.0 * m * n * k
        tops = flop / ms / 1e9
        total_ms += ms
        total_flop += flop
        out.append({"shape": shape, "gemm": name, "m": m, "n": n, "k": k, "ms": round(ms, 4), "tops": round(tops, 1),
                    "frac_int8_peak": round(tops / INT8_PEAK_TOPS, 3)})
    layers = SHAPES[shape][3]
    tops = total_flop / total_ms / 1e9
    out.append({"shape": shape, "block_gemm_ms": round(total_ms, 3), "step_gemm_ms": round(total_ms * layers, 1),
                "tops": round(tops, 1), "frac_int8_peak": round(tops / INT8_PEAK_TOPS, 3), "calls": iters,
                "sm_clock_throttle_before": before, "sm_clock_throttle_after": clock_state()})
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--shape", default="both", choices=("A", "B", "both"))
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gemm_shapes.py measures on the GPU; no CUDA device found")
    from turbodiffusion_b200 import _lib
    print(json.dumps({**device_info(), "library": _lib.LIB_PATH}), flush=True)
    for shape in (("A", "B") if args.shape == "both" else (args.shape,)):
        for row in run_shape(shape, args.iters, args.warmup):
            print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
