"""Time the dense attention JVP operator (ops.dense_attention_jvp, the dense_attn_jvp_kernel) on one GPU, bf16 (or fp16 with
--dtype fp16), against the dense forward and the cheapest torch JVP that runs, at the shapes the models run attention at.

    python tools/dense_attention_jvp.py [--iters 60] [--warmup 10] [--only NAME] [--dtype bf16|fp16] [--out-dir DIR]

Shapes (queries x keys, heads x head dim):
  A-cross   32760 x 512,   12 x 128   Wan2.1-1.3B at 480p, cross-attention over the text tokens
  A-self    32760 x 32760, 12 x 128   dense self-attention at shape A
  B-cross   75600 x 512,   40 x 128   Wan2.1-14B at 720p, cross-attention
  C-512     28672 x 512,   32 x 128   LTX shape C's video stream, text keys padded
Legs: the JVP operator (output and tangent); ops.dense_attention and F.scaled_dot_product_attention (fed the transposed views
block.py feeds it), the forward alone, for scale; torch.func.jvp of an explicit-softmax attention in bf16, which torch's fused
SDPA kernels cannot give (they have no forward-AD formula).  That leg materialises the score matrix, its tangent, P and P's
tangent in bf16: where those four need more than the free device memory it is not run, and the row says so.
Per shape, in one process: every leg warmed up, then --iters rounds of one CUDA-event-timed call of each leg, alternating;
median, minimum, maximum and the 10th / 90th percentiles per leg.  TFLOP/s count 12 * B * H * Lq * Lk * D for the JVP legs
and 4 * B * H * Lq * Lk * D for the forward legs, with the share of the H100 SXM data sheet's 989 TFLOP/s (dense bf16, a 700 W
figure, not a rate reached here).  The rel-L2 distance between the two JVP legs' tangents is printed where both run.  Which
kernels each leg launches, and their times, come from a torch.profiler pass of its own after the timed window (three calls
per leg; traces go to --out-dir).  One JSON line with the device name, power limit and maximum SM clock, then one per shape
with the SM clock and throttle reasons read before and after its timed window.
There is no CPU timing: without a CUDA device the script exits with an error."""
from __future__ import annotations

import argparse
import json
import os
import sys
import tempfile

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from dense_attention import _kernels, _spread  # noqa: E402
from sla_block_families import _timed, clock_state, device_info  # noqa: E402

D = 128
SHAPES = {"A-cross": (32760, 512, 12), "A-self": (32760, 32760, 12), "B-cross": (75600, 512, 40), "C-512": (28672, 512, 32)}


def _attn(q, k, v, sm_scale):
    """explicit-softmax attention of [B, L, H, D] tensors"""
    s = (q.transpose(1, 2) @ k.transpose(1, 2).transpose(-1, -2)) * sm_scale
    return (torch.softmax(s, -1) @ v.transpose(1, 2)).transpose(1, 2)


def run_shape(name, iters, warmup, out_dir, dtype="bf16"):
    from turbodiffusion_b200 import ops
    lq, lk, h = SHAPES[name]
    g = torch.Generator(device="cuda").manual_seed(0)
    dt = {"bf16": torch.bfloat16, "fp16": torch.float16}[dtype]
    q, q_t = (torch.randn(1, lq, h, D, device="cuda", generator=g).to(dt) for _ in range(2))
    k, v, k_t, v_t = (torch.randn(1, lk, h, D, device="cuda", generator=g).to(dt) for _ in range(4))
    sm_scale = D ** -0.5
    legs = {"dense_attention_jvp": lambda: ops.dense_attention_jvp(q, k, v, q_t, k_t, v_t, sm_scale),
            "dense_attention": lambda: ops.dense_attention(q, k, v, sm_scale),
            "sdpa": lambda: F.scaled_dot_product_attention(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2),
                                                           scale=sm_scale).transpose(1, 2)}
    torch.cuda.empty_cache()
    score_bytes = 4 * h * lq * lk * 2
    free = torch.cuda.mem_get_info()[0]
    row = {"shape": name, "Lq": lq, "Lk": lk, "heads": h, "head_dim": D, "dtype": dtype}
    if score_bytes < 0.8 * free:
        legs["torch_func_jvp"] = lambda: torch.func.jvp(lambda a, b, c: _attn(a, b, c, sm_scale), (q, k, v), (q_t, k_t, v_t))
    else:
        row["torch_func_jvp"] = (f"not run: S, S_t, P and P_t in bf16 need {score_bytes / 2**30:.1f} GiB, "
                                 f"{free / 2**30:.1f} GiB free")
    for _ in range(warmup):
        for fn in legs.values():
            fn()
    if "torch_func_jvp" in legs:
        ours, lib_t = legs["dense_attention_jvp"]()[1].double(), legs["torch_func_jvp"]()[1].double()
        row["rel_l2_between_the_jvp_tangents"] = float(f"{((ours - lib_t).norm() / lib_t.norm()).item():.3e}")
        del ours, lib_t
    torch.cuda.synchronize()
    flop = {n: (12 if "jvp" in n else 4) * h * lq * lk * D for n in legs}
    row["sm_clock_throttle_before"] = clock_state()
    times = {n: [] for n in legs}
    for _ in range(iters):
        for n, fn in legs.items():
            times[n].append(_timed(fn))
    row["sm_clock_throttle_after"] = clock_state()
    for n in legs:
        row[n] = {"flop": flop[n], **_spread(times[n], flop[n])}
    for n, fn in legs.items():
        row[n]["kernels_ms_per_call"] = _kernels(fn, 3, os.path.join(out_dir, f"{name}_{n}.trace.json"))
    row["calls_per_leg"] = iters
    return row


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--iters", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--only", choices=tuple(SHAPES), default=None)
    ap.add_argument("--dtype", choices=("bf16", "fp16"), default="bf16")
    ap.add_argument("--out-dir", default=None, help="where the profiler traces go (default: a new temporary directory)")
    args = ap.parse_args()
    if args.iters < 50:
        ap.error("--iters: at least 50 timed calls per leg")
    if not torch.cuda.is_available():
        raise SystemExit("dense_attention_jvp.py measures on the GPU; no CUDA device found")
    out_dir = args.out_dir or tempfile.mkdtemp(prefix="dense_attention_jvp_")
    os.makedirs(out_dir, exist_ok=True)
    print(json.dumps({**device_info(), "torch": torch.__version__, "traces": out_dir}), flush=True)
    for name in ((args.only,) if args.only else SHAPES):
        print(json.dumps(run_shape(name, args.iters, args.warmup, out_dir, args.dtype)), flush=True)


if __name__ == "__main__":
    main()
