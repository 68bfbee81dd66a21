"""Time SparseLinearAttention (16-bit Q.K^T) at its two served block geometries, (BLKQ, BLKK) = (128, 64) and the
constructor's default (64, 64), on one GPU.

    python tools/sla_q64_16bit.py [--shape A|B|both] [--topk 0.1] [--iters 20] [--warmup 5] [--dtype bf16|fp16]

Per shape and geometry, in one run, geometries alternated call by call, CUDA events, medians over --iters calls:
  * the module's inference forward (no grad: block selection, linear moments, fused attention) and its block-selection prep
    alone (pooled means + top-k: quant_qk at (128, 64); the query and key halves of the prepass at (64, 64));
  * the training forward (grad-requiring inputs) and the module backward (loss = sum(out * g));
  * each sparse-attention kernel of the inference forward, the training forward and the backward, from a torch.profiler pass
    of its own (mean device time per launch).
FLOPs (Mblk = ceil(L / BLKQ), topk = int(r * ceil(L / BLKK))): F = H * Mblk * topk * 4 * BLKQ * BLKK * D for a forward; the dQ
kernel executes 1.5 F (S, dP, dQ), the dK/dV kernel 2.0 F (S, dP, dV, dK).  One JSON line with the device name and power
limit, then one per shape; the SM clock and throttle reasons are read before and after each shape's timed window.  --dtype
(bf16 by default) is the type of q, k, v, the module and its output.
"""
from __future__ import annotations

import argparse
import json
import os
import re
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from sla_backward import _median_ms  # noqa: E402
from sla_block_families import DTYPES, SHAPES, clock_state, device_info  # noqa: E402

GEOMETRIES = ((128, 64), (64, 64))


def _kernel_times(fn, iters):
    """Mean device ms per call of every sla_ kernel fn launches."""
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        m = re.search(r"(sla_\w+)(?:<([^>]*)>)?", ev.key)
        if m and ev.device_time_total > 0:
            lse = m.group(1).startswith("sla_attn_fwd") and (m.group(2) or "").replace(" ", "").endswith("true")
            key = m.group(1) + ("<lse>" if lse else "")
            out[key] = round(out.get(key, 0.0) + ev.device_time_total / 1e3 / iters, 3)
    return out


def run_shape(name, topk_ratio, iters, warmup, dtype):
    from turbodiffusion_b200.SLA import SparseLinearAttention
    from turbodiffusion_b200.SLA.core import block_map_from_pools, select_prep
    l, h, d = SHAPES[name]
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(0)
    q, k, v = (torch.randn(1, l, h, d, device=dev, generator=g, dtype=dtype) for _ in range(3))
    gout = torch.randn(q.shape, device=dev, generator=g, dtype=dtype)
    qg, kg, vg = (t.clone().requires_grad_() for t in (q, k, v))
    legs = {}
    for blkq, blkk in GEOMETRIES:
        mod = SparseLinearAttention(d, topk_ratio, BLKQ=blkq, BLKK=blkk, use_bf16=dtype == torch.bfloat16).to(dev)
        _, sel = mod.forward_with_lut(q, k, v)
        topk = sel["topk"]
        state = {}

        def infer(mod=mod):
            with torch.no_grad():
                mod(q, k, v)

        def prep(blkq=blkq, blkk=blkk, topk=topk):
            p = select_prep(q, k, blkq, blkk)
            block_map_from_pools(p.q_pool, p.k_pool, topk)

        def train_fwd(mod=mod, state=state):
            state["out"] = mod(qg, kg, vg)

        def train_bwd(state=state):
            state["out"].backward(gout)

        legs[(blkq, blkk)] = dict(topk=topk, infer=infer, prep=prep, train_fwd=train_fwd, train_bwd=train_bwd,
                                  times={n: [] for n in ("infer", "prep", "train_fwd", "train_bwd")})
    for _ in range(warmup):
        for leg in legs.values():
            leg["infer"](), leg["prep"](), leg["train_fwd"](), leg["train_bwd"]()
    torch.cuda.synchronize()
    row = {"shape": name, "L": l, "heads": h, "head_dim": d, "dtype": str(dtype)[6:], "topk_ratio": topk_ratio, "sm_clock_throttle_before": clock_state()}
    for _ in range(iters):
        for leg in legs.values():
            for n in ("infer", "prep", "train_fwd", "train_bwd"):
                leg["times"][n].append(_median_ms(leg[n], 1))
    row["sm_clock_throttle_after"] = clock_state()
    med = statistics.median
    for (blkq, blkk), leg in legs.items():
        topk = leg["topk"]
        f = h * ((l + blkq - 1) // blkq) * topk * 4 * blkq * blkk * d
        kernels = _kernel_times(leg["infer"], iters)
        kernels.update(_kernel_times(lambda: (leg["train_fwd"](), leg["train_bwd"]()), iters))
        t = {n: med(x) for n, x in leg["times"].items()}
        out = {"topk_blocks": topk, "fwd_flop": f,
               "module_infer_ms": round(t["infer"], 3), "prep_ms": round(t["prep"], 3),
               "prep_share_of_infer": round(t["prep"] / t["infer"], 3),
               "train_fwd_ms": round(t["train_fwd"], 3), "module_bwd_ms": round(t["train_bwd"], 3), "kernel_ms": kernels}
        fused = [ms for kname, ms in kernels.items() if kname.startswith("sla_attn_fwd") and not kname.endswith("<lse>")]
        lse_k = [ms for kname, ms in kernels.items() if kname.endswith("<lse>")]
        dq = [ms for kname, ms in kernels.items() if kname.startswith("sla_bwd_dq")]
        dkdv = [ms for kname, ms in kernels.items() if kname.startswith("sla_bwd_dkdv")]
        if fused:
            out["fused_fwd_kernel_tflops"] = round(f / fused[0] / 1e9, 1)
        if lse_k:
            out["lse_fwd_kernel_tflops"] = round(f / lse_k[0] / 1e9, 1)
        if dq:
            out["dq_kernel_tflops_executed"] = round(1.5 * f / dq[0] / 1e9, 1)
        if dkdv:
            out["dkdv_kernel_tflops_executed"] = round(2.0 * f / dkdv[0] / 1e9, 1)
        row[f"{blkq}x{blkk}"] = out
    row["calls"] = iters
    return row


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--shape", default="both", choices=("A", "B", "both"))
    ap.add_argument("--topk", type=float, default=0.1)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--dtype", default="bf16", choices=sorted(DTYPES))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sla_q64_16bit.py measures on the GPU; no CUDA device found")
    print(json.dumps(device_info()), flush=True)
    for name in (("A", "B") if args.shape == "both" else (args.shape,)):
        print(json.dumps(run_shape(name, args.topk, args.iters, args.warmup, DTYPES[args.dtype])), flush=True)


if __name__ == "__main__":
    main()
