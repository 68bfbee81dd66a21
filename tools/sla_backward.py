"""Time the SparseLinearAttention training path (16-bit Q.K^T, BLKQ = 128, BLKK = 64, bf16) on one GPU.

    python tools/sla_backward.py [--shape A|B|both] [--topk 0.1] [--iters 20] [--warmup 5]

Per shape, in one run, after warm-up, with CUDA events (medians over --iters calls):
  * the module's training-path forward (block selection, sparse branch with lse, torch linear branch) and its backward
    (loss = sum(out * g): the sparse backward kernels plus torch's linear-branch and proj_l backward);
  * the sparse backward alone (tdb200_sla_attn_bwd_qk16: four launches), and each of its kernels from a torch.profiler pass
    of its own (mean device time per launch over --iters calls);
  * torch's dense F.scaled_dot_product_attention forward and backward on the same q, k, v, as context.
FLOP convention (Mblk = ceil(L/128)): forward F = H * Mblk * topk * 4 * 128 * 64 * D; useful backward FLOPs = 2.5 F (dQ, dK, dV
and the recomputed S); executed backward FLOPs = 3.5 F (the dQ kernel recomputes S and dP as well).  Dense SDPA: forward
4 * L^2 * H * D, backward 2.5x that.  One JSON line per shape, preceded by the device name and power limit; the SM clock and
throttle reasons are read before and after each shape's timed window.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from sla_block_families import SHAPES, clock_state, device_info  # noqa: E402

KERNELS = ("sla_bwd_delta_kernel", "sla_bwd_kmajor_index_kernel", "sla_bwd_dq_kernel", "sla_bwd_dkdv_kernel")


def _median_ms(fn, iters):
    times = []
    for _ in range(iters):
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        fn()
        end.record()
        end.synchronize()
        times.append(start.elapsed_time(end))
    return statistics.median(times)


def run_shape(name, topk_ratio, iters, warmup):
    from turbodiffusion_b200.SLA import SparseLinearAttention
    from turbodiffusion_b200.SLA.core import attn_bwd_qk16, attn_fwd_qk16_lse
    l, h, d = SHAPES[name]
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(0)
    q, k, v = (torch.randn(1, l, h, d, device=dev, generator=g, dtype=torch.bfloat16) for _ in range(3))
    mod = SparseLinearAttention(d, topk_ratio, BLKQ=128, BLKK=64).to(dev)
    qg, kg, vg = (t.clone().requires_grad_() for t in (q, k, v))
    gout = torch.randn(q.shape, device=dev, generator=g, dtype=torch.bfloat16)
    _, sel = mod.forward_with_lut(q, k, v)
    lut, topk = sel["lut"], sel["topk"]
    o_s, lse = attn_fwd_qk16_lse(q, k, v, lut, topk, d ** -0.5)

    state = {}

    def fwd():
        state["out"] = mod(qg, kg, vg)

    def bwd():
        state["out"].backward(gout)

    def sparse_bwd():
        attn_bwd_qk16(q, k, v, o_s, gout, lse, lut, topk, d ** -0.5)

    qh, kh, vh = (t.transpose(1, 2).clone().requires_grad_() for t in (q, k, v))

    def sdpa_fwd():
        state["dense"] = F.scaled_dot_product_attention(qh, kh, vh)

    def sdpa_bwd():
        state["dense"].backward(gout.transpose(1, 2))

    for _ in range(warmup):
        fwd(), bwd(), sparse_bwd(), sdpa_fwd(), sdpa_bwd()
    torch.cuda.synchronize()
    row = {"shape": name, "L": l, "heads": h, "head_dim": d, "topk_ratio": topk_ratio, "topk_blocks": topk,
           "sm_clock_throttle_before": clock_state()}
    t_fwd, t_bwd, t_sdpa_f, t_sdpa_b = [], [], [], []
    for _ in range(iters):   # module and dense legs interleaved, forward and backward timed separately
        t_fwd.append(_median_ms(fwd, 1))
        t_bwd.append(_median_ms(bwd, 1))
        t_sdpa_f.append(_median_ms(sdpa_fwd, 1))
        t_sdpa_b.append(_median_ms(sdpa_bwd, 1))
    t_sparse = _median_ms(sparse_bwd, iters)
    row["sm_clock_throttle_after"] = clock_state()

    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            sparse_bwd()
        torch.cuda.synchronize()
    per_kernel = {}
    for ev in prof.key_averages():
        for kname in KERNELS:
            if kname in ev.key:
                per_kernel[kname] = per_kernel.get(kname, 0.0) + ev.device_time_total / 1e3 / iters

    mblk = (l + 127) // 128
    f = h * mblk * topk * 4 * 128 * 64 * d
    dense_f = 4 * l * l * h * d
    med = statistics.median
    row.update({
        "module_fwd_ms": round(med(t_fwd), 3), "module_bwd_ms": round(med(t_bwd), 3),
        "sparse_bwd_ms": round(t_sparse, 3),
        "sparse_bwd_useful_tflops": round(2.5 * f / t_sparse / 1e9, 1),
        "sparse_bwd_executed_tflops": round(3.5 * f / t_sparse / 1e9, 1),
        "kernel_ms": {kname: round(ms, 3) for kname, ms in per_kernel.items()},
        # F is two block products (S and P.V); the dQ kernel runs three (S, dP, dQ), the dK/dV kernel four (S, dP, dV, dK)
        "dq_kernel_tflops_executed": round(1.5 * f / per_kernel["sla_bwd_dq_kernel"] / 1e9, 1),
        "dkdv_kernel_tflops_executed": round(2.0 * f / per_kernel["sla_bwd_dkdv_kernel"] / 1e9, 1),
        "sdpa_fwd_ms": round(med(t_sdpa_f), 3), "sdpa_bwd_ms": round(med(t_sdpa_b), 3),
        "sdpa_bwd_tflops": round(2.5 * dense_f / med(t_sdpa_b) / 1e9, 1),
        "module_bwd_over_sdpa_bwd": round(med(t_bwd) / med(t_sdpa_b), 3),
        "calls": iters,
    })
    return row


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--shape", default="both", choices=("A", "B", "both"))
    ap.add_argument("--topk", type=float, default=0.1)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sla_backward.py measures on the GPU; no CUDA device found")
    print(json.dumps(device_info()), flush=True)
    for name in (("A", "B") if args.shape == "both" else (args.shape,)):
        print(json.dumps(run_shape(name, args.topk, args.iters, args.warmup)), flush=True)


if __name__ == "__main__":
    main()
