"""Time SparseLinearAttention's linear branch on the CUDA kernels ("fused", SLA.core.linear_branch) against the reference torch
composition ("reference", the module's _linear_branch), alternating the two legs call by call.  bf16, d = 128, (BLKQ, BLKK) =
(128, 64).  Legs: the linear branch alone (forward; forward + backward; forward + tangent) and the module's training forward +
backward, forward_jvp without grad, forward_jvp with grad + backward, and torch.func.jvp through forward, each with its peak
memory.  Prints the device, power limit, SM clock and throttle reasons, then one JSON line per (shape, leg, path) with the
median and 10th / 90th percentiles in ms; then a torch.profiler pass per path (reference first) at shape A listing every
kernel of the branch's forward + backward and forward + tangent with its time.

    python tools/sla_linear_branch.py [--calls 50] [--shapes A,B,C]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SHAPES = {"A": (32760, 12, 0.1), "B": (75600, 40, 0.1), "C": (28672, 32, 0.3)}   # (L, heads, top-k)


def device_report():
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks_throttle_reasons.active"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout
    except OSError:
        out = "nvidia-smi unavailable"
    return {"device": torch.cuda.get_device_name(), "nvidia_smi": out.strip()}


def pct(xs, p):
    xs = sorted(xs)
    return xs[min(len(xs) - 1, int(round(p / 100 * (len(xs) - 1))))]


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def profile(fwd_bwd, tangent):
    """Per-kernel CUDA times of the linear branch's forward + backward and forward + tangent, reference path first."""
    from torch.profiler import ProfilerActivity, profile as prof
    for path in ("reference", "fused"):
        for leg, fn in (("fwd_bwd", fwd_bwd), ("fwd_tangent", tangent)):
            fn(path)
            torch.cuda.synchronize()
            with prof(activities=[ProfilerActivity.CUDA]) as p:
                for _ in range(5):
                    fn(path)
                torch.cuda.synchronize()
            rows = {}
            for e in p.events():
                if e.device_type == torch.autograd.DeviceType.CUDA:
                    r = rows.setdefault(e.name, [0, 0.0])
                    r[0] += 1
                    r[1] += e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
            for kname, (n, us) in sorted(rows.items(), key=lambda kv: -kv[1][1]):
                print(json.dumps({"profile": path, "leg": leg, "kernel": kname[:90], "launches_per_call": n / 5,
                                  "us_per_call": round(us / 5, 1)}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--shapes", default="A,B,C")
    args = ap.parse_args()
    from turbodiffusion_b200.SLA import utils
    import torch.autograd.forward_ad as fwAD
    from turbodiffusion_b200.SLA.core import SparseLinearAttention, linear_branch, linear_branch_jvp
    print(json.dumps(device_report()))
    for name in args.shapes.split(","):
        l, h, topk = SHAPES[name]
        torch.manual_seed(0)
        q, k, v, do = (torch.randn(1, l, h, 128, device="cuda", dtype=torch.bfloat16) for _ in range(4))
        m = SparseLinearAttention(128, topk, "softmax", BLKQ=128, BLKK=64).cuda()
        with torch.no_grad():
            m.proj_l.weight.normal_(0, 128 ** -0.5)
        qg, kg, vg = (t.clone().requires_grad_() for t in (q, k, v))

        def branch(path):
            if path == "fused":
                return linear_branch(qg, kg, vg, m.proj_l.weight, m.proj_l.bias, m.feature)
            return m._linear_branch(qg, kg, vg)

        def fwd(path):
            with torch.no_grad():
                branch(path)

        def fwd_bwd(path):
            branch(path).backward(do)

        qt, kt, vt = (torch.randn_like(q) for _ in range(3))

        def tangent(path):
            with torch.no_grad():
                if path == "fused":
                    return linear_branch_jvp(q, k, v, qt, kt, vt, m.proj_l.weight, m.proj_l.bias, m.feature)
                with fwAD.dual_level():
                    return fwAD.unpack_dual(m._linear_branch(fwAD.make_dual(q, qt), fwAD.make_dual(k, kt),
                                                             fwAD.make_dual(v, vt)))

        def selected(fn):
            def run(path):
                utils.set_linear_branch(path)
                try:
                    return fn()
                finally:
                    utils.set_linear_branch("reference")
            return run

        def jvp_nograd():
            with torch.no_grad():
                m.forward_jvp(q, k, v, qt, kt, vt)

        legs = (("linear_branch_fwd", fwd), ("linear_branch_fwd_bwd", fwd_bwd), ("linear_branch_fwd_tangent", tangent),
                ("module_train_fwd_bwd", selected(lambda: m(qg, kg, vg).backward(do))),
                ("module_forward_jvp", selected(jvp_nograd)),
                ("module_forward_jvp_grad_bwd", selected(lambda: m.forward_jvp(qg, kg, vg, qt, kt, vt)[0].backward(do))),
                ("module_func_jvp", selected(lambda: torch.func.jvp(lambda a, b, c: m(a, b, c), (q, k, v), (qt, kt, vt)))))
        if name == "A":
            profile(fwd_bwd, tangent)
        for leg, fn in legs:
            times = {"reference": [], "fused": []}
            peak = {}
            for path in times:            # warm-up
                fn(path)
            for _ in range(args.calls):
                for path in times:
                    torch.cuda.reset_peak_memory_stats()
                    times[path].append(timed(lambda: fn(path)))
                    peak[path] = max(peak.get(path, 0), torch.cuda.max_memory_allocated())
            for path, xs in times.items():
                print(json.dumps({"shape": name, "L": l, "heads": h, "leg": leg, "path": path, "calls": len(xs),
                                  "median_ms": round(pct(xs, 50), 4), "p10_ms": round(pct(xs, 10), 4),
                                  "p90_ms": round(pct(xs, 90), 4), "peak_mib": round(peak[path] / 2 ** 20)}))
            qg.grad = kg.grad = vg.grad = None
            m.zero_grad()
    print(json.dumps(device_report()))


if __name__ == "__main__":
    main()
