"""torch.compile over the tdb200:: operators at shape A (L = 32760, dim 1536, 12 heads of 128, FFN 8960, 30 blocks).

Prints, as JSON lines: the card, its power limit and SM clock; the graph breaks TorchDynamo reports for one block and for each
module (torch._dynamo.explain); the 30-block WanHotPath.step eager vs torch.compile(fullgraph=True) vs mode="reduce-overhead";
and the SparseLinearAttention training step (forward + backward) eager vs compiled.  Times are CUDA-event milliseconds per
step after warm-up, with the eager step's host enqueue time beside them.

    python tools/compile_step.py [--steps N] [--breaks-only]
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from turbodiffusion_b200 import ops  # noqa: E402
from turbodiffusion_b200.block import WanHotPath  # noqa: E402
from turbodiffusion_b200.SLA import SageSparseLinearAttention, SparseLinearAttention  # noqa: E402

L, DIM, HEADS, FFN, LAYERS, LC = 32760, 1536, 12, 8960, 30, 512


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), (s.strip() for s in out.split(","))))
    except (OSError, IndexError, subprocess.SubprocessError):
        return {"name": torch.cuda.get_device_name(0), "power.limit": "unavailable", "clocks.sm": "unavailable"}


def timed(fn, steps, warmup=2):
    """(device ms per call, host enqueue ms per call) over `steps` calls after `warmup`."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.perf_counter()
    s.record()
    for _ in range(steps):
        fn()
    e.record()
    t1 = time.perf_counter()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / steps, (t1 - t0) * 1e3 / steps


def breaks(fn, *args):
    torch._dynamo.reset()
    return torch._dynamo.explain(fn)(*args).graph_break_count


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--breaks-only", action="store_true", help="report graph-break counts and stop")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    print(json.dumps({"card": card(), "torch": torch.__version__}), flush=True)
    g = torch.Generator().manual_seed(7)
    x = torch.randn(L, DIM, generator=g).bfloat16().to(dev)
    e0 = (torch.randn(6, DIM, generator=g) * 0.1).to(dev)
    ctx = torch.randn(LC, DIM, generator=g).bfloat16().to(dev)
    ang = ops.wan_rope_angles(21, 30, 52, DIM // HEADS, dev)
    d = DIM // HEADS

    # graph breaks: one block, each module (inference), the SLA training step
    model = WanHotPath(DIM, FFN, HEADS, 1 if args.breaks_only else LAYERS, dev, topk=0.1, seed=1234)
    blk = model.blocks[0]
    lin = torch.nn.Linear(DIM, DIM).to(dev, torch.bfloat16)
    qkv = [torch.randn(1, 4096, HEADS, d, generator=g).bfloat16().to(dev) for _ in range(3)]
    rep = {"block": breaks(blk.forward, x, e0, ang, ctx),
           "Int8Linear": breaks(ops.Int8Linear.from_linear(lin), x),
           "FastRMSNorm": breaks(ops.FastRMSNorm(DIM).to(dev), x),
           "FastLayerNorm": breaks(ops.FastLayerNorm(DIM).to(dev), x),
           "SageSparseLinearAttention": breaks(SageSparseLinearAttention(d, 0.1).to(dev), *qkv),
           "SparseLinearAttention": breaks(SparseLinearAttention(d, 0.1, BLKQ=128, BLKK=64).to(dev), *qkv),
           "SparseLinearAttention_train": breaks(SparseLinearAttention(d, 0.1, BLKQ=128, BLKK=64).to(dev),
                                                 *[t.clone().requires_grad_() for t in qkv])}
    print(json.dumps({"graph_breaks": rep}), flush=True)
    if args.breaks_only:
        return

    # the 30-block denoise step
    res = {}
    eager = model.step(x, e0, ang, ctx)
    res["eager_ms"], res["eager_host_enqueue_ms"] = timed(lambda: model.step(x, e0, ang, ctx), args.steps)
    for name, kw in (("compiled_ms", dict(fullgraph=True)), ("reduce_overhead_ms", dict(fullgraph=True, mode="reduce-overhead"))):
        torch._dynamo.reset()
        step = torch.compile(model.step, **kw)
        t0 = time.perf_counter()
        out = step(x, e0, ang, ctx)
        torch.cuda.synchronize()
        res[name.replace("_ms", "_compile_s")] = round(time.perf_counter() - t0, 1)
        res[name], _ = timed(lambda: step(x, e0, ang, ctx), args.steps)
        out = step(x, e0, ang, ctx)
        # relative L2 to the eager step (a second eager step, below, is bit-identical: the moments are summed in a fixed order)
        res[name.replace("_ms", "_rel_l2_vs_eager")] = ((out.float() - eager.float()).norm() / eager.float().norm()).item()
    again = model.step(x, e0, ang, ctx)
    res["eager_rel_l2_vs_eager"] = ((again.float() - eager.float()).norm() / eager.float().norm()).item()
    print(json.dumps({"wan_step_shape_a": res}), flush=True)

    # SparseLinearAttention training step at shape A: forward + backward of q, k, v and proj_l
    mod = SparseLinearAttention(d, 0.1, BLKQ=128, BLKK=64).to(dev)
    with torch.no_grad():
        mod.proj_l.weight.normal_(0, 0.05, generator=None)
    q, k, v = (torch.randn(1, L, HEADS, d, generator=g).bfloat16().to(dev).requires_grad_() for _ in range(3))
    gout = torch.randn(1, L, HEADS, d, generator=g).bfloat16().to(dev)

    def train_step(m):
        def run():
            for t in (q, k, v):
                t.grad = None
            mod.zero_grad(set_to_none=True)
            m(q, k, v).backward(gout)
        return run

    tr = {}
    tr["eager_ms"], tr["eager_host_enqueue_ms"] = timed(train_step(mod), args.steps)
    torch._dynamo.reset()
    cm = torch.compile(mod, fullgraph=True)
    tr["compiled_ms"], _ = timed(train_step(cm), args.steps)
    print(json.dumps({"sla_train_step_shape_a": tr}), flush=True)


if __name__ == "__main__":
    main()
