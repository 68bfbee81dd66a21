"""Time the dense attention training path (ops.dense_attention / ops.dense_attention_jvp with grad, whose backward is
tdb200_attn_dense_bwd) against F.scaled_dot_product_attention's forward and backward on one GPU, bf16, batch 1.

    python tools/dense_attention_bwd.py [--iters 50] [--warmup 5] [--only NAME] [--out-dir DIR]

Shapes (queries x keys, heads x head dim):
  A-cross   32760 x 512,   12 x 128   Wan2.1-1.3B at 480p, cross-attention over the text tokens
  A-self    32760 x 32760, 12 x 128   dense self-attention at shape A
  B-cross   75600 x 512,   40 x 128   Wan2.1-14B at 720p, cross-attention
  C-512     28672 x 512,   32 x 128   LTX shape C's video stream, text keys padded
Legs, each a forward with grad and the backward of one incoming gradient:
  dense        ops.dense_attention (lse forward, then the dense backward)
  sdpa         F.scaled_dot_product_attention (cuDNN on torch 2.11), fed the transposed views block.py feeds it
  jvp          ops.dense_attention_jvp with grad (output and tangent in one kernel), then the backward of its output: the
               primal path of a consistency-distillation step
  jvp_sdpa     what a caller had to do before: the JVP without grad, then SDPA's forward with grad and its backward
Per shape, in one process: every leg warmed up, then --iters rounds of one CUDA-event-timed call of each leg, alternating in
a rotating order; median and 10th / 90th percentiles per leg.  Kernel times come from a torch.profiler pass of their own after
the timed window (three calls per leg, traces in --out-dir); the backward's kernels are those whose names mark them as
backward kernels.  Backward TFLOP/s count useful = 10 * H * Lq * Lk * D (the five products of FlashAttention-2's backward)
and executed = 14 * H * Lq * Lk * D (the dQ and dK/dV kernels each recompute S and dP) over the backward's kernel time.
One JSON line with the device name, power limit and maximum SM clock, then one per shape with the SM clock and throttle reasons
read before and after its timed window.

    python tools/dense_attention_bwd.py --baseline-lib PATH

compares this tree's libtdb200.so with another build of the same C ABI (for example the parent commit's) on seeded inputs:
the SLA backward (tdb200_sla_attn16_bwd) at (BLKQ, BLKK) = (128, 64) and (64, 64) in bf16 and fp16 at shape A's self-attention
size, and the dense forward and JVP entry points.  The two builds alternate call by call; per leg and build the median and
10th / 90th percentile call time.  Every output is compared byte for byte; the script exits non-zero if any differs.
There is no CPU timing: without a CUDA device the script exits with an error."""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import re
import statistics
import sys
import tempfile

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from dense_attention import _kernels  # noqa: E402
from sla_block_families import _pct, _timed, clock_state, device_info  # noqa: E402

D = 128
SHAPES = {"A-cross": (32760, 512, 12), "A-self": (32760, 32760, 12), "B-cross": (75600, 512, 40), "C-512": (28672, 512, 32)}
BWD_KERNEL = re.compile(r"bwd|bprop|backward|dot_do_o|convert_dq")   # ours: sla_bwd_*; cuDNN: dO.O, bprop, dQ conversion


def _spread(ms):
    return {"median_ms": round(statistics.median(ms), 4), "p10_ms": round(_pct(ms, 0.1), 4), "p90_ms": round(_pct(ms, 0.9), 4)}


def _sdpa(q, k, v, sm_scale):
    return F.scaled_dot_product_attention(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2), scale=sm_scale).transpose(1, 2)


def run_shape(name, iters, warmup, out_dir):
    from turbodiffusion_b200 import ops
    lq, lk, h = SHAPES[name]
    g = torch.Generator(device="cuda").manual_seed(0)
    q, q_t, d_out = (torch.randn(1, lq, h, D, device="cuda", generator=g).bfloat16() for _ in range(3))
    k, v, k_t, v_t = (torch.randn(1, lk, h, D, device="cuda", generator=g).bfloat16() for _ in range(4))
    leaves = [t.clone().requires_grad_() for t in (q, k, v)]
    sm_scale = D ** -0.5

    def backward(out):   # fresh gradients every call: no accumulation into the previous call's
        for t in leaves:
            t.grad = None
        out.backward(d_out)

    def dense():
        backward(ops.dense_attention(*leaves, sm_scale))

    def sdpa():
        backward(_sdpa(*leaves, sm_scale))

    def jvp():
        backward(ops.dense_attention_jvp(*leaves, q_t, k_t, v_t, sm_scale)[0])

    def jvp_sdpa():
        with torch.no_grad():
            ops.dense_attention_jvp(q, k, v, q_t, k_t, v_t, sm_scale)
        backward(_sdpa(*leaves, sm_scale))

    legs = {"dense": dense, "sdpa": sdpa, "jvp": jvp, "jvp_sdpa": jvp_sdpa}
    for _ in range(warmup):
        for fn in legs.values():
            fn()
    torch.cuda.synchronize()
    row = {"shape": name, "Lq": lq, "Lk": lk, "heads": h, "head_dim": D, "dtype": "bf16", "batch": 1,
           "dkdv_ctas": -(-lk // 64) * h, "dq_ctas": -(-lq // 128) * h, "sm_clock_throttle_before": clock_state()}
    names = list(legs)
    times = {n: [] for n in names}
    for i in range(iters):
        r = i % len(names)
        for n in names[r:] + names[:r]:
            times[n].append(_timed(legs[n]))
    row["sm_clock_throttle_after"] = clock_state()
    useful, executed = 10 * h * lq * lk * D, 14 * h * lq * lk * D
    for n in names:
        kern = _kernels(legs[n], 3, os.path.join(out_dir, f"{name}_{n}.trace.json"))
        bwd_ms = sum(ms for k_, ms in kern.items() if BWD_KERNEL.search(k_))
        row[n] = {**_spread(times[n]), "kernels_ms_per_call": kern, "backward_kernels_ms": round(bwd_ms, 4)}
        if bwd_ms > 0:
            row[n]["backward_tflops_useful"] = round(useful / bwd_ms / 1e9, 1)
            if n in ("dense", "jvp"):
                row[n]["backward_tflops_executed"] = round(executed / bwd_ms / 1e9, 1)
    row["calls_per_leg"] = iters
    return row


# ------------------------------------------------------------------------------------------------ two builds
def _load(path):
    from turbodiffusion_b200 import _lib
    handle = ctypes.CDLL(path)
    for name in ("tdb200_sla_attn16_bwd", "tdb200_sla_attn16_bwd_workspace_bytes", "tdb200_attn_dense_fwd", "tdb200_attn_dense_jvp"):
        fn = getattr(handle, name)
        fn.argtypes = _lib._PROTOS[name]
        fn.restype = _lib._RESTYPES.get(name, ctypes.c_int)
    return handle


def _check(rc, what):
    if rc != 0:
        raise RuntimeError(f"{what} returned {rc}")


def _builds_legs(lib, ins, sla, dtype):
    """Per leg: a call of one build's entry point and the fresh output buffers it writes."""
    from turbodiffusion_b200._lib import DTYPE_TAG, ptr
    q, k, v, d_out, q_t, k_t, v_t = ins
    b, l, h, d = q.shape
    tag, st, sm = DTYPE_TAG[dtype], torch.cuda.current_stream().cuda_stream, d ** -0.5
    legs = {}
    for blkq, (lut, topk, o_s, lse) in sla.items():
        dq, dk, dv = (torch.empty_like(q) for _ in range(3))
        nbytes = lib.tdb200_sla_attn16_bwd_workspace_bytes(b, h, l, topk, blkq)
        ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")

        def call(blkq=blkq, lut=lut, topk=topk, o_s=o_s, lse=lse, dq=dq, dk=dk, dv=dv, ws=ws, nbytes=nbytes):
            _check(lib.tdb200_sla_attn16_bwd(ptr(q), ptr(k), ptr(v), ptr(o_s), ptr(d_out), ptr(lse), tag, ptr(lut), topk, ptr(dq),
                                             ptr(dk), ptr(dv), ptr(ws), nbytes, b, l, h, d, sm, blkq, 64, st), "sla_attn16_bwd")
        legs[f"sla_bwd_{blkq}x64"] = (call, [dq, dk, dv])
    lq = 4000                                              # the dense operators on a ragged cross-attention slice
    qc, qtc, kc, vc, ktc, vtc = (t[:, :n].contiguous() for t, n in ((q, lq), (q_t, lq), (k, 600), (v, 600), (k_t, 600), (v_t, 600)))
    out, out2, out_t = (torch.empty_like(qc) for _ in range(3))
    legs["dense_fwd"] = (lambda: _check(lib.tdb200_attn_dense_fwd(ptr(qc), ptr(kc), ptr(vc), tag, ptr(out), b, lq, 600, h, d, sm, st),
                                        "attn_dense_fwd"), [out])
    legs["dense_jvp"] = (lambda: _check(lib.tdb200_attn_dense_jvp(ptr(qc), ptr(kc), ptr(vc), ptr(qtc), ptr(ktc), ptr(vtc), tag,
                                                                  ptr(out2), ptr(out_t), b, lq, 600, h, d, sm, st),
                                        "attn_dense_jvp"), [out2, out_t])
    return legs


def run_builds(baseline_lib, iters, warmup):
    from turbodiffusion_b200 import _lib
    from turbodiffusion_b200.SLA.core import attn_fwd_qk16_lse
    l, h = 32760, 12
    builds = {"this": _load(_lib.LIB_PATH), "baseline": _load(baseline_lib)}
    rows, same_all = [], True
    for dtype in (torch.bfloat16, torch.float16):
        g = torch.Generator(device="cuda").manual_seed(7)
        ins = [torch.randn(1, l, h, D, generator=g, device="cuda").to(dtype) for _ in range(7)]
        sla = {}
        for blkq in (128, 64):
            mblk, nblk = -(-l // blkq), -(-l // 64)
            topk = nblk // 10
            lut = torch.rand(1, h, mblk, nblk, generator=g, device="cuda").topk(topk, -1).indices.int().contiguous()
            o_s, lse = attn_fwd_qk16_lse(ins[0], ins[1], ins[2], lut, topk, D ** -0.5, blkq)
            sla[blkq] = (lut, topk, o_s, lse)
        legs = {bn: _builds_legs(lib, ins, sla, dtype) for bn, lib in builds.items()}
        calls = [(leg, bn) for leg in legs["this"] for bn in builds]
        times = {c: [] for c in calls}
        for i in range(warmup + iters):
            r = i % len(calls)
            for leg, bn in calls[r:] + calls[:r]:
                t = _timed(legs[bn][leg][0])
                if i >= warmup:
                    times[(leg, bn)].append(t)
        for leg in legs["this"]:
            same = all(torch.equal(a.view(torch.uint8), b.view(torch.uint8))
                       for a, b in zip(legs["this"][leg][1], legs["baseline"][leg][1]))
            same_all &= same
            row = {"leg": leg, "dtype": str(dtype).replace("torch.", ""), "L": l, "heads": h, "outputs_byte_identical": same,
                   "calls": iters, **{bn: _spread(times[(leg, bn)]) for bn in builds}}
            row["median_ratio_this_over_baseline"] = round(row["this"]["median_ms"] / row["baseline"]["median_ms"], 4)
            rows.append(row)
    return rows, same_all


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--only", choices=tuple(SHAPES), default=None)
    ap.add_argument("--out-dir", default=None, help="where the profiler traces go (default: a new temporary directory)")
    ap.add_argument("--baseline-lib", default=None,
                    help="another libtdb200.so with the same C ABI: compare its outputs and times with this tree's build")
    args = ap.parse_args()
    if args.iters < 50:
        ap.error("--iters: at least 50 timed calls per leg")
    if not torch.cuda.is_available():
        raise SystemExit("dense_attention_bwd.py measures on the GPU; no CUDA device found")
    if args.baseline_lib is not None:
        from turbodiffusion_b200 import _lib
        print(json.dumps({**device_info(), "builds": {"this": _lib.LIB_PATH, "baseline": os.path.abspath(args.baseline_lib)}}),
              flush=True)
        rows, same = run_builds(os.path.abspath(args.baseline_lib), args.iters, args.warmup)
        for row in rows:
            print(json.dumps(row), flush=True)
        if not same:
            raise SystemExit("the two builds' outputs differ")
        return
    out_dir = args.out_dir or tempfile.mkdtemp(prefix="dense_attention_bwd_")
    os.makedirs(out_dir, exist_ok=True)
    print(json.dumps({**device_info(), "torch": torch.__version__, "traces": out_dir}), flush=True)
    for name in ((args.only,) if args.only else SHAPES):
        print(json.dumps(run_shape(name, args.iters, args.warmup, out_dir)), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
