"""Compare the two SageSLA block families on one GPU: BLKQ=128 / BLKK=64 (the Sage2++ family, served as "sm100") and
BLKQ=64 / BLKK=128 (SpargeAttn's Hopper family, served as "sm90").

    python tools/sla_block_families.py [--shape A|B|both] [--iters 50] [--warmup 10] [--topk 0.1] [--dtype bf16|fp16]

Both families run in the same process and are timed with CUDA events, call by call, in an order that rotates every
iteration (so no timing always follows the same predecessor): the whole SageSparseLinearAttention forward, the fused
attention launch alone (on that family's own prep, LUT and moments), and the work the forward does before the attention
(prep: quantisation, block map, moments, projection); forward ~ prep + attention is a consistency check of the run.  The SM
clock and the active throttle reasons are read before and after each shape's timed window.
Reported per family: median times, the attention's TFLOP/s with FLOPs = H*Mblk*topk*4*BLKQ*BLKK*D (the count bench.py uses;
BLKQ*BLKK = 8192 in both families), and the fraction of keys each query attends to (topk*BLKK/L).  One JSON line per
(shape, family), preceded by one line with the device name and power limit read in the same run.

    python tools/sla_block_families.py --ranks 1,2,4,8 [--shape ...]

times instead, for each world size N, rank 0's share of one sequence-parallel attention layer (dist.py) on this one GPU, both
families in the same rotating order: in the all-gather mode its own key prep (128-row partial sums, key mean, INT8 and
pooling of its rows), its Q prep and block map and the fused attention of its query rows over the whole gathered slab
("allgather"; the fused attention alone is "allgather_attn"); in the Ulysses mode the single-GPU pipeline on its H/N heads
(rank 0 takes the extra head of an uneven split).  The collectives and their overlap with compute are not timed.  One JSON
line per (shape, N, family).

    python tools/sla_block_families.py --baseline-lib PATH [--shape ...]

compares this tree's libtdb200.so with another build of the same C ABI (for example the parent commit's), loaded side by
side: at each shape the fused attention of both INT8 families, the 16-bit (128, 64) forward and its lse forward, and the
16-bit (64, 64) forward are called through the C entry points on the same inputs, the two builds alternating call by call in
a rotating order.  Per leg and build:
median, 10th and 90th percentile of the call time.  Every output of the two builds (out, and lse for the lse forward) is
compared byte for byte; the script exits non-zero if any leg differs.

--dtype (bf16 by default) is the type of q, k, v, the output and every 16-bit MMA operand, in all three modes.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SHAPES = {"A": (32760, 12, 128), "B": (75600, 40, 128)}   # (L, heads, head dim): Wan2.1-1.3B and Wan2.1-14B at 480p / 720p
FAMILIES = ("sm100", "sm90")


def device_info():
    name = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError) as e:
        power = f"unavailable ({e})"
    return {"device": name, "power_limit_and_max_sm_clock": power}


def clock_state():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks_throttle_reasons.active", "--format=csv,noheader",
                               "-i", "0"], capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError) as e:
        return f"unavailable ({e})"


def _timed(fn):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end)


def _module(d, ratio, device, dtype=torch.bfloat16):
    from turbodiffusion_b200.SLA import SageSparseLinearAttention
    mod = SageSparseLinearAttention(d, ratio, use_bf16=dtype == torch.bfloat16).to(device)
    with torch.no_grad():
        mod.proj_l.weight.normal_(0, 0.05)
        mod.proj_l.bias.normal_(0, 0.05)
    return mod


def setup(arch, q, k, v, ratio):
    """The module and one family's attention inputs, built by the same calls its forward makes."""
    from turbodiffusion_b200.SLA.core import attn_fwd, linear_moments, project_moments
    from turbodiffusion_b200.SLA.utils import block_map_from_pools, quant_qk, set_served_arch
    set_served_arch(arch)
    d = q.shape[-1]
    mod = _module(d, ratio, q.device, q.dtype)
    blkq, blkk = mod.block_sizes(q.device.index)
    prep = quant_qk(q, k, blkq=blkq, blkk=blkk)
    topk = max(1, min(prep.nblk, int(ratio * prep.nblk)))
    _, lut = block_map_from_pools(prep.q_pool, prep.k_pool, topk)
    kv, ksum = linear_moments(k, v)
    kvw = project_moments(mod.proj_l.weight, kv, q.dtype)
    pb = mod.proj_l.bias.float().contiguous()

    def attn():
        attn_fwd(prep, v, q, lut, topk, kvw, ksum, pb, d ** -0.5, blkq=blkq, blkk=blkk)

    def forward():
        mod(q, k, v)

    def prep_only():   # what forward() runs before the fused attention
        p = quant_qk(q, k, blkq=blkq, blkk=blkk)
        block_map_from_pools(p.q_pool, p.k_pool, topk)
        project_moments(mod.proj_l.weight, linear_moments(k, v)[0], q.dtype)

    return {"blkq": blkq, "blkk": blkk, "mblk": prep.mblk, "topk": topk, "attn": attn, "forward": forward, "prep": prep_only}


DTYPES = {"bf16": torch.bfloat16, "fp16": torch.float16}


def inputs(name, dtype):
    """Seeded q, k, v [1, L, H, D] of shape `name` in `dtype`, keys with a shared offset per head."""
    l, h, d = SHAPES[name]
    g = torch.Generator(device="cuda").manual_seed(0)
    q, k, v = (torch.randn(1, l, h, d, generator=g, device="cuda").to(dtype) for _ in range(3))
    k += torch.randn(1, 1, h, d, generator=g, device="cuda").to(dtype) * 2
    return q, k, v


def run_shape(name, ratio, iters, warmup, dtype):
    from turbodiffusion_b200.SLA.utils import set_served_arch
    l, h, d = SHAPES[name]
    q, k, v = inputs(name, dtype)
    prev = set_served_arch("sm100")
    try:
        fams = {arch: setup(arch, q, k, v, ratio) for arch in FAMILIES}
        kinds = ("attn", "forward", "prep")
        times = {arch: {what: [] for what in kinds} for arch in FAMILIES}
        calls = [(arch, what) for arch in FAMILIES for what in kinds]
        clocks = {}
        for i in range(warmup + iters):
            if i == warmup:
                clocks["sm_clock_throttle_before"] = clock_state()
            r = i % len(calls)
            for arch, what in calls[r:] + calls[:r]:
                set_served_arch(arch)
                t = _timed(fams[arch][what])
                if i >= warmup:
                    times[arch][what].append(t)
        clocks["sm_clock_throttle_after"] = clock_state()
    finally:
        set_served_arch(prev)
    rows = []
    for arch in FAMILIES:
        f = fams[arch]
        attn_ms = statistics.median(times[arch]["attn"])
        flops = h * f["mblk"] * f["topk"] * 4 * f["blkq"] * f["blkk"] * d
        rows.append({"shape": name, "L": l, "heads": h, "head_dim": d, "dtype": str(q.dtype)[6:], "family": arch, "blkq": f["blkq"], "blkk": f["blkk"],
                     "topk": f["topk"], "keys_per_query": round(f["topk"] * f["blkk"] / l, 4),
                     "attn_ms_median": round(attn_ms, 4), "attn_tflops": round(flops / attn_ms / 1e9, 1),
                     "forward_ms_median": round(statistics.median(times[arch]["forward"]), 4),
                     "prep_ms_median": round(statistics.median(times[arch]["prep"]), 4), "calls": iters, **clocks})
    base, hop = rows
    hop["attn_tflops_vs_sm100"] = round(hop["attn_tflops"] / base["attn_tflops"], 3)
    return rows


def _load_build(path):
    """The attention entry points of the libtdb200.so at `path`, typed from this tree's prototypes."""
    import ctypes
    from turbodiffusion_b200 import _lib
    handle = ctypes.CDLL(path)
    fns = {}
    for name in ("tdb200_sla_attn_fwd", "tdb200_sla_attn16_fwd", "tdb200_sla_attn16_fwd_lse"):
        fn = getattr(handle, name)
        fn.argtypes = _lib._PROTOS[name]
        fn.restype = ctypes.c_int
        fns[name] = fn
    return fns


def _build_legs(fns, q, k, v, ratio):
    """Per leg, a call of one build's entry point and the output buffers it writes (fresh for this build)."""
    from turbodiffusion_b200._lib import DTYPE_TAG, ptr
    from turbodiffusion_b200.SLA.core import linear_moments, project_moments
    from turbodiffusion_b200.SLA.core import select_prep
    from turbodiffusion_b200.SLA.utils import block_map_from_pools, quant_qk
    b, l, h, d = q.shape
    g = torch.Generator(device="cuda").manual_seed(1)
    w = torch.randn(d, d, generator=g, device="cuda") * 0.05
    pb = (torch.randn(d, generator=g, device="cuda") * 0.05).contiguous()
    kv, ksum = linear_moments(k, v)
    kvw = project_moments(w, kv, q.dtype)
    stream = torch.cuda.current_stream().cuda_stream
    tag, sm_scale = DTYPE_TAG[q.dtype], d ** -0.5
    legs = {}

    def check(rc, what):
        if rc != 0:
            raise RuntimeError(f"{what} returned {rc}")

    for fam, (blkq, blkk) in (("sm100", (128, 64)), ("sm90", (64, 128))):
        prep = quant_qk(q, k, blkq=blkq, blkk=blkk)
        topk = max(1, min(prep.nblk, int(ratio * prep.nblk)))
        _, lut = block_map_from_pools(prep.q_pool, prep.k_pool, topk)
        out = torch.empty_like(q)

        def call(prep=prep, lut=lut, topk=topk, out=out, blkq=blkq, blkk=blkk):
            check(fns["tdb200_sla_attn_fwd"](ptr(prep.q_i8), ptr(prep.q_scale), ptr(prep.k_i8), ptr(prep.k_scale), ptr(v), ptr(q),
                                             tag, ptr(lut), topk, ptr(kvw), ptr(ksum), ptr(pb), ptr(out), b, l, l, h, d, sm_scale,
                                             0, blkq, blkk, 0, stream), "tdb200_sla_attn_fwd")
        legs[fam] = {"call": call, "outputs": [out], "mblk": prep.mblk, "topk": topk, "blkq": blkq, "blkk": blkk}
        if fam == "sm100":   # the 16-bit (128, 64) kernels on the same 128 x 64 block list
            out16, o_s = torch.empty_like(q), torch.empty_like(q)
            lse = torch.empty(b, h, l, dtype=torch.float32, device=q.device)

            def call16(lut=lut, topk=topk):
                check(fns["tdb200_sla_attn16_fwd"](ptr(q), ptr(k), ptr(v), tag, ptr(lut), topk, ptr(kvw), ptr(ksum), ptr(pb),
                                                   ptr(out16), b, l, l, h, d, sm_scale, 0, 128, 64, stream), "tdb200_sla_attn16_fwd")

            def call16_lse(lut=lut, topk=topk):
                check(fns["tdb200_sla_attn16_fwd_lse"](ptr(q), ptr(k), ptr(v), tag, ptr(lut), topk, ptr(o_s), ptr(lse), b, l, h, d,
                                                       sm_scale, 128, 64, stream), "tdb200_sla_attn16_fwd_lse")
            common = {"mblk": prep.mblk, "topk": topk, "blkq": 128, "blkk": 64}
            legs["attn16"] = {"call": call16, "outputs": [out16], **common}
            legs["attn16_lse"] = {"call": call16_lse, "outputs": [o_s, lse], **common}
    prep = select_prep(q, k, 64, 64)      # the 16-bit (64, 64) forward on its own selection
    topk = max(1, min(prep.nblk, int(ratio * prep.nblk)))
    _, lut = block_map_from_pools(prep.q_pool, prep.k_pool, topk)
    out64 = torch.empty_like(q)

    def call16_q64(lut=lut, topk=topk):
        check(fns["tdb200_sla_attn16_fwd"](ptr(q), ptr(k), ptr(v), tag, ptr(lut), topk, ptr(kvw), ptr(ksum), ptr(pb), ptr(out64),
                                           b, l, l, h, d, sm_scale, 0, 64, 64, stream), "tdb200_sla_attn16_fwd")
    legs["attn16_q64"] = {"call": call16_q64, "outputs": [out64], "mblk": prep.mblk, "topk": topk, "blkq": 64, "blkk": 64}
    return legs


def _pct(xs, f):
    xs = sorted(xs)
    return xs[min(len(xs) - 1, int(round(f * (len(xs) - 1))))]


def run_builds(name, ratio, iters, warmup, baseline_lib, dtype):
    """This tree's build against `baseline_lib`, leg by leg, alternated call by call; returns (rows, all outputs identical)."""
    from turbodiffusion_b200 import _lib
    l, h, d = SHAPES[name]
    q, k, v = inputs(name, dtype)
    builds = {"this": _load_build(_lib.LIB_PATH), "baseline": _load_build(baseline_lib)}
    legs = {bn: _build_legs(fns, q, k, v, ratio) for bn, fns in builds.items()}
    names = list(legs["this"])
    calls = [(leg, bn) for leg in names for bn in builds]
    times = {c: [] for c in calls}
    clocks = {}
    for i in range(warmup + iters):
        if i == warmup:
            clocks["sm_clock_throttle_before"] = clock_state()
        r = i % len(calls)
        for leg, bn in calls[r:] + calls[:r]:
            t = _timed(legs[bn][leg]["call"])
            if i >= warmup:
                times[(leg, bn)].append(t)
    clocks["sm_clock_throttle_after"] = clock_state()
    rows, same_all = [], True
    for leg in names:
        f = legs["this"][leg]
        same = all(torch.equal(a.view(torch.uint8), b_.view(torch.uint8))
                   for a, b_ in zip(legs["this"][leg]["outputs"], legs["baseline"][leg]["outputs"]))
        same_all &= same
        flops = h * f["mblk"] * f["topk"] * 4 * f["blkq"] * f["blkk"] * d
        row = {"shape": name, "L": l, "heads": h, "head_dim": d, "dtype": str(dtype)[6:], "leg": leg, "blkq": f["blkq"], "blkk": f["blkk"], "topk": f["topk"],
               "outputs_byte_identical": same, "calls": iters, **clocks}
        for bn in builds:
            ts = times[(leg, bn)]
            med = statistics.median(ts)
            row[bn] = {"ms_median": round(med, 4), "ms_p10": round(_pct(ts, 0.1), 4), "ms_p90": round(_pct(ts, 0.9), 4),
                       "tflops": round(flops / med / 1e9, 1)}
        row["median_ratio_this_over_baseline"] = round(row["this"]["ms_median"] / row["baseline"]["ms_median"], 4)
        rows.append(row)
    return rows, same_all


def setup_rank0(arch, q, k, v, ratio, world):
    """Rank 0's share of one sequence-parallel layer on `world` GPUs (dist.py), on one family's blocks, built from the real
    per-rank primitives.  The gathered slab rank 0 attends over is made here from the whole sequence; the split key prep
    reproduces it bit for bit (tests/test_gpu_sp_hopper_blocks.py)."""
    from turbodiffusion_b200.dist import GpuPrimitives, UlyssesGpuPrims, shard_rows, split_heads
    from turbodiffusion_b200.SLA.core import attn_fwd, linear_moments, project_moments
    from turbodiffusion_b200.SLA.utils import block_map_from_pools, kmean_from_partials, kmean_partials, quant_k_seq, set_served_arch
    set_served_arch(arch)
    _, l, h, d = q.shape
    mod = _module(d, ratio, q.device, q.dtype)
    gp, up = GpuPrimitives(mod, arch), UlyssesGpuPrims(mod, arch)
    blkq, blkk = gp.blkq, gp.blkk
    begin, end, rows_pad = shard_rows(l, world, 0)
    q0, k0 = q[:, begin:end].contiguous(), k[:, begin:end].contiguous()
    partials = kmean_partials(k)                               # every rank's partials, as gathered
    kmean = kmean_from_partials(partials, l)
    k8 = torch.zeros(1, world * rows_pad, h, d, dtype=torch.int8, device=q.device)
    _, k_scale, k_pool = quant_k_seq(k, kmean, k8[:, :l], blkk=blkk)
    v_full = torch.zeros(1, world * rows_pad, h, d, dtype=v.dtype, device=v.device)
    v_full[:, :l] = v
    kv, ksum = linear_moments(k, v)
    pb = mod.proj_l.bias.float().contiguous()

    def allgather():     # own key prep (partials, mean, INT8 + pooling of its rows), Q prep + block map, fused attention
        gp.k_partials(k0)
        gp.k_quant(k0, gp.k_mean(partials, l))
        gp.attention_i8(q0, gp.prepare_q(q0), k8, k_scale, k_pool, kmean, v_full, l, kv, ksum)

    prep = gp.prepare_q(q0)
    prep.kmean, prep.k_i8, prep.k_scale, prep.k_pool, prep.nblk, prep.k_seq_major = kmean, k8, k_scale, k_pool, k_scale.shape[-1], True
    topk = min(prep.nblk, int(ratio * prep.nblk))
    _, lut = block_map_from_pools(prep.q_pool, prep.k_pool, topk)
    kvw = project_moments(mod.proj_l.weight, kv, q.dtype)

    def allgather_attn():
        attn_fwd(prep, v_full, q0, lut, topk, kvw, ksum, pb, d ** -0.5, lk=l, blkq=blkq, blkk=blkk)

    hl = split_heads(h, world)[0][0]                           # rank 0 holds the most heads
    qh, kh, vh = (t[:, :, :hl].contiguous() for t in (q, k, v))

    def ulysses():       # the single-GPU pipeline on rank 0's heads of the whole sequence
        up.attend(lambda: qh, lambda: kh, lambda: vh)

    return {"blkq": blkq, "blkk": blkk, "rows": end - begin, "heads": hl, "mblk": prep.mblk, "topk": topk,
            "allgather": allgather, "allgather_attn": allgather_attn, "ulysses": ulysses}


def run_ranks(name, ratio, iters, warmup, ranks, dtype):
    """Rank 0's share per family for each world size; collectives are not timed."""
    from turbodiffusion_b200.SLA.utils import set_served_arch
    l, h, d = SHAPES[name]
    q, k, v = inputs(name, dtype)
    rows = []
    prev = set_served_arch("sm100")
    try:
        for world in ranks:
            fams = {arch: setup_rank0(arch, q, k, v, ratio, world) for arch in FAMILIES}
            kinds = ("allgather", "allgather_attn", "ulysses")
            times = {arch: {what: [] for what in kinds} for arch in FAMILIES}
            calls = [(arch, what) for arch in FAMILIES for what in kinds]
            clocks = {}
            for i in range(warmup + iters):
                if i == warmup:
                    clocks["sm_clock_throttle_before"] = clock_state()
                r = i % len(calls)
                for arch, what in calls[r:] + calls[:r]:
                    set_served_arch(arch)
                    t = _timed(fams[arch][what])
                    if i >= warmup:
                        times[arch][what].append(t)
            clocks["sm_clock_throttle_after"] = clock_state()
            out = []
            for arch in FAMILIES:
                f = fams[arch]
                med = {what: statistics.median(times[arch][what]) for what in kinds}
                flops = h * f["mblk"] * f["topk"] * 4 * f["blkq"] * f["blkk"] * d
                out.append({"shape": name, "L": l, "heads": h, "head_dim": d, "world": world, "family": arch,
                            "blkq": f["blkq"], "blkk": f["blkk"], "rank0_rows": f["rows"], "rank0_query_blocks": f["mblk"],
                            "rank0_ulysses_heads": f["heads"], "topk": f["topk"],
                            "allgather_ms_median": round(med["allgather"], 4),
                            "allgather_attn_ms_median": round(med["allgather_attn"], 4),
                            "allgather_attn_tflops": round(flops / med["allgather_attn"] / 1e9, 1),
                            "ulysses_ms_median": round(med["ulysses"], 4), "calls": iters, **clocks})
            base, hop = out
            for what in kinds:
                hop[f"{what}_speedup_vs_sm100"] = round(base[f"{what}_ms_median"] / hop[f"{what}_ms_median"], 3)
            rows += out
            del fams
            torch.cuda.empty_cache()
    finally:
        set_served_arch(prev)
    return rows


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--shape", default="both", choices=["A", "B", "both"])
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--topk", type=float, default=0.1)
    ap.add_argument("--dtype", default="bf16", choices=sorted(DTYPES))
    ap.add_argument("--baseline-lib", default=None,
                    help="another libtdb200.so with the same C ABI: time it against this tree's build and compare the outputs")
    ap.add_argument("--ranks", default=None,
                    help="comma-separated world sizes, e.g. 1,2,4,8: time rank 0's share of a sequence-parallel layer instead")
    args = ap.parse_args()
    ranks = None
    if args.ranks is not None:
        ranks = [int(n) for n in args.ranks.split(",")]
        if not ranks or min(ranks) < 1:
            raise SystemExit("--ranks: positive world sizes, e.g. 1,2,4,8")
    if not torch.cuda.is_available():
        raise SystemExit("sla_block_families.py measures on a CUDA device; none is available")
    if args.iters < 50:
        raise SystemExit("--iters: the medians are taken over at least 50 calls")
    if args.baseline_lib is not None:
        from turbodiffusion_b200 import _lib
        print(json.dumps({**device_info(), "builds": {"this": _lib.LIB_PATH, "baseline": os.path.abspath(args.baseline_lib)}}),
              flush=True)
        identical = True
        for name in (["A", "B"] if args.shape == "both" else [args.shape]):
            rows, same = run_builds(name, args.topk, args.iters, args.warmup, os.path.abspath(args.baseline_lib),
                                    DTYPES[args.dtype])
            identical &= same
            for row in rows:
                print(json.dumps(row), flush=True)
        if not identical:
            raise SystemExit("the two builds' outputs differ")
        return
    print(json.dumps(device_info()), flush=True)
    for name in (["A", "B"] if args.shape == "both" else [args.shape]):
        rows = run_shape(name, args.topk, args.iters, args.warmup, DTYPES[args.dtype]) if ranks is None else \
            run_ranks(name, args.topk, args.iters, args.warmup, ranks, DTYPES[args.dtype])
        for row in rows:
            print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
