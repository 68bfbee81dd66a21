"""What SageSLA's FP8 P.V option (SLA.utils.set_sage_pv("fp8")) costs and saves against the 16-bit P.V, on one GPU.

    python tools/sla_fp8_pv.py [--shape A|B|both] [--iters 20] [--warmup 5] [--topk 0.1] [--rows 256]

For each shape (A: L = 32760, 12 heads; B: L = 75600, 40 heads; d = 128), both SageSLA block families ((128, 64) "sm100" and
(64, 128) "sm90") and both 16-bit dtypes, five legs are timed with CUDA events, call by call, in an order that rotates every
iteration: the V pass (tdb200_sla_quant_v_fp8), the fused attention with 16-bit V and with e4m3 V (each on the same prep, LUT
and moments; the e4m3 leg on codes made once), and the whole SageSparseLinearAttention forward under "bf16" and "fp8".
Reported per leg: median, 10th and 90th percentile in ms.  Accuracy: rel-L2 and cosine of both forwards against float64
SageSLA (sparse branch on the kernel's own block map, plus the linear branch and proj_l) on `--rows` sampled query rows of
four heads.  One JSON line per (shape, family, dtype), preceded by one with the device name, power limit and SM clock, and
followed by one with the SM clock read again.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = {"A": (32760, 12), "B": (75600, 40)}
FAMILIES = {"sm100": (128, 64), "sm90": (64, 128)}


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks_throttle_reasons.active"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as ex:  # noqa: BLE001
        return f"nvidia-smi unavailable: {ex}"


def pct(ts, p):
    ts = sorted(ts)
    return ts[min(len(ts) - 1, int(round(p / 100 * (len(ts) - 1))))]


def sampled_reference(q, k, v, lut, blkq, blkk, mod, rows, heads):
    """float64 SageSLA (softmax feature map) at `rows` of `heads`: [len(heads) * len(rows), d]."""
    l = q.shape[1]
    w, b = mod.proj_l.weight.detach().double(), mod.proj_l.bias.detach().double()
    out = []
    for head in heads:
        qh, kh, vh = (t[0, :, head].double() for t in (q, k, v))
        s = (qh[rows] @ kh.t()) * qh.shape[-1] ** -0.5
        mask = torch.zeros(len(rows), (l + blkk - 1) // blkk, dtype=torch.bool, device=q.device)
        mask.scatter_(-1, lut[0, head, rows // blkq].long(), True)
        s = s.masked_fill(~mask.repeat_interleave(blkk, 1)[:, :l], float("-inf"))
        pq, pk = torch.softmax(qh[rows], -1), torch.softmax(kh, -1)
        o_l = (pq @ (pk.t() @ vh)) / (1e-5 + pq @ pk.sum(0))[:, None]
        out.append(torch.softmax(s, -1) @ vh + o_l @ w.t() + b)
    return torch.cat(out)


def stats(a, ref):
    a, ref = a.double().flatten(), ref.flatten()
    return {"rel_l2": float((a - ref).norm() / ref.norm()), "cos": float(a @ ref / (a.norm() * ref.norm()))}


def run(shape, family, dtype, args, dev):
    from turbodiffusion_b200 import _ops
    from turbodiffusion_b200.SLA import SageSparseLinearAttention, core, utils
    l, h = SHAPES[shape]
    blkq, blkk = FAMILIES[family]
    utils.set_served_arch(family)
    g = torch.Generator(device=dev).manual_seed(l + h)
    q, k, v = (torch.randn(1, l, h, 128, generator=g, device=dev).to(dtype) for _ in range(3))
    k += (torch.randn(1, 1, h, 128, generator=g, device=dev) * 2).to(dtype)
    mod = SageSparseLinearAttention(128, args.topk, use_bf16=dtype == torch.bfloat16).to(dev)
    with torch.no_grad():
        mod.proj_l.weight.normal_(0, 0.05, generator=g)
        mod.proj_l.bias.normal_(0, 0.05, generator=g)
    prep = utils.quant_qk(q, k, blkq=blkq, blkk=blkk)
    topk = max(1, min(prep.nblk, int(args.topk * prep.nblk)))
    _, lut = utils.block_map_from_pools(prep.q_pool, prep.k_pool, topk)
    kv, ksum = core.linear_moments(k, v, 0)
    kvw = core.project_moments(mod.proj_l.weight.detach(), kv, dtype)
    pb = mod.proj_l.bias.detach().float().contiguous()
    v_fp8, v_scale = _ops.sla_quant_v_fp8(v, l, blkk)

    def fwd(mode):
        utils.set_sage_pv(mode)
        return mod(q, k, v)

    legs = {
        "v_prep": lambda: _ops.sla_quant_v_fp8(v, l, blkk),
        "attn_bf16v": lambda: _ops.sla_attn_fwd(prep.q_i8, prep.q_scale, prep.k_i8, prep.k_scale, v, q, lut, topk, kvw, ksum, pb,
                                                128 ** -0.5, l, 0, blkq, blkk, False),
        "attn_fp8v": lambda: _ops.sla_attn_fwd_fp8v(prep.q_i8, prep.q_scale, prep.k_i8, prep.k_scale, v_fp8, v_scale, q, lut, topk,
                                                    kvw, ksum, pb, 128 ** -0.5, l, 0, blkq, blkk, False),
        "forward_bf16": lambda: fwd("bf16"),
        "forward_fp8": lambda: fwd("fp8"),
    }
    names = list(legs)
    times = {n: [] for n in names}
    for it in range(args.warmup + args.iters):
        order = names[it % len(names):] + names[:it % len(names)]
        for n in order:
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            legs[n]()
            e.record()
            torch.cuda.synchronize()
            if it >= args.warmup:
                times[n].append(s.elapsed_time(e))
    utils.set_sage_pv("bf16")
    out = {"shape": shape, "L": l, "H": h, "family": family, "blocks": [blkq, blkk], "dtype": str(dtype).split(".")[-1],
           "topk": topk, "iters": args.iters}
    for n in names:
        out[n + "_ms"] = {"median": round(pct(times[n], 50), 4), "p10": round(pct(times[n], 10), 4), "p90": round(pct(times[n], 90), 4)}
    gen = torch.Generator().manual_seed(l)
    rows = torch.cat([torch.arange(16), torch.randint(16, l - 16, (args.rows - 32,), generator=gen), torch.arange(l - 16, l)]).to(dev)
    heads = sorted({0, h // 3, 2 * h // 3, h - 1})
    mod._keep_selection = {}
    for mode in ("bf16", "fp8"):
        utils.set_sage_pv(mode)
        o = mod(q, k, v)
        ref = sampled_reference(q, k, v, mod._keep_selection["lut"], blkq, blkk, mod, rows, heads)
        out["accuracy_" + mode] = stats(torch.cat([o[0, rows, hh] for hh in heads]), ref)
    mod._keep_selection = None
    utils.set_sage_pv("bf16")
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shape", default="both", choices=["A", "B", "both"])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--topk", type=float, default=0.1)
    ap.add_argument("--rows", type=int, default=256)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("sla_fp8_pv.py measures on a CUDA device; none is visible")
    dev = torch.device("cuda:0")
    print(json.dumps({"device": torch.cuda.get_device_name(0), "nvidia_smi": gpu_info()}), flush=True)
    with torch.no_grad():
        for shape in (["A", "B"] if args.shape == "both" else [args.shape]):
            for family in FAMILIES:
                for dtype in (torch.bfloat16, torch.float16):
                    print(json.dumps(run(shape, family, dtype, args, dev)), flush=True)
    print(json.dumps({"nvidia_smi_after": gpu_info()}), flush=True)


if __name__ == "__main__":
    main()
