"""Time the SLA modules with per-entry lengths (forward(..., seq_lens=...), the _vl entry points) on one GPU, bf16, batch 2,
inference (no grad), topk ratio 0.1 (bench.py's).

    python tools/sla_seq_lens.py [--iters 50] [--warmup 3]

Pairs (padded L, heads x 128; lengths):
  Wan-A   32760, 12; (32760, 20280)   two Wan2.1-1.3B 480p clips of 81 and 49 frames (bench.py shape A)
  Wan-B   75600, 40; (75600, 46800)   two Wan2.1-14B 720p clips of 81 and 49 frames (bench.py shape B)
Modules: SageSparseLinearAttention (the default (BLKQ, BLKK) = (128, 64)) and SparseLinearAttention(BLKQ=128, BLKK=64).
Legs, per module:
  vl        one call on the padded pair with seq_lens
  trimmed   one call per entry on q, k and v cut to its length: what a caller had to do before
  padded    one call on the padded pair without lengths: wrong for the shorter entry, the cost floor of one launch per kernel
Per pair and module, in one process: every leg warmed up, then --iters rounds in which each leg, in an order shuffled per round,
is timed with CUDA events over one call.  Median and 10th / 90th percentiles per leg, vl / trimmed and vl / padded, and the
work ratio sum_i mblk_i * topk_i / (B * mblk * topk) of the sparse attention, counted from the shapes with the modules' rule
(topk_i = max(1, min(nblk_i, int(0.1 * nblk_i)))).  One JSON line with the device name, power limit and maximum SM clock, then
one per pair and module with the SM clock and throttle reasons read before and after its timed window.  There is no CPU timing:
without a CUDA device the script exits with an error."""
from __future__ import annotations

import argparse
import json
import os
import random
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from sla_block_families import _pct, _timed, clock_state, device_info  # noqa: E402

D = 128
RATIO = 0.1
PAIRS = {"Wan-A": (32760, 12, (32760, 20280)), "Wan-B": (75600, 40, (75600, 46800))}


def _spread(ms):
    return {"median_ms": round(statistics.median(ms), 4), "p10_ms": round(_pct(ms, 0.1), 4), "p90_ms": round(_pct(ms, 0.9), 4)}


def _cdiv(a, b):
    return (a + b - 1) // b


def _topk(n, blkk):
    nblk = _cdiv(n, blkk)
    return max(1, min(nblk, int(RATIO * nblk)))


def work_ratio(l, lens, blkq, blkk):
    """sum_i mblk_i * topk_i / (B * mblk * topk): the share of the padded call's (query block, key block) products the vl call keeps."""
    return sum(_cdiv(n, blkq) * _topk(n, blkk) for n in lens) / (len(lens) * _cdiv(l, blkq) * _topk(l, blkk))


def modules():
    from turbodiffusion_b200.SLA import SageSparseLinearAttention, SparseLinearAttention
    g = torch.Generator().manual_seed(0)
    out = {"SageSLA": SageSparseLinearAttention(D, RATIO), "SLA": SparseLinearAttention(D, RATIO, BLKQ=128, BLKK=64)}
    for m in out.values():
        with torch.no_grad():   # a live linear branch: proj_l is zero-initialised
            m.proj_l.weight.copy_(torch.randn(D, D, generator=g) * 0.05)
            m.proj_l.bias.copy_(torch.randn(D, generator=g) * 0.05)
        m.cuda()
    return out


def run(pair, name, mod, iters, warmup):
    l, h, lens = PAIRS[pair]
    g = torch.Generator(device="cuda").manual_seed(1)
    q, k, v = (torch.randn(len(lens), l, h, D, device="cuda", generator=g).bfloat16() for _ in range(3))
    per = [tuple(t[i:i + 1, :n].contiguous() for t in (q, k, v)) for i, n in enumerate(lens)]
    sl = torch.tensor(lens, dtype=torch.int32, device="cuda")

    def trimmed():
        for p in per:
            mod(*p)

    legs = {"vl": lambda: mod(q, k, v, seq_lens=sl), "trimmed": trimmed, "padded": lambda: mod(q, k, v)}
    with torch.no_grad():
        for _ in range(warmup):
            for fn in legs.values():
                fn()
        torch.cuda.synchronize()
        blkq, blkk = mod.block_sizes(q.device.index)
        row = {"pair": pair, "module": name, "L_padded": l, "lens": list(lens), "heads": h, "head_dim": D, "dtype": "bf16",
               "topk_ratio": RATIO, "blocks": [blkq, blkk], "work_vl_over_padded": round(work_ratio(l, lens, blkq, blkk), 4),
               "sm_clock_throttle_before": clock_state()}
        names = list(legs)
        times = {n: [] for n in names}
        rng = random.Random(0)
        for _ in range(iters):
            rng.shuffle(names)
            for n in names:
                times[n].append(_timed(legs[n]))
        row["sm_clock_throttle_after"] = clock_state()
    for n in legs:
        row[n] = _spread(times[n])
    vl = row["vl"]["median_ms"]
    row["vl_over_trimmed"] = round(vl / row["trimmed"]["median_ms"], 3)
    row["vl_over_padded"] = round(vl / row["padded"]["median_ms"], 3)
    row["timed_windows_per_leg"] = iters
    return row


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if args.iters < 50:
        ap.error("--iters: at least 50 timed calls per leg")
    if not torch.cuda.is_available():
        raise SystemExit("sla_seq_lens.py measures on the GPU; no CUDA device found")
    print(json.dumps({**device_info(), "torch": torch.__version__}), flush=True)
    mods = modules()
    for pair in PAIRS:
        for name, mod in mods.items():
            print(json.dumps(run(pair, name, mod, args.iters, args.warmup)), flush=True)
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
