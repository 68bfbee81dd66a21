"""Time the sparse attention JVP (tdb200_sla_attn16_jvp, SparseLinearAttention.forward_jvp) on one GPU, bf16 (or fp16 with
--dtype fp16), against the sparse forward and the dense JVP on the same inputs, at the shapes the models run sparse attention at.

    python tools/sla_jvp.py [--iters 50] [--warmup 5] [--only NAME] [--dtype bf16|fp16]

Shapes (tokens, heads x head dim, top-k ratio of the 64-key blocks):
  A   32760, 12 x 128, 0.1 and 0.15   Wan2.1-1.3B at 480p (51 and 76 of 512 key blocks)
  B   75600, 40 x 128, 0.1 and 0.15   Wan2.1-14B at 720p (118 and 177 of 1182 key blocks)
  C   28672, 32 x 128, 0.3            LTX shape C's video stream (134 of 448 key blocks)
Legs: the sparse JVP (attn_jvp_qk16, o_s and o_s_t); the sparse forward with lse (tdb200_sla_attn16_fwd_lse, o_s alone) on
the same LUT; the dense JVP (ops.dense_attention_jvp) on the same q, k, v and tangents, once per shape (it does not depend on
top-k); SparseLinearAttention.forward_jvp without grad, with grad, and with grad followed by the backward of o.sum().  The LUT
is random distinct key blocks per query block, ascending (the order block selection produces).
Per row, in one process: every leg warmed up, then --iters rounds of one CUDA-event-timed call of each leg, alternating;
median, minimum, maximum and the 10th / 90th percentiles per leg.  TFLOP/s count 12 * B * H * Mblk * topk * 128 * 64 * D for the
sparse JVP (12 * B * H * L * L * D for the dense JVP, 4 * B * H * Mblk * topk * 128 * 64 * D for the sparse forward), with the
share of the H100 SXM data sheet's 989 TFLOP/s (dense bf16, a 700 W figure, not a rate reached here).  The ratio of the sparse
JVP's median to the dense JVP's, next to topk / nblk, says what the per-CTA fixed cost adds.  One JSON line with the device
name, power limit and maximum SM clock, then one per row with the SM clock and throttle reasons read before and after its
timed window.  There is no CPU timing: without a CUDA device the script exits with an error."""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from dense_attention import _spread  # noqa: E402
from sla_block_families import _timed, clock_state, device_info  # noqa: E402

D, BLKQ, BLKK = 128, 128, 64
SHAPES = {"A": (32760, 12, (0.1, 0.15)), "B": (75600, 40, (0.1, 0.15)), "C": (28672, 32, (0.3,))}


def _lut(h, l, topk, seed):
    mblk, nblk = (l + BLKQ - 1) // BLKQ, (l + BLKK - 1) // BLKK
    g = torch.Generator(device="cuda").manual_seed(seed)
    ids = torch.rand(h * mblk, nblk, device="cuda", generator=g).argsort(-1)[:, :topk].sort(-1).values
    return ids.view(1, h, mblk, topk).int().contiguous()


def run_row(name, ratio, with_dense, iters, warmup, dtype="bf16"):
    from turbodiffusion_b200 import ops
    from turbodiffusion_b200.SLA import SparseLinearAttention
    from turbodiffusion_b200.SLA.core import attn_fwd_qk16_lse, attn_jvp_qk16
    l, h, _ = SHAPES[name]
    mblk, nblk = (l + BLKQ - 1) // BLKQ, (l + BLKK - 1) // BLKK
    topk = int(ratio * nblk)
    g = torch.Generator(device="cuda").manual_seed(0)
    dt = {"bf16": torch.bfloat16, "fp16": torch.float16}[dtype]
    q, k, v, q_t, k_t, v_t = (torch.randn(1, l, h, D, device="cuda", generator=g).to(dt) for _ in range(6))
    lut = _lut(h, l, topk, seed=1)
    sm = D ** -0.5
    mod = SparseLinearAttention(D, ratio, BLKQ=BLKQ, BLKK=BLKK, use_bf16=dtype == "bf16").cuda()
    with torch.no_grad():
        mod.proj_l.weight.normal_(0, 0.05)
        mod.proj_l.bias.normal_(0, 0.05)
    qg, kg, vg = (t.clone().requires_grad_() for t in (q, k, v))

    def jvp_nograd():
        with torch.no_grad():
            return mod.forward_jvp(q, k, v, q_t, k_t, v_t)

    def jvp_grad_backward():
        qg.grad = kg.grad = vg.grad = None
        o, _ = mod.forward_jvp(qg, kg, vg, q_t, k_t, v_t)
        o.float().sum().backward()

    def sla_fwd_lse():
        with torch.no_grad():
            return attn_fwd_qk16_lse(q, k, v, lut, topk, sm)

    legs = {"sla_jvp": lambda: attn_jvp_qk16(q, k, v, q_t, k_t, v_t, lut, topk, sm),
            "sla_fwd_lse": sla_fwd_lse,
            "forward_jvp_no_grad": jvp_nograd,
            "forward_jvp_grad": lambda: mod.forward_jvp(qg, kg, vg, q_t, k_t, v_t),
            "forward_jvp_grad_and_backward": jvp_grad_backward}
    if with_dense:
        legs["dense_jvp"] = lambda: ops.dense_attention_jvp(q, k, v, q_t, k_t, v_t, sm)
    sparse_flop = h * mblk * topk * BLKQ * BLKK * D
    flop = {"sla_jvp": 12 * sparse_flop, "sla_fwd_lse": 4 * sparse_flop, "dense_jvp": 12 * h * l * l * D}
    row = {"shape": name, "L": l, "heads": h, "head_dim": D, "dtype": dtype, "topk_ratio": ratio, "topk": topk, "nblk": nblk,
           "topk_over_nblk": round(topk / nblk, 4)}
    for _ in range(warmup):
        for fn in legs.values():
            fn()
    torch.cuda.synchronize()
    row["sm_clock_throttle_before"] = clock_state()
    times = {n: [] for n in legs}
    for _ in range(iters):
        for n, fn in legs.items():
            times[n].append(_timed(fn))
    row["sm_clock_throttle_after"] = clock_state()
    for n in legs:
        row[n] = _spread(times[n], flop[n]) if n in flop else {k: v for k, v in _spread(times[n], 1).items() if k.endswith("_ms")}
    if with_dense:
        row["sla_jvp_over_dense_jvp"] = round(row["sla_jvp"]["median_ms"] / row["dense_jvp"]["median_ms"], 4)
    row["sla_jvp_over_sla_fwd_lse"] = round(row["sla_jvp"]["median_ms"] / row["sla_fwd_lse"]["median_ms"], 4)
    row["calls_per_leg"] = iters
    return row


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--only", choices=tuple(SHAPES), default=None)
    ap.add_argument("--dtype", choices=("bf16", "fp16"), default="bf16")
    args = ap.parse_args()
    if args.iters < 50:
        ap.error("--iters: at least 50 timed calls per leg")
    if not torch.cuda.is_available():
        raise SystemExit("sla_jvp.py measures on the GPU; no CUDA device found")
    print(json.dumps({**device_info(), "torch": torch.__version__}), flush=True)
    for name in ((args.only,) if args.only else SHAPES):
        for i, ratio in enumerate(SHAPES[name][2]):
            print(json.dumps(run_row(name, ratio, i == 0, args.iters, args.warmup, args.dtype)), flush=True)
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
