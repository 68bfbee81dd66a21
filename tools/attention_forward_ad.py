"""Time the attention operators' forward-AD rules on one GPU, bf16: the lse forward plus the tangent kernel
(tdb200_attn_dense_tangent, tdb200_sla_attn16_tangent) against the fused JVP kernel on the same inputs.

    python tools/attention_forward_ad.py [--iters 50] [--warmup 5] [--only NAME]

Shapes (query tokens x key tokens, heads x head dim; top-k ratio of the 64-key blocks for SLA):
  A-cross    32760 x 512,   12 x 128   Wan2.1-1.3B at 480p, cross-attention over the text tokens
  B-cross    75600 x 512,   40 x 128   Wan2.1-14B at 720p, cross-attention
  C-512      28672 x 512,   32 x 128   LTX shape C's video stream, text keys padded
  C-226      28672 x 226,   32 x 128   the same over the 226 text tokens
  A-self     32760 x 32760, 12 x 128   dense self-attention at shape A
  A-sla      32760, 12 x 128, top-k 0.1 and 0.15   SparseLinearAttention's sparse branch at shape A
  B-sla      75600, 40 x 128, top-k 0.1 and 0.15   the same at shape B
Legs: "fused_jvp" (tdb200_attn_dense_jvp / tdb200_sla_attn16_jvp: out and out_t from one kernel); "fwd_lse" and "tangent"
(the two kernels of the forward-AD rule, timed separately) and "fwd_lse_plus_tangent" (both, back to back); "func_jvp"
(torch.func.jvp through ops.dense_attention, or through the sparse branch's autograd Function with the LUT fixed, so that the
legs compare the same work).  The SLA LUT is random distinct key blocks per query block, ascending.
Per row, in one process: every leg warmed up, then --iters rounds of one CUDA-event-timed call of each leg, alternating;
median, minimum, maximum and the 10th / 90th percentiles.  TFLOP/s count 4 * B * H * Lq * Lk * D for the forward,
10 * B * H * Lq * Lk * D for the tangent kernel (five products) and 12 * B * H * Lq * Lk * D for the fused JVP (Lk the keys a
query row visits: topk * 64 for SLA).  The ratios to the fused JVP's median are the result.  One JSON line with the device name,
power limit and maximum SM clock, then one per row with the SM clock and throttle reasons read before and after its timed
window.  There is no CPU timing: without a CUDA device the script exits with an error."""
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
SHAPES = {"A-cross": (32760, 512, 12, None), "B-cross": (75600, 512, 40, None), "C-512": (28672, 512, 32, None),
          "C-226": (28672, 226, 32, None), "A-self": (32760, 32760, 12, None), "A-sla": (32760, 32760, 12, (0.1, 0.15)),
          "B-sla": (75600, 75600, 40, (0.1, 0.15))}


def _lut(h, l, topk, seed):
    mblk, nblk = (l + BLKQ - 1) // BLKQ, (l + BLKK - 1) // BLKK
    g = torch.Generator(device="cuda").manual_seed(seed)
    ids = torch.rand(h * mblk, nblk, device="cuda", generator=g).argsort(-1)[:, :topk].sort(-1).values
    return ids.view(1, h, mblk, topk).int().contiguous()


def _call(name, *args):
    from turbodiffusion_b200 import _lib
    _lib.check(getattr(_lib.lib(), "tdb200_" + name)(*args), name)


def dense_legs(q, k, v, q_t, k_t, v_t):
    from turbodiffusion_b200 import ops
    from turbodiffusion_b200._lib import stream_ptr
    b, lq, h, _ = q.shape
    lk, sm, st = k.shape[1], D ** -0.5, stream_ptr(q.device)
    out, out_t, f_out, f_out_t = (torch.empty_like(q) for _ in range(4))
    lse = torch.empty(b, h, lq, dtype=torch.float32, device="cuda")
    p = [t.data_ptr() for t in (q, k, v, q_t, k_t, v_t)]
    fwd = lambda: _call("attn_dense_fwd_lse", *p[:3], 0, out.data_ptr(), lse.data_ptr(), b, lq, lk, h, D, sm, st)
    tangent = lambda: _call("attn_dense_tangent", *p, out.data_ptr(), lse.data_ptr(), 0, out_t.data_ptr(), b, lq, lk, h, D, sm, st)
    fused = lambda: _call("attn_dense_jvp", *p, 0, f_out.data_ptr(), f_out_t.data_ptr(), b, lq, lk, h, D, sm, st)
    fwd()
    return {"fused_jvp": fused, "fwd_lse": fwd, "tangent": tangent, "fwd_lse_plus_tangent": lambda: (fwd(), tangent()),
            "func_jvp": lambda: torch.func.jvp(ops.dense_attention, (q, k, v), (q_t, k_t, v_t))}, lk


def sla_legs(q, k, v, q_t, k_t, v_t, ratio):
    from turbodiffusion_b200._lib import stream_ptr
    from turbodiffusion_b200.SLA.core import _SparseAttention16AD, attn_fwd_qk16_lse, attn_jvp_qk16
    from turbodiffusion_b200.SLA import core
    b, l, h, _ = q.shape
    nblk = (l + BLKK - 1) // BLKK
    topk, sm, st = int(ratio * nblk), D ** -0.5, stream_ptr(q.device)
    lut = _lut(h, l, topk, seed=1)
    o_s, lse = attn_fwd_qk16_lse(q, k, v, lut, topk, sm)
    o_s_t = torch.empty_like(q)
    p = [t.data_ptr() for t in (q, k, v, q_t, k_t, v_t)]
    tangent = lambda: _call("sla_attn16_tangent", *p, o_s.data_ptr(), lse.data_ptr(), 0, lut.data_ptr(), topk, o_s_t.data_ptr(),
                            b, l, h, D, sm, BLKQ, BLKK, st)
    fwd = lambda: attn_fwd_qk16_lse(q, k, v, lut, topk, sm)

    class _Prep:     # the LUT above stands in for block selection, so every leg runs the same key blocks
        q_pool = k_pool = None
    select, block_map = core.select_prep, core.block_map_from_pools

    def func_jvp():
        core.select_prep, core.block_map_from_pools = (lambda *a: _Prep()), (lambda *a: (None, lut))
        try:
            return torch.func.jvp(lambda a, b_, c: _SparseAttention16AD.apply(a, b_, c, topk, sm, None)[0], (q, k, v), (q_t, k_t, v_t))
        finally:
            core.select_prep, core.block_map_from_pools = select, block_map
    return {"fused_jvp": lambda: attn_jvp_qk16(q, k, v, q_t, k_t, v_t, lut, topk, sm), "fwd_lse": fwd, "tangent": tangent,
            "fwd_lse_plus_tangent": lambda: (fwd(), tangent()), "func_jvp": func_jvp}, topk * BLKK


def run_row(name, ratio, iters, warmup):
    lq, lk, h, _ = SHAPES[name]
    g = torch.Generator(device="cuda").manual_seed(0)
    q, q_t = (torch.randn(1, lq, h, D, device="cuda", generator=g).bfloat16() for _ in range(2))
    k, v, k_t, v_t = (torch.randn(1, lk, h, D, device="cuda", generator=g).bfloat16() for _ in range(4))
    legs, keys = sla_legs(q, k, v, q_t, k_t, v_t, ratio) if ratio else dense_legs(q, k, v, q_t, k_t, v_t)
    unit = h * lq * keys * D
    flop = {"fused_jvp": 12 * unit, "fwd_lse": 4 * unit, "tangent": 10 * unit, "fwd_lse_plus_tangent": 14 * unit,
            "func_jvp": 14 * unit}
    row = {"shape": name, "Lq": lq, "Lk": lk, "keys_per_row": keys, "heads": h, "head_dim": D, "dtype": "bf16"}
    if ratio:
        row["topk_ratio"] = ratio
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
        row[n] = _spread(times[n], flop[n])
    for n in ("fwd_lse_plus_tangent", "func_jvp", "tangent"):
        row[f"{n}_over_fused_jvp"] = round(row[n]["median_ms"] / row["fused_jvp"]["median_ms"], 4)
    row["calls_per_leg"] = iters
    return row


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--only", choices=tuple(SHAPES), default=None)
    args = ap.parse_args()
    if args.iters < 50:
        ap.error("--iters: at least 50 timed calls per leg")
    if not torch.cuda.is_available():
        raise SystemExit("attention_forward_ad.py measures on the GPU; no CUDA device found")
    print(json.dumps({**device_info(), "torch": torch.__version__}), flush=True)
    for name in ((args.only,) if args.only else SHAPES):
        for ratio in SHAPES[name][3] or (None,):
            print(json.dumps(run_row(name, ratio, args.iters, args.warmup)), flush=True)
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
