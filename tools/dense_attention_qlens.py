"""Time the dense attention operators with per-sample query lengths (ops.dense_attention / ops.dense_attention_jvp with q_lens,
the _vl entry points) on one GPU, bf16, batch 2: self-attention over a padded batch, and a cross-attention whose queries and
keys are both padded.

    python tools/dense_attention_qlens.py [--iters 50] [--warmup 3] [--reps 1]

Shapes (padded queries x padded keys, heads x head dim; query lengths; key lengths):
  Wan-self   32760 x 32760, 12 x 128; (32760, 20280); the same   two Wan2.1-1.3B 480p clips of 81 and 49 frames
  C-self     28672 x 28672, 32 x 128; (28672, 16384); the same   LTX shape C's video stream at two clip lengths
  A-cross    32760 x 512,   12 x 128; (32760, 20280); (512, 226) shape A's cross-attention over the same pair of clips
Legs, per operation (fwd: forward without grad; jvp: output and tangent without grad; fwd+bwd: forward with grad and the
backward of one incoming gradient, zero in the padded query rows):
  vl        one call on the padded batch with q_lens and k_lens
  padded    one call with k_lens only, the padded query rows computed: what a caller can do without q_lens
  trimmed   one call per sample on q, k and v cut to its lengths
  sdpa      F.scaled_dot_product_attention with the boolean key-padding mask [2, 1, 1, Lk], padded query rows computed (fwd and
            fwd+bwd; it has no JVP)
Per shape, in one process: every leg warmed up, then --iters rounds in which each leg, in an order shuffled per round, is timed
with CUDA events over --reps back-to-back calls (per-call time = the window over --reps; these calls take milliseconds, so one
call per window already amortises the host's wake-up that dense_attention_klens.py spreads over five).  Median and 10th / 90th
percentiles per leg, and vl / trimmed, vl / padded and the shape's sum(lq_i * lk_i) / sum(lq * lk_i), the share of the padded
call's work that the vl call keeps.  One JSON line with the device name, power limit and maximum SM clock, then one per shape
with the SM clock and throttle reasons read before and after its timed window.  There is no CPU timing: without a CUDA device
the script exits with an error."""
from __future__ import annotations

import argparse
import json
import os
import random
import statistics
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from sla_block_families import _pct, _timed, clock_state, device_info  # noqa: E402

D = 128
# name: (lq, lk, heads, query lengths, key lengths)
SHAPES = {
    "Wan-self": (32760, 32760, 12, (32760, 20280), (32760, 20280)),
    "C-self": (28672, 28672, 32, (28672, 16384), (28672, 16384)),
    "A-cross": (32760, 512, 12, (32760, 20280), (512, 226)),
}


def _spread(ms):
    return {"median_ms": round(statistics.median(ms), 4), "p10_ms": round(_pct(ms, 0.1), 4), "p90_ms": round(_pct(ms, 0.9), 4)}


def legs_for(lq, lk, h, q_lens, k_lens):
    from turbodiffusion_b200 import ops
    b = len(q_lens)
    g = torch.Generator(device="cuda").manual_seed(0)
    q, q_t, d_out = (torch.randn(b, lq, h, D, device="cuda", generator=g).bfloat16() for _ in range(3))
    k, v, k_t, v_t = (torch.randn(b, lk, h, D, device="cuda", generator=g).bfloat16() for _ in range(4))
    for i, n in enumerate(q_lens):
        d_out[i, n:] = 0
    ql = torch.tensor(q_lens, dtype=torch.int32, device="cuda")
    kl = torch.tensor(k_lens, dtype=torch.int32, device="cuda")
    mask = (torch.arange(lk, device="cuda")[None, :] < kl[:, None])[:, None, None, :]
    per = [tuple(t[i:i + 1, :n].contiguous() for t in (q, q_t, d_out)) + tuple(t[i:i + 1, :m].contiguous() for t in (k, v, k_t, v_t))
           for i, (n, m) in enumerate(zip(q_lens, k_lens))]
    leaves = [t.clone().requires_grad_() for t in (q, k, v)]
    leaves_i = [[t.clone().requires_grad_() for t in (p[0], p[3], p[4])] for p in per]

    def backward(out, ls, grad):   # fresh gradients every call
        for t in ls:
            t.grad = None
        out.backward(grad)

    def sdpa(q_, k_, v_):
        return F.scaled_dot_product_attention(q_.transpose(1, 2), k_.transpose(1, 2), v_.transpose(1, 2), attn_mask=mask,
                                              scale=D ** -0.5).transpose(1, 2)

    def fwd_trimmed():
        for p in per:
            ops.dense_attention(p[0], p[3], p[4])

    def jvp_trimmed():
        for p in per:
            ops.dense_attention_jvp(p[0], p[3], p[4], p[1], p[5], p[6])

    def train_trimmed():
        for p, ls in zip(per, leaves_i):
            backward(ops.dense_attention(*ls), ls, p[2])

    return {
        "fwd": {"vl": lambda: ops.dense_attention(q, k, v, q_lens=ql, k_lens=kl),
                "padded": lambda: ops.dense_attention(q, k, v, k_lens=kl), "trimmed": fwd_trimmed, "sdpa": lambda: sdpa(q, k, v)},
        "jvp": {"vl": lambda: ops.dense_attention_jvp(q, k, v, q_t, k_t, v_t, q_lens=ql, k_lens=kl),
                "padded": lambda: ops.dense_attention_jvp(q, k, v, q_t, k_t, v_t, k_lens=kl), "trimmed": jvp_trimmed},
        "fwd+bwd": {"vl": lambda: backward(ops.dense_attention(*leaves, q_lens=ql, k_lens=kl), leaves, d_out),
                    "padded": lambda: backward(ops.dense_attention(*leaves, k_lens=kl), leaves, d_out),
                    "trimmed": train_trimmed, "sdpa": lambda: backward(sdpa(*leaves), leaves, d_out)},
    }


def run(name, iters, warmup, reps):
    lq, lk, h, q_lens, k_lens = SHAPES[name]
    ops_legs = legs_for(lq, lk, h, q_lens, k_lens)
    legs = {f"{op} {leg}": fn for op, d in ops_legs.items() for leg, fn in d.items()}
    for _ in range(warmup):
        for fn in legs.values():
            fn()
    torch.cuda.synchronize()
    work = sum(n * m for n, m in zip(q_lens, k_lens)) / sum(lq * m for m in k_lens)
    row = {"shape": name, "Lq_padded": lq, "Lk_padded": lk, "q_lens": list(q_lens), "k_lens": list(k_lens), "heads": h,
           "head_dim": D, "dtype": "bf16", "batch": len(q_lens), "work_vl_over_padded": round(work, 4),
           "sm_clock_throttle_before": clock_state()}
    names = list(legs)
    times = {n: [] for n in names}
    rng = random.Random(0)

    def repeated(fn):
        return lambda: [fn() for _ in range(reps)]

    for _ in range(iters):
        rng.shuffle(names)
        for n in names:
            times[n].append(_timed(repeated(legs[n])) / reps)
    row["sm_clock_throttle_after"] = clock_state()
    for op, d in ops_legs.items():
        row[op] = {leg: _spread(times[f"{op} {leg}"]) for leg in d}
        vl = row[op]["vl"]["median_ms"]
        row[op]["vl_over_trimmed"] = round(vl / row[op]["trimmed"]["median_ms"], 3)
        row[op]["vl_over_padded"] = round(vl / row[op]["padded"]["median_ms"], 3)
        if "sdpa" in d:
            row[op]["sdpa_over_vl"] = round(row[op]["sdpa"]["median_ms"] / vl, 3)
    row["timed_windows_per_leg"], row["calls_per_window"] = iters, reps
    return row


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=1, help="back-to-back calls per timed window")
    args = ap.parse_args()
    if args.iters < 50:
        ap.error("--iters: at least 50 timed calls per leg")
    if not torch.cuda.is_available():
        raise SystemExit("dense_attention_qlens.py measures on the GPU; no CUDA device found")
    print(json.dumps({**device_info(), "torch": torch.__version__}), flush=True)
    for name in SHAPES:
        print(json.dumps(run(name, args.iters, args.warmup, args.reps)), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
