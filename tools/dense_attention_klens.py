"""Time the dense attention operators with per-sample key lengths (ops.dense_attention / ops.dense_attention_jvp with k_lens,
the _kl entry points) on one GPU, bf16, batch 2: the batched text cross-attention of two prompts of different lengths.

    python tools/dense_attention_klens.py [--iters 50] [--warmup 5] [--reps 5]

Shapes (queries x padded keys, heads x head dim), each with key lengths (512, 226) and (512, 77):
  C-512     28672 x 512, 32 x 128   LTX shape C's video stream
  A-cross   32760 x 512, 12 x 128   Wan2.1-1.3B at 480p, cross-attention
Legs, per operation (fwd: forward without grad; jvp: output and tangent without grad; fwd+bwd: forward with grad and the
backward of one incoming gradient):
  klens     one call on the padded batch with k_lens
  trimmed   what a caller does without k_lens: one call per sample on its keys cut to its length
  sdpa      F.scaled_dot_product_attention with the boolean key-padding mask [2, 1, 1, 512] (fwd and fwd+bwd; it has no JVP)
Per shape and lengths, in one process: every leg warmed up, then --iters rounds in which each leg, in an order shuffled per
round, is timed with CUDA events over --reps back-to-back calls (per-call time = the window over --reps).  A leg timed right
after a long one pays the host's wake-up inside its first call, so a fixed order would charge it to whichever leg follows the
longest; shuffling spreads it and the back-to-back calls amortise it.  Median and 10th / 90th percentiles per leg.  One JSON
line with the device name, power limit and maximum SM clock, then one per (shape, lengths) with the SM clock and throttle
reasons read before and after its timed window.  There is no CPU timing: without a CUDA device the script exits with an
error."""
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
SHAPES = {"C-512": (28672, 512, 32), "A-cross": (32760, 512, 12)}
LENGTHS = ((512, 226), (512, 77))


def _spread(ms):
    return {"median_ms": round(statistics.median(ms), 4), "p10_ms": round(_pct(ms, 0.1), 4), "p90_ms": round(_pct(ms, 0.9), 4)}


def legs_for(lq, lk, h, lens):
    from turbodiffusion_b200 import ops
    b = len(lens)
    g = torch.Generator(device="cuda").manual_seed(0)
    q, q_t, d_out = (torch.randn(b, lq, h, D, device="cuda", generator=g).bfloat16() for _ in range(3))
    k, v, k_t, v_t = (torch.randn(b, lk, h, D, device="cuda", generator=g).bfloat16() for _ in range(4))
    k_lens = torch.tensor(lens, dtype=torch.int32, device="cuda")
    mask = (torch.arange(lk, device="cuda")[None, :] < k_lens[:, None])[:, None, None, :]
    per = [tuple(t[i:i + 1, :n].contiguous() for t in (k, v, k_t, v_t)) for i, n in enumerate(lens)]
    qs = [tuple(t[i:i + 1].contiguous() for t in (q, q_t, d_out)) for i in range(b)]
    leaves = [t.clone().requires_grad_() for t in (q, k, v)]
    leaves_i = [[t.clone().requires_grad_() for t in (qs[i][0], per[i][0], per[i][1])] for i in range(b)]

    def backward(out, ls, grad):   # fresh gradients every call
        for t in ls:
            t.grad = None
        out.backward(grad)

    def sdpa(q_, k_, v_):
        return F.scaled_dot_product_attention(q_.transpose(1, 2), k_.transpose(1, 2), v_.transpose(1, 2), attn_mask=mask,
                                              scale=D ** -0.5).transpose(1, 2)

    def fwd_trimmed():
        for i in range(b):
            ops.dense_attention(qs[i][0], per[i][0], per[i][1])

    def jvp_trimmed():
        for i in range(b):
            ops.dense_attention_jvp(qs[i][0], per[i][0], per[i][1], qs[i][1], per[i][2], per[i][3])

    def train_trimmed():
        for i in range(b):
            backward(ops.dense_attention(*leaves_i[i]), leaves_i[i], qs[i][2])

    return {
        "fwd": {"klens": lambda: ops.dense_attention(q, k, v, k_lens=k_lens), "trimmed": fwd_trimmed,
                "sdpa": lambda: sdpa(q, k, v)},
        "jvp": {"klens": lambda: ops.dense_attention_jvp(q, k, v, q_t, k_t, v_t, k_lens=k_lens), "trimmed": jvp_trimmed},
        "fwd+bwd": {"klens": lambda: backward(ops.dense_attention(*leaves, k_lens=k_lens), leaves, d_out),
                    "trimmed": train_trimmed, "sdpa": lambda: backward(sdpa(*leaves), leaves, d_out)},
    }


def run(name, lens, iters, warmup, reps):
    lq, lk, h = SHAPES[name]
    ops_legs = legs_for(lq, lk, h, lens)
    legs = {f"{op} {leg}": fn for op, d in ops_legs.items() for leg, fn in d.items()}
    for _ in range(warmup):
        for fn in legs.values():
            fn()
    torch.cuda.synchronize()
    row = {"shape": name, "Lq": lq, "Lk_padded": lk, "k_lens": list(lens), "heads": h, "head_dim": D, "dtype": "bf16",
           "batch": len(lens), "sm_clock_throttle_before": clock_state()}
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
        base = row[op]["klens"]["median_ms"]
        row[op]["trimmed_over_klens"] = round(row[op]["trimmed"]["median_ms"] / base, 3)
        if "sdpa" in d:
            row[op]["sdpa_over_klens"] = round(row[op]["sdpa"]["median_ms"] / base, 3)
    row["timed_windows_per_leg"], row["calls_per_window"] = iters, reps
    return row


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=5, help="back-to-back calls per timed window")
    args = ap.parse_args()
    if args.iters < 50:
        ap.error("--iters: at least 50 timed calls per leg")
    if not torch.cuda.is_available():
        raise SystemExit("dense_attention_klens.py measures on the GPU; no CUDA device found")
    print(json.dumps({**device_info(), "torch": torch.__version__}), flush=True)
    for name in SHAPES:
        for lens in LENGTHS:
            print(json.dumps(run(name, lens, args.iters, args.warmup, args.reps)), flush=True)
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
