"""Stage-by-stage checks of one Wan DiT block call (turbodiffusion_b200/block.py), shared by the GPU test
(test_gpu_block_stages.py) and its host test on a block chain built from the CPU oracle (test_block_stages_host.py).

A block call is recorded as a list of `Call`s: operator name, arguments, outputs.  `block_stages(cfg)` lists the operators
the block must call for a configuration, in order, and where each argument must come from: a block input (`x`, `e0`,
`angles`, `context`), a state-dict tensor (`sd:<key>`), a chunk of e = modulation[0] + e0 (`e.<i>`), or an earlier stage's
output.  `check_chain` holds a recording to that list bit for bit; `check_stage` holds one stage's recorded output to a
reference evaluated on the values the list names, with the bar of the operator's own unit test.  Because the references
read their inputs by name, a wiring fault (a swapped modulation chunk, the wrong norm weight, a permuted projection) can be
restated by changing the named values (`faults`), and the recorded output must then fail the stage's bar.

Everything here is plain torch on whatever device the tensors live on; the oracle functions run on CPU copies of sampled
128-row tiles (the first, a middle one and the ragged last one) with every column and every head.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Callable, Dict, List, Optional

import torch
import torch.nn.functional as F

from oracle import td_oracle as O

SKIP = object()   # an argument the chain does not check: the preallocated output of an in-place GEMM


@dataclass
class Call:
    name: str
    args: tuple
    kwargs: dict
    out: tuple


class Recorder:
    """Wraps callables so that every top-level call appends a Call (nested calls of wrapped names are not recorded)."""

    def __init__(self):
        self.calls: List[Call] = []
        self._depth = 0

    def wrap(self, name: str, fn: Callable, out_arg: Optional[int] = None) -> Callable:
        def wrapped(*args, **kwargs):
            if self._depth:
                return fn(*args, **kwargs)
            self._depth += 1
            try:
                res = fn(*args, **kwargs)
            finally:
                self._depth -= 1
            out = (args[out_arg],) if out_arg is not None else (tuple(res) if isinstance(res, (tuple, list)) else (res,))
            self.calls.append(Call(name, args, dict(kwargs), out))
            return res
        return wrapped


class AttentionRecorder:
    """A plain callable standing in for the block's attention module: records (q, k, v) -> o.  It has no `q_first`,
    `start_k` or `start_kv`, so the block takes its single-GPU path, and it is not an `attn_hook`, so FUSE_QKV="auto"
    keeps the fused q/k/v GEMM."""

    def __init__(self, rec: Recorder, fn: Callable):
        self.fn = rec.wrap("attention", fn)
        self.module = fn

    def __call__(self, q, k, v):
        return self.fn(q, k, v)


# ---------------------------------------------------------------------------------------------------- the stage list
@dataclass
class Stage:
    label: str
    op: str
    args: tuple               # argument sources: env key, (env key, view), or a literal compared with ==
    outs: tuple               # env keys bound to the outputs
    kind: str                 # reference and bar, see check_stage
    ref: tuple = ()           # env keys the reference reads
    proj: tuple = ()          # projections (state-dict prefixes) of a GEMM stage, one per output part
    kwargs: dict = field(default_factory=dict)


@dataclass
class Config:
    dim: int
    heads: int
    dtype: torch.dtype
    fused_qkv: bool
    fused_ckv: bool
    ffn: str = "fused"             # block.FFN_ACT_MODE
    stats_in: bool = False         # the block is handed the row statistics of x (WanHotPath, every block after the first)
    want_stats: bool = False       # the block returns the statistics of its output
    eps: float = 1e-6


def _gemm(label, a, proj, out, dt):
    return Stage(label, "gemm_cuda_swizzle_bias", (a + "q", a + "s", f"sd:{proj}.int8_weight", f"sd:{proj}.scale", SKIP,
                                                  f"sd:{proj}.bias"), (out,), "gemm", (a + "q", a + "s"), (proj,))


def block_stages(cfg: Config) -> List[Stage]:
    """The operators WanBlockB200.forward calls for `cfg`, in order, with the source of every argument."""
    dt, eps, h = cfg.dtype, cfg.eps, cfg.heads
    st: List[Stage] = []
    if cfg.stats_in:
        st.append(Stage("ln self", "layernorm_modulate_quant_from_stats", ("x", "stats", "e.1", "e.0"), ("xq", "xs"),
                        "ln_quant", ("x", "e.1", "e.0")))
    else:
        st.append(Stage("ln self", "layernorm_modulate_quant", ("x", "e.1", "e.0", eps), ("xq", "xs"), "ln_quant",
                        ("x", "e.1", "e.0")))
    rope = lambda which, src: Stage(f"rope {which}", "rmsnorm_rope", (src, f"sd:self_attn.norm_{which}.weight", "angles", eps, h),
                                    (which,), "rope", (src, f"sd:self_attn.norm_{which}.weight", "angles"))
    if cfg.fused_qkv:
        st.append(Stage("qkv", "gemm_cuda_split", ("xq", "xs", "qkv.w", "qkv.s", "qkv.b", dt, 3), ("qkv",), "gemm",
                        ("xq", "xs"), ("self_attn.q", "self_attn.k", "self_attn.v")))
        st += [rope("k", "qkv.1"), rope("q", "qkv.0")]
        v = "qkv.2"
    else:
        st += [_gemm("k", "x", "self_attn.k", "k_raw", dt), rope("k", "k_raw"), _gemm("v", "x", "self_attn.v", "v", dt),
               _gemm("q", "x", "self_attn.q", "q_raw", dt), rope("q", "q_raw")]
        v = "v"
    st.append(Stage("attention", "attention", (("q", "blhd"), ("k", "blhd"), (v, "blhd")), ("a",), "attention", ("q", "k", v)))
    st.append(Stage("quant a", "quant_cuda", ("a",), ("aq", "as"), "quant", ("a",)))
    st.append(_gemm("o", "a", "self_attn.o", "y_o", dt))
    st.append(Stage("gate self", "gate_residual", ("x", "y_o", "e.2"), ("x1",), "gate", ("x", "y_o", "e.2")))
    st.append(Stage("norm3", "fast_layernorm", ("x1", "sd:norm3.weight", "sd:norm3.bias", eps), ("hn",), "layernorm",
                    ("x1", "sd:norm3.weight", "sd:norm3.bias")))
    st.append(Stage("quant hn", "quant_cuda", ("hn",), ("hnq", "hns"), "quant", ("hn",)))
    st.append(_gemm("cross q", "hn", "cross_attn.q", "cq_raw", dt))
    st.append(Stage("cross norm q", "fast_rmsnorm", ("cq_raw", "sd:cross_attn.norm_q.weight", eps), ("cq",), "rmsnorm",
                    ("cq_raw", "sd:cross_attn.norm_q.weight")))
    st.append(Stage("quant context", "quant_cuda", ("context",), ("cxq", "cxs"), "quant", ("context",)))
    if cfg.fused_ckv:
        st.append(Stage("cross kv", "gemm_cuda_split", ("cxq", "cxs", "ckv.w", "ckv.s", "ckv.b", dt, 2), ("ckv",), "gemm",
                        ("cxq", "cxs"), ("cross_attn.k", "cross_attn.v")))
    else:
        st += [_gemm("cross k", "cx", "cross_attn.k", "ckv.0", dt), _gemm("cross v", "cx", "cross_attn.v", "ckv.1", dt)]
    st.append(Stage("cross norm k", "fast_rmsnorm", ("ckv.0", "sd:cross_attn.norm_k.weight", eps), ("ck",), "rmsnorm",
                    ("ckv.0", "sd:cross_attn.norm_k.weight")))
    st.append(Stage("sdpa", "sdpa", (("cq", "bhld"), ("ck", "bhld"), ("ckv.1", "bhld")), ("ca",), "sdpa", ("cq", "ck", "ckv.1")))
    st.append(Stage("quant ca", "quant_cuda", ("ca",), ("caq", "cas"), "quant", ("ca",)))
    st.append(_gemm("cross o", "ca", "cross_attn.o", "y_c", dt))
    st.append(Stage("cross residual", "gate_residual_stats", ("x1", "y_c", None, eps), ("x2", "st2"), "residual_stats",
                    ("x1", "y_c", None)))
    st.append(Stage("ln ffn", "layernorm_modulate_quant_from_stats", ("x2", "st2", "e.4", "e.3"), ("hq", "hs"), "ln_quant",
                    ("x2", "e.4", "e.3")))
    if cfg.ffn == "fused":
        st.append(Stage("ffn up", "gemm_cuda_quant_out", ("hq", "hs", "sd:ffn.0.int8_weight", "sd:ffn.0.scale", "sd:ffn.0.bias", dt),
                        ("uq", "us"), "ffn_up_fused", ("hq", "hs"), ("ffn.0",), {"gelu": True}))
    else:
        st.append(_gemm("ffn up", "h", "ffn.0", "u", dt))
        st.append(Stage("gelu quant", "gelu_quant_cuda", ("u",), ("uq", "us"), "gelu_quant", ("u",)))
    st.append(_gemm("ffn down", "u", "ffn.2", "y_f", dt))
    if cfg.want_stats:
        st.append(Stage("gate ffn", "gate_residual_stats", ("x2", "y_f", "e.5", eps), ("out", "stats_out"), "residual_stats",
                        ("x2", "y_f", "e.5")))
    else:
        st.append(Stage("gate ffn", "gate_residual", ("x2", "y_f", "e.5"), ("out",), "gate", ("x2", "y_f", "e.5")))
    return st


def block_env(sd: Dict[str, torch.Tensor], x, e0, angles, context, stats=None) -> dict:
    """The named values a block call starts from.  `stats`: the row statistics of x the block is handed, if any."""
    e = (sd["modulation"][0].float() + e0.float()).contiguous()    # the `e` stage: modulation[0] + e0 in fp32
    env = {"x": x, "e0": e0, "angles": angles, "context": context, "stats": stats, "head_split": "lhd"}
    env.update({f"sd:{k}": v for k, v in sd.items()})
    env.update({f"e.{i}": e[i] for i in range(6)})
    for key, names in (("qkv", ("self_attn.q", "self_attn.k", "self_attn.v")), ("ckv", ("cross_attn.k", "cross_attn.v"))):
        for suffix, short in ((".int8_weight", "w"), (".scale", "s"), (".bias", "b")):
            env[f"{key}.{short}"] = torch.cat([sd[n + suffix] for n in names], dim=0)
    return env


class ChainError(AssertionError):
    pass


def _arg_view(arg, view, ref, h, d):
    if view == "blhd":      # [1, L, H, D] view of an [L, H*D] matrix (the attention module's layout)
        if arg.dim() != 4 or arg.shape[0] != 1 or arg.shape[2:] != (h, d):
            raise ChainError(f"expected a [1, L, {h}, {d}] view, got {tuple(arg.shape)}")
        return arg.reshape(ref.shape)
    if view == "bhld":      # [1, H, L, D] view (scaled_dot_product_attention's layout)
        if arg.dim() != 4 or arg.shape[0] != 1 or arg.shape[1] != h or arg.shape[3] != d:
            raise ChainError(f"expected a [1, {h}, L, {d}] view, got {tuple(arg.shape)}")
        return arg.transpose(1, 2).reshape(ref.shape)
    if arg.shape != ref.shape:
        raise ChainError(f"shape {tuple(arg.shape)} != {tuple(ref.shape)}")
    return arg


def bind_outputs(env, stage, call, h, d):
    outs = call.out
    if stage.op == "gemm_cuda_split":
        (t,) = outs
        env[stage.outs[0]] = t
        for i in range(t.shape[0]):
            env[f"{stage.outs[0]}.{i}"] = t[i]
        return
    if stage.op == "attention":
        (t,) = outs
        env[stage.outs[0]] = t.reshape(t.shape[1], -1)
        return
    if stage.op == "sdpa":
        (t,) = outs
        if t.dim() != 4 or t.shape[0] != 1 or t.shape[1] != h:
            raise ChainError(f"sdpa output {tuple(t.shape)}")
        env[stage.outs[0]] = t.transpose(1, 2).reshape(t.shape[2], -1)
        return
    if len(outs) != len(stage.outs):
        raise ChainError(f"{stage.label}: {len(outs)} outputs, expected {len(stage.outs)}")
    for k, t in zip(stage.outs, outs):
        env[k] = t


def check_chain(calls: List[Call], stages: List[Stage], env: dict, h: int, d: int, ret=None) -> dict:
    """Holds the recorded calls to the stage list: same operators in the same order, every argument equal (by value, after
    the block's reshape) to its named source, and the block's return value equal to the last stage's output.  Binds each
    stage's recorded outputs into `env` (returned) for the stage checks.  Raises ChainError on the first mismatch."""
    names = [c.name for c in calls]
    want = [s.op for s in stages]
    if names != want:
        raise ChainError(f"call sequence {names} != expected {want}")
    for stage, call in zip(stages, calls):
        if len(call.args) != len(stage.args):
            raise ChainError(f"{stage.label}: {len(call.args)} arguments, expected {len(stage.args)}")
        for i, (arg, src) in enumerate(zip(call.args, stage.args)):
            if src is SKIP:
                continue
            key, view = src if isinstance(src, tuple) else (src, None)
            if isinstance(key, str):
                ref = env[key]
                ok = torch.is_tensor(arg) and arg.dtype == ref.dtype and torch.equal(_arg_view(arg, view, ref, h, d), ref)
                if not ok:
                    raise ChainError(f"{stage.label}: argument {i} is not `{key}`")
            elif key is None:
                if arg is not None:
                    raise ChainError(f"{stage.label}: argument {i} should be None")
            elif arg != key:
                raise ChainError(f"{stage.label}: argument {i} = {arg!r}, expected {key!r}")
        if call.kwargs != stage.kwargs:
            raise ChainError(f"{stage.label}: keyword arguments {call.kwargs} != {stage.kwargs}")
        bind_outputs(env, stage, call, h, d)
    if ret is not None:
        last = stages[-1].outs
        got = ret if isinstance(ret, tuple) else (ret,)
        if len(got) != len(last) or not all(torch.equal(g, env[k]) for g, k in zip(got, last)):
            raise ChainError("the block's return value is not the last stage's output")
    return env


# --------------------------------------------------------------------------------------------------------- references
def row_tiles(m: int, blk: int = 128):
    """The first, a middle and the last (ragged) 128-row tile of an m-row matrix."""
    nt = O.cdiv(m, blk)
    return [(t * blk, min(m, (t + 1) * blk)) for t in sorted({0, nt // 2, nt - 1})]


def _rows(t, tiles):
    return torch.cat([t[r0:r1] for r0, r1 in tiles])


def _block_rows(s, tiles):
    return torch.cat([s[r0 // 128: r0 // 128 + 1] for r0, _ in tiles])


def _fma32(p, c):
    """fp32 fma(a, b, c) where p = a*b is exact in float64: the float64 sum is made round-to-odd (TwoSum residual), which
    rounds to fp32 exactly as the fused fp32 operation does (53 >= 24 + 2 bits)."""
    cd = c.double()
    s = p + cd
    bp = s - cd
    err = (p - bp) + (cd - (s - bp))
    even = (s.view(torch.int64) & 1) == 0
    inf = torch.tensor(math.inf, dtype=torch.float64, device=s.device)
    s = torch.where((err != 0) & even, torch.nextafter(s, torch.where(err > 0, inf, -inf)), s)
    return s.float()


def gemm_ref(a_q, a_s_rows, b_q, b_s, bias, dtype):
    """O.int8_gemm's arithmetic on any device: per 128-deep K-block, acc = fma(float(int dot), a_s*b_s (fp32), acc),
    then T(T(acc) + bias).  `a_s_rows` holds one scale row per row of a_q.  The integer dots are exact in float64."""
    k = a_q.shape[1]
    n = b_q.shape[0]
    cols = torch.arange(n, device=b_q.device) // 128
    acc = torch.zeros(a_q.shape[0], n, dtype=torch.float32, device=a_q.device)
    for kb in range(k // 128):
        sl = slice(kb * 128, (kb + 1) * 128)
        dot = a_q[:, sl].double() @ b_q[:, sl].double().t()
        scale = a_s_rows[:, kb].float()[:, None] * b_s[cols, kb].float()[None, :]
        acc = _fma32(dot * scale.double(), acc)
    y = acc.to(dtype)
    return y if bias is None else y + bias.to(dtype)


def _ulp(t, dtype):
    return t.float().abs().clamp_min(1e-30).log2().floor().exp2() * \
        (2.0 ** -7 if dtype == torch.bfloat16 else 2.0 ** -10)


def ulp_report(got, ref, floor_frac=2e-2):
    """test_gpu_norm._ulp_report: (fraction of elements that differ, worst difference in ulps of the 16-bit type at
    max(|ref|, floor_frac * max|ref|))."""
    g, r = got.float(), ref.float()
    neq = g != r
    if not neq.any():
        return 0.0, 0.0
    mag = torch.maximum(r.abs(), floor_frac * r.abs().max())
    return neq.float().mean().item(), ((g - r).abs() / _ulp(mag, ref.dtype)).max().item()


def _exact(got, ref):
    if torch.equal(got, ref):
        return 0.0, "bit-exact"
    return math.inf, f"{(got != ref).float().mean().item():.3g} of the elements differ"


def _dequant(q, s, n):
    return q.float() * s.float().repeat_interleave(128, dim=1)[:, :n]


def _stats_bar(x, stats, eps):
    """Row statistics (mean, rstd) of x against float64, with the reference's padding quirk.  The bound follows fp32
    summation in any order: |sum error| <= (n-1) u sum|x_j| for the mean, (n+2) u sum d_j^2 for the centred squares, one
    rounding per remaining operation.  Returns (worst |err|/bound over both, the textbook rstd's distance in bounds)."""
    u = 2.0 ** -24
    xd = x.double()
    n = xd.shape[1]
    pad = O.next_pow2(n) - n
    m = xd.mean(1)
    dlt = xd - m[:, None]
    s2 = (dlt * dlt).sum(1)
    var = (s2 + pad * m * m) / n
    rstd = 1.0 / torch.sqrt(var + eps)
    bm = u * xd.abs().sum(1) + 2 * u * m.abs()
    s2h = s2 + n * bm * bm                                      # the centred squares about a mean off by up to bm
    num_err = (n + 3) * u * s2h + n * bm * bm + pad * ((2 * m.abs() + bm) * bm + 3 * u * (m.abs() + bm) ** 2)
    rel = num_err / (s2 + pad * m * m) + 3 * u
    b_rstd = rstd * (rel / 2 + 3 * u) * 1.01
    mean_got, rstd_got = stats.double().view(-1, 2).unbind(1)
    worst = max(((mean_got - m).abs() / bm).max().item(), ((rstd_got - rstd).abs() / b_rstd).max().item())
    textbook = 1.0 / torch.sqrt(s2 / n + eps)
    apart = ((textbook - rstd_got).abs() / b_rstd)
    return worst, apart, m.abs() / torch.sqrt(s2 / n)


@dataclass
class StageResult:
    label: str
    kind: str
    worst: float      # worst element or row as a fraction of the stage's bar (<= 1 passes)
    detail: str
    textbook: Optional[float] = None   # residual_stats at a non-power-of-two width: the textbook rstd's least distance, in bounds

    def __str__(self):
        return f"{self.label:15s} {self.kind:15s} worst {self.worst:10.4g} of its bar   {self.detail}"


def _heads(t, l, h, d, split):
    """[L, H*D] -> [1, L, H, D] as the block splits heads; split='ldh' restates a split done as (L, D, H)."""
    if split == "ldh":
        return t.reshape(1, l, d, h).transpose(2, 3).contiguous()
    return t.reshape(1, l, h, d)


def check_stage(stage: Stage, env: dict, cfg: Config, attention: Optional[Callable] = None) -> StageResult:
    """The recorded outputs of `stage` (bound in env) against a reference on the named inputs in `env`."""
    h, d, eps, dt = cfg.heads, cfg.dim // cfg.heads, cfg.eps, cfg.dtype
    ins = [env[k] if isinstance(k, str) else k for k in stage.ref]
    outs = [env[k] for k in stage.outs]
    cpu = lambda t: t.detach().cpu()
    kind = stage.kind
    if kind == "ln_quant":
        x, scale, shift = ins
        q, s = outs
        tiles = row_tiles(x.shape[0])
        xt, scale, shift = cpu(_rows(x, tiles)), cpu(scale), cpu(shift)
        ref = O.ln_modulate(xt, scale, shift, eps)
        hmid = O.fast_layernorm(xt, None, None, eps)
        qt, st = cpu(_rows(q, tiles)), cpu(_block_rows(s, tiles)).repeat_interleave(128, 0)[: xt.shape[0]]
        deq = _dequant(qt, st, xt.shape[1])
        # a code is within half a step of the kernel's 16-bit value, a full step where +amax saturates to 127
        step = st.repeat_interleave(128, dim=1)[:, : xt.shape[1]]
        bound = torch.where(qt == 127, step, step / 2) + _ulp(hmid, dt) * (1 + scale).abs() + _ulp(ref, dt)
        r = ((deq - ref.float()).abs() / bound).max().item()
        return StageResult(stage.label, kind, r, "dequantised codes vs O.ln_modulate")
    if kind == "gemm":
        a_q, a_s = ins
        (y,) = outs
        tiles = row_tiles(a_q.shape[0])
        aq = _rows(a_q, tiles)
        as_rows = _block_rows(a_s, tiles).repeat_interleave(128, 0)[: aq.shape[0]]
        parts = [y] if y.dim() == 2 else list(y.unbind(0))
        if len(parts) != len(stage.proj):
            return StageResult(stage.label, kind, math.inf, "wrong number of parts")
        worst, det = 0.0, "bit-exact"
        for p, part in zip(stage.proj, parts):
            ref = gemm_ref(aq, as_rows, env[f"sd:{p}.int8_weight"], env[f"sd:{p}.scale"], env.get(f"sd:{p}.bias"), dt)
            r, dd = _exact(_rows(part, tiles), ref)
            if r > worst:
                worst, det = r, f"{p}: {dd}"
        return StageResult(stage.label, kind, worst, det)
    if kind == "rope":
        x, w, ang = ins
        (y,) = outs
        tiles = row_tiles(x.shape[0])
        xt, at = cpu(_rows(x, tiles)), cpu(_rows(ang, tiles))
        ref = O.rms_norm_rope(xt.reshape(-1, h, d), cpu(w), at, eps)
        got = cpu(_rows(y, tiles)).reshape(-1, h, d)
        frac, worst = ulp_report(got, ref)
        # test_rope_and_fused_rmsnorm_rope's bar, <= 2 ulp, and the mechanism its comment names: the rotation reads the
        # T-rounded norm value, which may sit one ulp away from the oracle's (summation order); that ulp moves the rotated
        # pair by ulp(n0)|c| + ulp(n1)|s|, which a small (cancelled) output can see as more than 2 of its own ulps
        n16 = O.fast_rmsnorm(xt, cpu(w), eps).reshape(-1, h, d)
        c, s_ = torch.cos(at)[:, None, :].abs(), torch.sin(at)[:, None, :].abs()
        u0, u1 = _ulp(n16[..., 0::2], dt), _ulp(n16[..., 1::2], dt)
        flip = torch.stack((u0 * c + u1 * s_, u0 * s_ + u1 * c), dim=-1).reshape(ref.shape) + _ulp(ref, dt)
        mag = torch.maximum(ref.float().abs(), 2e-2 * ref.float().abs().max())
        bound = torch.maximum(2.0 * _ulp(mag, dt), flip)
        r_el = ((got.float() - ref.float()).abs() / bound).max().item()
        return StageResult(stage.label, kind, max(r_el, frac / 5e-3),
                           f"{worst:.3g} ulp ({r_el:.3g} of max(2 ulp, one flipped norm ulp rotated)), {frac:.3g} differ")
    if kind == "attention":
        q, k, v = ins
        (o,) = outs
        l = q.shape[0]
        split = env.get("head_split", "lhd")
        ref = attention(*(_heads(t, l, h, d, split) for t in (q, k, v)))
        if split == "ldh":      # merged back the same way
            ref = ref.transpose(2, 3)
        return StageResult(stage.label, kind, *_exact(o, ref.reshape(o.shape)))
    if kind == "quant":
        (x,) = ins
        q, s = outs
        tiles = row_tiles(x.shape[0])
        q_ref, s_ref = O.int8_quant(cpu(_rows(x, tiles)))
        rq, dq = _exact(cpu(_rows(q, tiles)), q_ref)
        rs, ds = _exact(cpu(_block_rows(s, tiles)), s_ref)
        return StageResult(stage.label, kind, max(rq, rs), f"codes {dq}, scales {ds}")
    if kind == "gate":
        x, y, g = ins
        (o,) = outs
        tiles = row_tiles(x.shape[0])
        ref = O.gate_residual(cpu(_rows(x, tiles)), cpu(_rows(y, tiles)), cpu(g))
        return StageResult(stage.label, kind, *_exact(cpu(_rows(o, tiles)), ref))
    if kind == "residual_stats":
        x, y, g = ins
        o, stats = outs
        tiles = row_tiles(x.shape[0])
        xt, yt = cpu(_rows(x, tiles)), cpu(_rows(y, tiles))
        ref = O.gate_residual(xt, yt, cpu(g)) if g is not None else xt + yt
        ot = cpu(_rows(o, tiles))
        r_out, d_out = _exact(ot, ref)
        st = cpu(torch.cat([stats.view(-1, 2)[r0:r1] for r0, r1 in tiles]))
        r_st, apart, mean_ratio = _stats_bar(ot, st, eps)
        detail = f"sum {d_out}; stats {r_st:.3g} of the fp32-summation bound"
        textbook = None
        if O.next_pow2(x.shape[1]) != x.shape[1]:
            # rows whose mean is a tenth of their spread or more: there the padding term must be visible
            sel = mean_ratio > 0.1
            textbook = apart[sel].min().item() if sel.float().mean().item() > 0.5 else 0.0
            detail += f"; textbook rstd >= {textbook:.3g} bounds away on {sel.float().mean().item():.3g} of the rows"
        return StageResult(stage.label, kind, max(r_out, r_st), detail, textbook)
    if kind in ("layernorm", "rmsnorm"):
        x = ins[0]
        (y,) = outs
        tiles = row_tiles(x.shape[0])
        xt = cpu(_rows(x, tiles))
        ref = O.fast_layernorm(xt, cpu(ins[1]), cpu(ins[2]), eps) if kind == "layernorm" else O.fast_rmsnorm(xt, cpu(ins[1]), eps)
        frac, worst = ulp_report(cpu(_rows(y, tiles)), ref)
        return StageResult(stage.label, kind, max(worst / 1.0, frac / 2e-3), f"<= 1 ulp: {worst:.3g} ulp, {frac:.3g} differ")
    if kind == "sdpa":
        cq, ck, cv = ins
        (ca,) = outs
        l, lc = cq.shape[0], ck.shape[0]
        split = env.get("head_split", "lhd")
        tiles = row_tiles(l)
        qt = _rows(cq, tiles)
        qh = _heads(qt, qt.shape[0], h, d, split)[0].double()
        kh = _heads(ck, lc, h, d, split)[0].double()
        vh = _heads(cv, lc, h, d, split)[0].double()
        p = torch.softmax(torch.einsum("rhd,khd->hrk", qh, kh) * d ** -0.5, dim=-1)
        r64 = torch.einsum("hrk,khd->rhd", p, vh)
        spread = torch.einsum("hrk,khd->rhd", p, vh.abs())
        got = _rows(ca, tiles).reshape(-1, h, d).double()
        bound = _ulp(r64.to(dt), dt).double().to(r64.device) + 2.0 ** -8 * spread
        r = ((got - r64).abs() / bound).max().item()
        return StageResult(stage.label, kind, r, "vs float64 softmax attention per head")
    if kind in ("ffn_up_fused", "gelu_quant"):
        q, s = outs
        if kind == "ffn_up_fused":
            a_q, a_s = ins
            tiles = row_tiles(a_q.shape[0])
            aq = _rows(a_q, tiles)
            as_rows = _block_rows(a_s, tiles).repeat_interleave(128, 0)[: aq.shape[0]]
            (p,) = stage.proj
            pre = cpu(gemm_ref(aq, as_rows, env[f"sd:{p}.int8_weight"], env[f"sd:{p}.scale"], env[f"sd:{p}.bias"], dt))
        else:
            (u,) = ins
            tiles = row_tiles(u.shape[0])
            pre = cpu(_rows(u, tiles))
        q_ref, s_ref = O.int8_quant(F.gelu(pre, approximate="tanh"))
        dq = (cpu(_rows(q, tiles)).to(torch.int16) - q_ref.to(torch.int16)).abs()
        ds = ((cpu(_block_rows(s, tiles)) - s_ref).abs() / (2.0 ** -7 * s_ref)).max().item()
        frac = (dq > 0).float().mean().item()
        r = max(dq.max().item() / 1.0, frac / 2e-2, ds)
        return StageResult(stage.label, kind, r, f"codes within {dq.max().item()} on {frac:.3g}, scales {ds:.3g} of 2^-7")
    raise ValueError(kind)


def check_block(stages, env, cfg, attention) -> List[StageResult]:
    """Every stage of a chained recording (env from check_chain) against its reference."""
    res = [StageResult("e", "modulation", 0.0, "modulation[0] + e0 in fp32: bit-exact (held by the chain)")]
    res += [check_stage(s, env, cfg, attention) for s in stages]
    return res


# -------------------------------------------------------------------------------------------------------------- faults
def _swap(*pairs):
    def f(env):
        env = dict(env)
        for a, b in pairs:
            env[a], env[b] = env[b], env[a]
        return env
    return f


def _swap_proj(a, b):
    return _swap(*((f"sd:{a}{s}", f"sd:{b}{s}") for s in (".int8_weight", ".scale", ".bias")))


def _cycle_proj(*names):
    def f(env):
        env = dict(env)
        for s in (".int8_weight", ".scale", ".bias"):
            vals = [env[f"sd:{n}{s}"] for n in names]
            for n, v in zip(names, vals[1:] + vals[:1]):
                env[f"sd:{n}{s}"] = v
        return env
    return f


def _set(key, fn):
    def f(env):
        env = dict(env)
        env[key] = fn(env[key])
        return env
    return f


def faults(cfg: Config):
    """(name, label of the stage it lands in, env transform restating the fault)."""
    qkv = "qkv" if cfg.fused_qkv else "q"
    ckv = "cross kv" if cfg.fused_ckv else "cross k"
    return [
        ("e[0] <-> e[1]", "ln self", _swap(("e.0", "e.1"))),
        ("e[3] <-> e[4]", "ln ffn", _swap(("e.3", "e.4"))),
        ("e[2] <-> e[5]", "gate self", _swap(("e.2", "e.5"))),
        ("e[2] <-> e[5]", "gate ffn", _swap(("e.2", "e.5"))),
        ("norm_q <-> norm_k weights", "rope q", _swap(("sd:self_attn.norm_q.weight", "sd:self_attn.norm_k.weight"))),
        ("norm_q <-> norm_k weights", "rope k", _swap(("sd:self_attn.norm_q.weight", "sd:self_attn.norm_k.weight"))),
        ("self/cross norm weights swapped", "cross norm q",
         _swap(("sd:self_attn.norm_q.weight", "sd:cross_attn.norm_q.weight"))),
        ("self/cross norm weights swapped", "cross norm k",
         _swap(("sd:self_attn.norm_k.weight", "sd:cross_attn.norm_k.weight"))),
        ("angles rolled by one row", "rope q", _set("angles", lambda a: a.roll(1, 0))),
        ("angles rolled by one row", "rope k", _set("angles", lambda a: a.roll(1, 0))),
        ("q/k/v parts permuted", qkv, _cycle_proj("self_attn.q", "self_attn.k", "self_attn.v")),
        ("cross k <-> v", ckv, _swap_proj("cross_attn.k", "cross_attn.v")),
        ("o-proj bias dropped", "o", _set("sd:self_attn.o.bias", torch.zeros_like)),
        ("ffn.0 bias dropped", "ffn up", _set("sd:ffn.0.bias", torch.zeros_like)),
        ("head split as (L, D, H)", "attention", _set("head_split", lambda _: "ldh")),
        ("head split as (L, D, H)", "sdpa", _set("head_split", lambda _: "ldh")),
    ]


def check_faults(stages, env, cfg, attention) -> List[tuple]:
    """Each fault of faults(cfg) restated in its stage's reference: (name, StageResult) of the recorded output against it."""
    by_label = {s.label: s for s in stages}
    return [(name, check_stage(by_label[label], fn(env), cfg, attention)) for name, label, fn in faults(cfg)]
