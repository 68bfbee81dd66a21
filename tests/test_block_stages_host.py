"""The Wan block's stage checks (tests/block_stages.py) on a block chain built from the CPU oracle, without a GPU: every stage
of the chain passes its bar, every wiring fault the GPU test restates fails its stage's bar, a mis-wired recording fails the
chain check, and the device-agnostic GEMM reference the checks use is the oracle's W8A8 GEMM bit for bit."""
import dataclasses

import pytest
import torch
import torch.nn.functional as F

from oracle import td_oracle as O

import block_stages as S


def _state(dim, ffn, heads, seed, dtype=torch.bfloat16):
    """random_block_state's layout and scales on the CPU (quantised with the oracle), with modulation chunks of distinct
    means 0.1 (i + 1) and std 0.3 so that swapping two of them moves every modulated value."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    shapes = {"self_attn.q": (dim, dim), "self_attn.k": (dim, dim), "self_attn.v": (dim, dim), "self_attn.o": (dim, dim),
              "cross_attn.q": (dim, dim), "cross_attn.k": (dim, dim), "cross_attn.v": (dim, dim),
              "cross_attn.o": (dim, dim), "ffn.0": (ffn, dim), "ffn.2": (dim, ffn)}
    for name, (n, k) in shapes.items():
        q, s = O.int8_quant((torch.randn(n, k, generator=g) * k ** -0.5).to(dtype))
        sd[name + ".int8_weight"], sd[name + ".scale"] = q, s
        sd[name + ".bias"] = (torch.randn(n, generator=g) * 0.02).to(dtype)
    for name in ("self_attn.norm_q", "self_attn.norm_k", "cross_attn.norm_q", "cross_attn.norm_k", "norm3"):
        sd[name + ".weight"] = 1.0 + 0.1 * torch.randn(dim, generator=g)
    sd["norm3.bias"] = 0.05 * torch.randn(dim, generator=g)
    sd["modulation"] = (0.1 * torch.arange(1, 7).float()[:, None] + 0.3 * torch.randn(6, dim, generator=g))[None]
    d = dim // heads
    sd["self_attn.attn_op.local_attn.proj_l.weight"] = torch.randn(d, d, generator=g) * 0.05
    sd["self_attn.attn_op.local_attn.proj_l.bias"] = torch.randn(d, generator=g) * 0.05
    return sd


def _oracle_op(op, args, kwargs, cfg, attention):
    eps = cfg.eps
    if op == "layernorm_modulate_quant":
        return O.int8_quant(O.ln_modulate(args[0], args[1], args[2], eps))
    if op == "layernorm_modulate_quant_from_stats":
        return O.int8_quant(O.ln_modulate(args[0], args[2], args[3], eps))
    if op == "gemm_cuda_split":
        xq, xs, w, ws, b, dt, parts = args
        y = O.int8_gemm(xq, xs, w, ws, dt, b)
        return (y.view(y.shape[0], parts, -1).transpose(0, 1).contiguous(),)
    if op == "gemm_cuda_swizzle_bias":
        xq, xs, w, ws, c, b = args
        c.copy_(O.int8_gemm(xq, xs, w, ws, c.dtype, b))
        return (c,)
    if op == "rmsnorm_rope":
        x, w, ang, e, h = args
        return (O.rms_norm_rope(x.view(x.shape[0], h, -1), w, ang, e).reshape(x.shape),)
    if op == "attention":
        return (attention(*args),)
    if op == "quant_cuda":
        return O.int8_quant(args[0])
    if op == "gate_residual":
        return (O.gate_residual(*args),)
    if op == "fast_layernorm":
        return (O.fast_layernorm(*args),)
    if op == "fast_rmsnorm":
        return (O.fast_rmsnorm(*args),)
    if op == "sdpa":
        return (F.scaled_dot_product_attention(*args),)
    if op == "gate_residual_stats":
        x, y, g, e = args
        out = O.gate_residual(x, y, g) if g is not None else x + y
        xf = out.float()
        n = xf.shape[1]
        mean = xf.sum(1) / n
        ss = ((xf - mean[:, None]) ** 2).sum(1) + float(O.next_pow2(n) - n) * mean * mean
        rstd = 1.0 / torch.sqrt(ss / n + e)
        return out, torch.stack((mean, rstd), 1).reshape(-1)
    if op == "gemm_cuda_quant_out":
        xq, xs, w, ws, b, dt = args
        return O.int8_quant(F.gelu(O.int8_gemm(xq, xs, w, ws, dt, b), approximate="tanh"))
    if op == "gelu_quant_cuda":
        return O.int8_quant(F.gelu(args[0], approximate="tanh"))
    raise ValueError(op)


def oracle_chain(cfg, env, attention):
    """Runs the stage list on the oracle: a recording of the block as the oracle computes it."""
    env = dict(env)
    h, d = cfg.heads, cfg.dim // cfg.heads
    calls = []
    for stage in S.block_stages(cfg):
        args = []
        for src in stage.args:
            if src is S.SKIP:
                args.append(torch.empty(env[stage.ref[0]].shape[0], env[f"sd:{stage.proj[0]}.int8_weight"].shape[0],
                                        dtype=cfg.dtype))
                continue
            key, view = src if isinstance(src, tuple) else (src, None)
            if not isinstance(key, str):
                args.append(key)
                continue
            t = env[key]
            args.append(t.reshape(1, -1, h, d) if view == "blhd" else
                        t.reshape(1, -1, h, d).transpose(1, 2) if view == "bhld" else t)
        out = tuple(_oracle_op(stage.op, args, stage.kwargs, cfg, attention))
        call = S.Call(stage.op, tuple(args), dict(stage.kwargs), out)
        calls.append(call)
        S.bind_outputs(env, stage, call, h, d)
    return calls


def _setup(dim, heads, ffn, fused, ffn_mode="fused", dtype=torch.bfloat16, thw=(2, 10, 15), lc=40, topk=0.3):
    cfg = S.Config(dim, heads, dtype, fused_qkv=fused, fused_ckv=fused, ffn=ffn_mode)
    sd = _state(dim, ffn, heads, seed=dim + ffn)
    g = torch.Generator().manual_seed(7)
    l = thw[0] * thw[1] * thw[2]
    x = (torch.randn(l, dim, generator=g) + 0.5).to(dtype)
    e0 = torch.randn(6, dim, generator=g) * 0.05
    ctx = torch.randn(lc, dim, generator=g).to(dtype)
    ang = O.wan_rope_angles(*thw, dim // heads)
    pw, pb = sd["self_attn.attn_op.local_attn.proj_l.weight"], sd["self_attn.attn_op.local_attn.proj_l.bias"]
    attention = lambda q, k, v: O.sla_forward(q, k, v, pw, pb, topk, mode="exact")
    env = S.block_env(sd, x, e0, ang, ctx)
    calls = oracle_chain(cfg, env, attention)
    return cfg, env, calls, attention


CASES = [(256, 2, 512, True, "fused", torch.bfloat16), (384, 3, 640, False, "split", torch.bfloat16),
         (256, 2, 512, True, "split", torch.float16)]


@pytest.mark.parametrize("dim,heads,ffn,fused,ffn_mode,dtype", CASES)
def test_stage_checks_pass_on_the_oracle_chain(dim, heads, ffn, fused, ffn_mode, dtype):
    cfg, env0, calls, attention = _setup(dim, heads, ffn, fused, ffn_mode, dtype)
    stages = S.block_stages(cfg)
    env = S.check_chain(calls, stages, dict(env0), heads, dim // heads, ret=calls[-1].out[0])
    for r in S.check_block(stages, env, cfg, attention):
        print(r)
        assert r.worst <= 1.0, r
        if r.textbook is not None:
            assert r.textbook > 1.0, r


@pytest.mark.parametrize("dim,heads,ffn,fused", [(256, 2, 512, True), (384, 3, 640, False)])
def test_stage_bars_reject_wiring_faults_host(dim, heads, ffn, fused):
    cfg, env0, calls, attention = _setup(dim, heads, ffn, fused)
    stages = S.block_stages(cfg)
    env = S.check_chain(calls, stages, dict(env0), heads, dim // heads)
    for name, r in S.check_faults(stages, env, cfg, attention):
        print(f"{name:32s} {r}")
        assert r.worst > 1.0, (name, r)


def test_chain_rejects_a_miswired_recording():
    cfg, env0, calls, attention = _setup(256, 2, 512, True)
    stages = S.block_stages(cfg)
    h, d = 2, 128
    S.check_chain(calls, stages, dict(env0), h, d)
    bad = list(calls)
    c = bad[0]
    bad[0] = dataclasses.replace(c, args=(c.args[0], c.args[2], c.args[1], c.args[3]))   # scale and shift swapped
    with pytest.raises(S.ChainError, match="ln self"):
        S.check_chain(bad, stages, dict(env0), h, d)
    with pytest.raises(S.ChainError, match="sequence"):
        S.check_chain(calls[:3] + calls[4:], stages, dict(env0), h, d)
    i = next(j for j, s in enumerate(stages) if s.label == "attention")
    c = calls[i]
    q = c.args[0].reshape(1, -1, d, h).transpose(2, 3)                                  # heads split as (L, D, H)
    bad = list(calls)
    bad[i] = dataclasses.replace(c, args=(q,) + c.args[1:])
    with pytest.raises(S.ChainError, match="attention"):
        S.check_chain(bad, stages, dict(env0), h, d)
    with pytest.raises(S.ChainError, match="return value"):
        S.check_chain(calls, stages, dict(env0), h, d, ret=env0["x"])


@pytest.mark.parametrize("m,n,k", [(300, 256, 384), (77, 384, 1280)])
def test_gemm_ref_is_the_oracle_gemm(m, n, k):
    g = torch.Generator().manual_seed(m + n + k)
    a_q, a_s = O.int8_quant((torch.randn(m, k, generator=g) * torch.rand(m, 1, generator=g) * 4).bfloat16())
    b_q, b_s = O.int8_quant((torch.randn(n, k, generator=g) * k ** -0.5).bfloat16())
    bias = (torch.randn(n, generator=g) * 0.1).bfloat16()
    ref = O.int8_gemm(a_q, a_s, b_q, b_s, torch.bfloat16, bias)
    got = S.gemm_ref(a_q, a_s.repeat_interleave(128, 0)[:m], b_q, b_s, bias, torch.bfloat16)
    assert torch.equal(got.view(torch.int16), ref.view(torch.int16))
    assert torch.equal(S.gemm_ref(a_q, a_s.repeat_interleave(128, 0)[:m], b_q, b_s, None, torch.float32),
                       O.int8_gemm_f32(a_q, a_s, b_q, b_s))
