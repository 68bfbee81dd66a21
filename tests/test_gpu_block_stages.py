"""The Wan block (turbodiffusion_b200/block.py) stage by stage on its own intermediates, and the denoise step against its
blocks.  Every operator the block calls is recorded; the recording must follow the block's wiring exactly (tests/
block_stages.py: check_chain), and every stage's output is held to a reference on its own recorded inputs with the bar of the
operator's unit test (check_stage), on the first, a middle and the ragged last 128-row tile, every column and every head.
The whole-block comparison in test_gpu_block.py cannot do this: its output is mostly the residual passing through, so
faults such as a swapped FFN scale and shift fit inside its bar."""
import contextlib
import dataclasses
import time

import pytest
import torch
import torch.nn.functional as F

from oracle import td_oracle as O

import block_stages as S

pytestmark = pytest.mark.gpu

OPS = ("layernorm_modulate_quant", "layernorm_modulate_quant_from_stats", "rmsnorm_rope", "gate_residual",
       "gate_residual_stats", "fast_layernorm", "fast_rmsnorm")
GEMMS = (("quant_cuda", None), ("gemm_cuda_split", None), ("gemm_cuda_swizzle_bias", 4), ("gemm_cuda_bias_gelu", 4),
         ("gemm_cuda_quant_out", None), ("gelu_quant_cuda", None))


@contextlib.contextmanager
def recording(blocks):
    """Records every operator call of the blocks' forward passes; restores everything afterwards."""
    from turbodiffusion_b200 import block as B, ops
    rec = S.Recorder()
    saved = [blk.sla for blk in blocks]
    with pytest.MonkeyPatch.context() as mp:
        for name in OPS:
            mp.setattr(ops, name, rec.wrap(name, getattr(ops, name)))
        for name, out_arg in GEMMS:
            mp.setattr(B, name, rec.wrap(name, getattr(B, name), out_arg))
        mp.setattr(F, "scaled_dot_product_attention", rec.wrap("sdpa", F.scaled_dot_product_attention))
        for blk in blocks:
            blk.sla = S.AttentionRecorder(rec, blk.sla)
        try:
            yield rec
        finally:
            for blk, sla in zip(blocks, saved):
                blk.sla = sla


def _state(dim, ffn, heads, seed, device, dtype):
    """random_block_state with modulation chunks of distinct means 0.1 (i + 1) and std 0.3 (norm weights already have std
    0.1 about 1), so that every wiring fault of block_stages.faults lands many bars away."""
    from turbodiffusion_b200.block import random_block_state
    sd = random_block_state(dim, ffn, heads, seed, device, dtype)
    g = torch.Generator(device=device).manual_seed(seed + 1)
    sd["modulation"] = (0.1 * torch.arange(1, 7, device=device).float()[:, None]
                        + 0.3 * torch.randn(6, dim, generator=g, device=device))[None]
    return sd


def _inputs(thw, dim, heads, lc, device, dtype, seed=0):
    g = torch.Generator(device=device).manual_seed(seed)
    l = thw[0] * thw[1] * thw[2]
    x = (torch.randn(l, dim, generator=g, device=device) + 0.5).to(dtype)     # non-zero row means: the LayerNorm padding quirk shows
    e0 = torch.randn(6, dim, generator=g, device=device) * 0.05
    ctx = torch.randn(lc, dim, generator=g, device=device).to(dtype)
    ang = O.wan_rope_angles(*thw, dim // heads).to(device)
    return x, e0, ang, ctx


def _config(B, dim, heads, dtype):
    fused_qkv = B.FUSE_QKV == "1" or (B.FUSE_QKV == "auto" and dim % 256 == 0)
    return S.Config(dim, heads, dtype, fused_qkv=fused_qkv, fused_ckv=B.FUSE_QKV != "0" and dim % 256 == 0, ffn=B.FFN_ACT_MODE)


def _run_block(cuda, dim, heads, ffn, thw, lc, dtype, attention="sagesla", topk=0.1, seed=3):
    """One recorded block call, chained: (cfg, stages, env, attention module)."""
    from turbodiffusion_b200 import block as B
    sd = _state(dim, ffn, heads, seed, cuda, dtype)
    blk = B.WanBlockB200(sd, dim, heads, topk=topk, attention=attention)
    x, e0, ang, ctx = _inputs(thw, dim, heads, lc, cuda, dtype)
    with recording([blk]) as rec:
        out = blk(x, e0, ang, ctx)
    torch.cuda.synchronize()
    cfg = _config(B, dim, heads, dtype)
    stages = S.block_stages(cfg)
    env = S.check_chain(rec.calls, stages, S.block_env(blk.sd, x, e0, ang, ctx), heads, dim // heads, ret=out)
    return cfg, stages, env, blk.sla


def _check_all(cfg, stages, env, attention):
    results = S.check_block(stages, env, cfg, attention)
    for r in results:
        print(r)
    bad = [r for r in results if not r.worst <= 1.0]
    assert not bad, "\n".join(map(str, bad))
    for r in results:
        if r.textbook is not None:
            assert r.textbook > 1.0, f"the textbook variance is inside the statistics bound: {r}"


@pytest.fixture
def served_arch(cuda):
    from turbodiffusion_b200.SLA.utils import set_served_arch
    prev = set_served_arch("sm100")
    yield set_served_arch
    set_served_arch(prev)


SMALL = [  # dim, heads, attention, FFN_ACT_MODE, FUSE_QKV, served arch, dtype
    (512, 4, "sagesla", "fused", "auto", "sm100", torch.bfloat16),
    (512, 4, "sagesla", "split", "0", "sm100", torch.bfloat16),
    (512, 4, "sagesla", "fused", "1", "sm90", torch.bfloat16),
    (512, 4, "sla", "split", "1", "sm100", torch.bfloat16),
    (512, 4, "sla", "fused", "0", "sm100", torch.bfloat16),
    (384, 3, "sagesla", "split", "auto", "sm90", torch.bfloat16),
    (384, 3, "sla", "fused", "0", "sm100", torch.bfloat16),
    (512, 4, "sagesla", "fused", "auto", "sm100", torch.float16),
    (384, 3, "sagesla", "split", "auto", "sm90", torch.float16),
]


@pytest.mark.parametrize("dim,heads,attention,ffn_mode,fuse,arch,dtype", SMALL)
def test_block_stages_small(cuda, served_arch, monkeypatch, dim, heads, attention, ffn_mode, fuse, arch, dtype):
    """L = 702 (thw 2x13x27: last row tile of 62 rows), 77 text tokens.  The block serves fp16 too: every operator takes
    fp16, and the attention module computes in bf16 and returns its input dtype."""
    from turbodiffusion_b200 import block as B
    monkeypatch.setattr(B, "FFN_ACT_MODE", ffn_mode)
    monkeypatch.setattr(B, "FUSE_QKV", fuse)
    served_arch(arch)
    cfg, stages, env, attn = _run_block(cuda, dim, heads, 2 * dim + 128, (2, 13, 27), 77, dtype, attention, topk=0.3)
    assert cfg.fused_qkv == (fuse == "1" or (fuse == "auto" and dim % 256 == 0))
    _check_all(cfg, stages, env, attn)


@pytest.mark.parametrize("shape", ["A", "B"])
def test_block_stages_full_size(cuda, shape):
    """Wan2.1 1.3B (A: L = 32760, dim 1536, 12 heads, FFN 8960) and 14B (B: L = 75600, dim 5120, 40 heads, FFN 13824) with
    512 text tokens, bf16, SageSLA, default modes.  Ragged last row tiles of 120 and 80 rows."""
    dim, heads, ffn, thw = {"A": (1536, 12, 8960, (21, 30, 52)), "B": (5120, 40, 13824, (21, 45, 80))}[shape]
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    cfg, stages, env, attn = _run_block(cuda, dim, heads, ffn, thw, 512, torch.bfloat16)
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    _check_all(cfg, stages, env, attn)
    print(f"shape {shape}: peak memory with the recording {peak:.1f} GiB, {time.perf_counter() - t0:.1f} s")


def test_stage_bars_reject_wiring_faults(cuda, served_arch, monkeypatch):
    """Each wiring fault of block_stages.faults restated in its stage's reference, on one recorded call: the block's
    recorded output must fail that stage's bar."""
    from turbodiffusion_b200 import block as B
    monkeypatch.setattr(B, "FFN_ACT_MODE", "fused")
    monkeypatch.setattr(B, "FUSE_QKV", "auto")
    cfg, stages, env, attn = _run_block(cuda, 512, 4, 1152, (2, 13, 27), 77, torch.bfloat16, topk=0.3)
    assert cfg.fused_qkv and cfg.fused_ckv
    failed_to_fail = []
    for name, r in S.check_faults(stages, env, cfg, attn):
        print(f"{name:32s} {r}")
        if not r.worst > 1.0:
            failed_to_fail.append(f"{name}: {r}")
    assert not failed_to_fail, "\n".join(failed_to_fail)


def test_step_matches_its_blocks(cuda):
    """WanHotPath.step over 3 layers at shape A's dims == x = blk(x, e0, angles, ctx) over the same blocks (no stats, no e),
    bit for bit; the step's recording follows the step's wiring (e_all[i] is block i's own table, each block after the first
    reads the previous block's statistics) and every threaded statistics vector is within its fp32 bound of float64."""
    from turbodiffusion_b200 import block as B
    dim, heads, ffn, thw = 1536, 12, 8960, (21, 30, 52)
    hp = B.WanHotPath(dim, ffn, heads, 3, cuda, seed=21)
    x, e0, ang, ctx = _inputs(thw, dim, heads, 512, cuda, torch.bfloat16, seed=5)
    ref = x
    for blk in hp.blocks:
        ref = blk(ref, e0, ang, ctx)
    with recording(hp.blocks) as rec:
        out = hp.step(x, e0, ang, ctx)
    torch.cuda.synchronize()
    assert torch.equal(out, ref), f"{(out != ref).float().mean().item():.3g} of the step's outputs differ from its blocks'"
    calls, xin, stats, last = rec.calls, x, None, len(hp.blocks) - 1
    for i, blk in enumerate(hp.blocks):
        cfg = dataclasses.replace(_config(B, dim, heads, torch.bfloat16), stats_in=i > 0, want_stats=i < last)
        stages = S.block_stages(cfg)
        mine, calls = calls[:len(stages)], calls[len(stages):]
        # e_all[i] must be block i's own table plus e0, bit for bit
        env = S.check_chain(mine, stages, S.block_env(blk.sd, xin, e0, ang, ctx, stats), heads, dim // heads)
        for st in stages:
            if st.kind == "residual_stats":
                r = S.check_stage(st, env, cfg)
                print(f"block {i}: {r}")
                assert r.worst <= 1.0 and (r.textbook is None or r.textbook > 1.0), r
        xin, stats = env["out"], env.get("stats_out")
    assert not calls
