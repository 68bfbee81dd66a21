"""GPU parity of the Hopper SageSLA block family (BLKQ=64 query rows, BLKK=128 key rows; SLA/core.py:191-193 on sm90), selected
with SLA.utils.set_served_arch("sm90").  Same tolerances as test_gpu_sla.py:
  * Sage INT8 codes and scales: exact vs the emulation on the kernel's own rounded key mean;
  * block map: an exact top-k of the rounded pooled scores, equal to the oracle's selection except at threshold ties;
  * attention output vs the fp32 block-sparse oracle on the kernel's own map: cosine >= 0.999, rel-L2 <= 2e-2;
    vs the INT8 emulation oracle: rel-L2 <= 1e-2.
"""
import os

import pytest
import torch

from oracle import td_oracle as O

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
BQ, BK = 64, 128


@pytest.fixture
def sm90(cuda):
    from turbodiffusion_b200.SLA.utils import set_served_arch
    prev = set_served_arch("sm90")
    yield cuda
    set_served_arch(prev)


def _qkv(b, l, h, d, seed, kbias=2.0, dtype=torch.bfloat16):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(b, l, h, d, generator=g)
    k = torch.randn(b, l, h, d, generator=g) + torch.randn(1, 1, h, d, generator=g) * kbias
    v = torch.randn(b, l, h, d, generator=g)
    return q.to(dtype), k.to(dtype), v.to(dtype)


def _module(d, ratio, cuda, seed=5, **kw):
    from turbodiffusion_b200.SLA import SageSparseLinearAttention
    g = torch.Generator().manual_seed(seed)
    mod = SageSparseLinearAttention(d, ratio, **kw).to(cuda)
    with torch.no_grad():
        mod.proj_l.weight.copy_(torch.randn(d, d, generator=g) * 0.05)
        mod.proj_l.bias.copy_(torch.randn(d, generator=g) * 0.05)
    return mod


@pytest.mark.parametrize("b,l,h,d,dtype", [(1, 600, 2, 128, torch.bfloat16), (2, 333, 3, 128, torch.bfloat16),
                                           (1, 1000, 2, 64, torch.bfloat16), (1, 600, 2, 128, torch.float16)])
def test_quant_qk_hopper_blocks_codes_scales_pools(sm90, b, l, h, d, dtype):
    from turbodiffusion_b200.SLA.utils import quant_qk
    q, k, _ = _qkv(b, l, h, d, 100 + l, dtype=dtype)
    prep = quant_qk(q.to(sm90), k.to(sm90), blkq=BQ, blkk=BK)
    torch.cuda.synchronize()
    assert prep.mblk == (l + 63) // 64 and prep.nblk == (l + 127) // 128
    qh, kh = q.transpose(1, 2).contiguous(), k.transpose(1, 2).contiguous()
    torch.testing.assert_close(prep.kmean.cpu(), kh.float().mean(-2), rtol=1e-5, atol=1e-5)
    arg_k = kh - prep.kmean.cpu().to(dtype)[:, :, None, :]
    pq_ref, pk_ref = O.mean_pool(qh, BQ).float(), O.mean_pool(arg_k, BK).float()
    assert (prep.q_pool.cpu().float() - pq_ref).abs().max() <= 2.0 ** -7 * pq_ref.abs().max() + 1e-6
    assert (prep.k_pool.cpu().float() - pk_ref).abs().max() <= 2.0 ** -7 * pk_ref.abs().max() + 1e-6
    q_i8, q_s = O.sage_quant_blocks(qh, BQ)
    k_i8, k_s = O.sage_quant_blocks(arg_k, BK)
    assert torch.equal(prep.q_scale.cpu(), q_s) and torch.equal(prep.k_scale.cpu(), k_s)
    assert torch.equal(prep.q_i8.cpu(), q_i8), (prep.q_i8.cpu() != q_i8).sum()
    assert torch.equal(prep.k_i8.cpu(), k_i8), (prep.k_i8.cpu() != k_i8).sum()


def _check_topk(scores, sm, lt, topk):
    """`sm` is a top-k of `scores` up to one 16-bit ulp at the threshold; LUT ascending and equal to the map."""
    assert (sm.sum(-1) == topk).all()
    sel = sm.bool()
    lo = torch.where(sel, scores, torch.full_like(scores, float("inf"))).amin(-1)
    hi = torch.where(~sel, scores, torch.full_like(scores, float("-inf"))).amax(-1)
    bad = hi > lo
    assert ((hi - lo)[bad] <= 2.0 ** -7 * hi[bad].abs() + 1e-6).all()
    if topk > 1:
        assert (lt[..., 1:] > lt[..., :-1]).all()
    rebuilt = torch.zeros_like(sm)
    rebuilt.scatter_(-1, lt.long(), 1)
    assert torch.equal(rebuilt, sm)


def _ties_only(ours, ref, scores):
    """`ours` and `ref` select the same blocks except where a score sits at the selection threshold."""
    diff = ours.bool() ^ ref.bool()
    if diff.any():
        thr = torch.where(ref.bool(), scores, torch.full_like(scores, float("inf"))).amin(-1, keepdim=True)
        near = (scores - thr).abs() <= 2.0 ** -6 * thr.abs() + 1e-6
        assert (near | ~diff).all(), "block maps differ away from the selection threshold"
        assert diff.float().mean() < 5e-3


@pytest.mark.parametrize("b,l,h,d,ratio", [(1, 600, 2, 128, 0.25), (2, 333, 3, 128, 0.5), (1, 4100, 2, 128, 0.1),
                                           (1, 1000, 2, 64, 0.3), (1, 600, 1, 128, 1.0)])
def test_block_map_hopper_blocks(sm90, b, l, h, d, ratio):
    from turbodiffusion_b200.SLA.utils import block_map_from_pools, get_block_map, quant_qk
    q, k, _ = _qkv(b, l, h, d, 7 + l)
    prep = quant_qk(q.to(sm90), k.to(sm90), blkq=BQ, blkk=BK)
    nblk = (l + 127) // 128
    topk = min(nblk, int(ratio * nblk))
    sparse_map, lut = block_map_from_pools(prep.q_pool, prep.k_pool, topk)
    sm, lt = sparse_map.cpu(), lut.cpu()
    assert sm.shape == (b, h, (l + 63) // 64, nblk)
    # scores from the kernel's own pooled vectors: fp32 dot, rounded to bf16
    scores = (prep.q_pool.cpu().float() @ prep.k_pool.cpu().float().transpose(-1, -2)).to(q.dtype).float()
    _check_topk(scores, sm, lt, topk)
    assert (sm == O.select_topk(scores, topk)[0]).float().mean().item() > 0.999
    # the public entry point, against the oracle's own block map
    qh, kh = q.transpose(1, 2).contiguous(), k.transpose(1, 2).contiguous()
    sm2, _, topk2 = get_block_map(qh.to(sm90), kh.to(sm90), ratio, BQ, BK)
    assert topk2 == topk and torch.equal(sm2.cpu(), sm)
    ref, _, _ = O.get_block_map(qh, kh, ratio, BQ, BK)
    _ties_only(sm, ref, O.pooled_scores(qh, kh, BQ, BK).float())


@pytest.mark.parametrize("name", ["sla_a", "sla_b"])
def test_block_map_hopper_blocks_on_the_golden_inputs(sm90, name):
    from turbodiffusion_b200.SLA.utils import get_block_map
    g = torch.load(os.path.join(GOLD, name + ".pt"))
    qh, kh = g["q"].transpose(1, 2).contiguous(), g["k"].transpose(1, 2).contiguous()
    sparse_map, _, topk = get_block_map(qh.to(sm90), kh.to(sm90), g["topk_ratio"], BQ, BK)
    ref, _, ref_topk = O.get_block_map(qh, kh, g["topk_ratio"], BQ, BK)
    assert topk == ref_topk and (sparse_map.sum(-1) == topk).all()
    _ties_only(sparse_map.cpu(), ref, O.pooled_scores(qh, kh, BQ, BK).float())


CASES = [
    # b, l, h, d, ratio, dtype
    (1, 600, 2, 128, 0.25, torch.bfloat16),   # ragged q tail (600 = 9*64 + 24), k tail of 88 keys; topk 1
    (2, 333, 3, 128, 0.5, torch.bfloat16),    # b = 2, last key block 77 keys
    (1, 1280, 2, 128, 0.3, torch.bfloat16),   # exact multiples, odd topk = 3
    (1, 700, 1, 128, 1.0, torch.bfloat16),    # dense; last key block 60 keys (< 64: a whole half of the tile masked)
    (1, 256, 2, 128, 0.3, torch.bfloat16),    # topk = 1: warpgroup 1 gets no key block
    (1, 1000, 2, 64, 0.5, torch.bfloat16),    # 64-wide heads, topk 4
    (2, 520, 2, 128, 0.4, torch.float16),     # fp16, last key block 8 keys
]


@pytest.mark.parametrize("b,l,h,d,ratio,dtype", CASES)
def test_sage_sla_forward_hopper_blocks_vs_oracle(sm90, b, l, h, d, ratio, dtype):
    q, k, v = _qkv(b, l, h, d, 1000 + l, dtype=dtype)
    mod = _module(d, ratio, sm90, use_bf16=dtype == torch.bfloat16)
    out, sel = mod.forward_with_lut(q.to(sm90), k.to(sm90), v.to(sm90))
    torch.cuda.synchronize()
    nblk = (l + 127) // 128
    assert out.shape == q.shape and out.dtype == dtype and not torch.isnan(out.float()).any()
    assert sel["lut"].shape[2] == (l + 63) // 64 and sel["topk"] == max(1, min(nblk, int(ratio * nblk)))
    lut = sel["lut"].cpu()
    w, bias = mod.proj_l.weight.detach().cpu(), mod.proj_l.bias.detach().cpu()
    exact = O.sla_forward(q, k, v, w, bias, ratio, BQ, BK, dtype=dtype, mode="exact", lut=lut)
    sage = O.sla_forward(q, k, v, w, bias, ratio, BQ, BK, dtype=dtype, mode="sage", lut=lut)
    s_exact, s_sage = O.stats(out.cpu(), exact), O.stats(out.cpu(), sage)
    assert s_exact["cos"] >= 0.999 and s_exact["rel_l2"] <= 2e-2, (s_exact, s_sage)
    assert s_sage["rel_l2"] <= 1e-2, (s_exact, s_sage)


@pytest.mark.parametrize("feature_map,d,l,h,ratio", [("elu", 128, 600, 2, 0.25), ("relu", 128, 333, 3, 0.5),
                                                     ("elu", 64, 700, 2, 0.3)])
def test_sage_sla_feature_maps_hopper_blocks(sm90, feature_map, d, l, h, ratio):
    q, k, v = _qkv(1, l, h, d, 6000 + l + d)
    q = (q.float() * 0.5).bfloat16()
    mod = _module(d, ratio, sm90, seed=8, feature_map=feature_map)
    out, sel = mod.forward_with_lut(q.to(sm90), k.to(sm90), v.to(sm90))
    torch.cuda.synchronize()
    lut = sel["lut"].cpu()
    w, bias = mod.proj_l.weight.detach().cpu(), mod.proj_l.bias.detach().cpu()
    for head in range(h):
        for m in range((l + 63) // 64):
            ref = O.sla_forward_block(q, k, v, w, bias, head, m, lut[0, head, m], BQ, BK, mode="exact", feature_map=feature_map)
            s = O.stats(out[0, m * 64:min(l, (m + 1) * 64), head].cpu(), ref)
            assert s["cos"] >= 0.999 and s["rel_l2"] <= 2e-2, (feature_map, d, head, m, s)


@pytest.mark.parametrize("pattern,qscale,l,h,ratio", [
    ("all", 8.0, 1280, 2, 0.5),
    ("all", 16.0, 700, 1, 1.0),          # ragged q tail (60 rows) and k tail (60 keys)
    ("half_warp", 16.0, 640, 2, 1.0),    # rows 0-7 of every 16-row warp slice are scaled
    ("one_warp", 16.0, 640, 2, 1.0),     # only the first warp's 16 rows of every 64-row query block
    ("ragged_last", 12.0, 1000, 2, 1.0), # the maximum of many rows sits in the ragged LAST key block (104 valid keys)
])
def test_sage_sla_hopper_blocks_large_scores_exercise_the_lazy_rescale(sm90, pattern, qscale, l, h, ratio):
    """The patterns of test_gpu_sla.py's lazy-rescale test on 64 x 128 blocks: running maxima that grow by more than 2^8
    between the key blocks one warpgroup sees, for all rows, part of a warp, one warp, and from the ragged last block."""
    d = 128
    q, k, v = _qkv(1, l, h, d, 4000 + l)
    qf = q.float()
    rows = torch.arange(l)
    if pattern in ("all", "ragged_last"):
        qf = qf * qscale
    elif pattern == "half_warp":
        qf[:, (rows % 16) < 8] *= qscale
    elif pattern == "one_warp":
        qf[:, (rows % 64) < 16] *= qscale
    if pattern == "ragged_last":
        nlast = l - (l // 128) * 128
        u = torch.ones(d) / d ** 0.5
        qf = qf + 2.0 * qscale * u
        kf = k.float()
        kf[:, -nlast:] += 6.0 * u
        k = kf.bfloat16()
    q = qf.bfloat16()
    mod = _module(d, ratio, sm90, seed=6)
    out, sel = mod.forward_with_lut(q.to(sm90), k.to(sm90), v.to(sm90))
    torch.cuda.synchronize()
    assert not torch.isnan(out.float()).any() and not torch.isinf(out.float()).any()
    qh, kh = q.transpose(1, 2).float(), k.transpose(1, 2).float()
    s = (qh @ (kh - kh.mean(-2, keepdim=True)).transpose(-1, -2)) * (d ** -0.5) * 1.4426950408889634
    blk_max = torch.stack([s[..., i:i + 128].amax(-1) for i in range(0, l, 128)], -1)
    run_max = torch.cummax(blk_max, -1).values
    grows = (run_max[..., 1:] - run_max[..., :-1]) > 8
    assert grows.any(-1).float().mean().item() > 0.05
    lut = sel["lut"].cpu()
    w, bias = mod.proj_l.weight.detach().cpu(), mod.proj_l.bias.detach().cpu()
    sage = O.sla_forward(q, k, v, w, bias, ratio, BQ, BK, mode="sage", lut=lut)
    exact = O.sla_forward(q, k, v, w, bias, ratio, BQ, BK, mode="exact", lut=lut)
    s_sage, s_exact = O.stats(out.cpu(), sage), O.stats(out.cpu(), exact)
    assert s_sage["rel_l2"] <= 3e-2, (s_sage, s_exact)
    assert s_exact["cos"] >= 0.99, (s_sage, s_exact)


@pytest.mark.parametrize("l,h,d", [(32760, 12, 128), (32760, 24, 64), (75600, 40, 128)])
def test_full_shapes_hopper_blocks_sampled(sm90, l, h, d):
    """Shapes A (both head splits) and B at topk 0.1: sampled query blocks (first, middle, ragged last) of three heads against
    the per-block oracle on the kernel's own selection."""
    g = torch.Generator(device=sm90).manual_seed(l + h)
    q, k, v = (torch.randn(1, l, h, d, generator=g, device=sm90).bfloat16() for _ in range(3))
    k += torch.randn(1, 1, h, d, generator=g, device=sm90).bfloat16() * 2
    mod = _module(d, 0.1, sm90, seed=9)
    out, sel = mod.forward_with_lut(q, k, v)
    torch.cuda.synchronize()
    mblk = (l + 63) // 64
    assert sel["lut"].shape == (1, h, mblk, int(0.1 * ((l + 127) // 128)))
    w, bias = mod.proj_l.weight.detach().cpu(), mod.proj_l.bias.detach().cpu()
    for head in (0, h // 2, h - 1):
        qc, kc, vc = (t[:, :, head:head + 1].cpu() for t in (q, k, v))
        for m in (0, mblk // 2, mblk - 1):
            ref = O.sla_forward_block(qc, kc, vc, w, bias, 0, m, sel["lut"][0, head, m].cpu(), BQ, BK, mode="exact")
            s = O.stats(out[0, m * 64:min(l, (m + 1) * 64), head].cpu(), ref)
            assert s["cos"] >= 0.999 and s["rel_l2"] <= 2e-2, (l, h, d, head, m, s)


def test_ltx_sm90_call_sequence(sm90):
    """TurboT2AV's _sparse_only_forward on its sm90 branch (ltx_distillation/acceleration.py:286-378): get_block_map(64, 128)
    -> get_vanilla_qk_quant(64, 128) -> block_map_lut_triton -> fused.* -> qattn.*_sm90; with proj_l == 0 it must equal
    SageSparseLinearAttention.forward under "sm90" bit for bit."""
    import turbodiffusion_b200.SLA.core as sla_core
    from turbodiffusion_b200.SLA import SageSparseLinearAttention
    b, l, h, d, topk = 1, 900, 2, 128, 0.3
    q, k, v = (t.to(sm90) for t in _qkv(b, l, h, d, 321))
    assert sla_core.get_cuda_arch(0) == "sm90"
    mod = SageSparseLinearAttention(d, topk).to(sm90)
    want = mod(q, k, v)
    qh, kh, vh = (t.transpose(1, 2).contiguous() for t in (q, k, v))
    sparse_map, _, _ = sla_core.get_block_map(qh, kh, topk_ratio=topk, BLKQ=64, BLKK=128)
    km = kh.mean(dim=-2, keepdim=True)
    q_int8, q_scale, k_int8, k_scale = sla_core.get_vanilla_qk_quant(qh, kh, km, 64, 128)
    assert q_scale.shape[-1] == (l + 63) // 64 and k_scale.shape[-1] == (l + 127) // 128
    lut, valid_block_num = sla_core.block_map_lut_triton(sparse_map)
    assert (valid_block_num == int(topk * ((l + 127) // 128))).all()
    o_s = torch.empty_like(qh)
    padded = (l + 127) // 128 * 128
    v_t = torch.empty((b, h, d, padded), dtype=vh.dtype, device=sm90)
    sla_core.fused.transpose_pad_permute_cuda(vh, v_t, 1)
    v_fp8 = torch.empty(v_t.shape, dtype=torch.float8_e4m3fn, device=sm90)
    v_scale = torch.empty((b, h, d), dtype=torch.float32, device=sm90)
    sla_core.fused.scale_fuse_quant_cuda(v_t, v_fp8, v_scale, l, 2.25, 1)
    pv = torch.full((h,), 1e6, dtype=torch.float32, device=sm90)
    sla_core.qattn.qk_int8_sv_f8_accum_f32_block_sparse_attn_inst_buf_fuse_v_scale_with_pv_threshold_sm90(
        q_int8, k_int8, v_fp8, o_s, lut, valid_block_num, pv, q_scale, k_scale, v_scale, 1, False, 1, 1.0 / d ** 0.5, 0)
    assert torch.equal(o_s.transpose(1, 2).contiguous(), want)
    with pytest.raises(NotImplementedError):
        sla_core.qattn.qk_int8_sv_f16_accum_f16_block_sparse_attn_inst_buf_with_pv_threshold
    with pytest.raises(NotImplementedError):
        sla_core.get_vanilla_qk_quant(qh, kh, km, 64, 64)


@pytest.mark.parametrize("zero_proj", [True, False])
def test_cuda_graph_replay_hopper_blocks(sm90, zero_proj):
    """A captured forward replays what the eager one computes.  The linear-attention moments are accumulated with fp32
    atomics (sla_moments.cu), so with a non-zero proj_l two eager calls may already differ in the last bit; with proj_l == 0
    (the module's initial state) the linear branch adds exact zeros and the output must be bit-identical."""
    b, l, h, d = 1, 2000, 4, 128
    q, k, v = (t.to(sm90) for t in _qkv(b, l, h, d, 77))
    mod = _module(d, 0.2, sm90)
    if zero_proj:
        mod.init_weights_()
    eager = mod(q, k, v)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        mod(q, k, v)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = mod(q, k, v)
    graph.replay()
    torch.cuda.synchronize()
    if zero_proj:
        assert torch.equal(out, eager)
    else:
        s = O.stats(out.cpu(), eager.cpu())
        assert s["rel_l2"] <= 1e-3, s


def test_served_arch_is_restored_after_the_fixture(cuda):
    from turbodiffusion_b200.SLA.utils import get_cuda_arch
    assert get_cuda_arch(0) == "sm100"
