"""GPU parity: a1 int8 block quant and a2 W8A8 wgmma GEMM against the CPU oracle (bit-exact)."""
import pytest
import torch

from oracle import td_oracle as O

pytestmark = pytest.mark.gpu


def _mk(m, k, seed, dtype=torch.bfloat16, outliers=True):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(m, k, generator=g)
    if outliers and k >= 16:
        x[:, :: max(1, k // 7)] *= 20.0  # outlier channels exercise the per-block scales
    return x.to(dtype)


@pytest.mark.parametrize("m,k", [(128, 128), (256, 1536), (120, 256), (1, 128), (333, 640), (513, 136), (7, 8)])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_quant_bit_exact(cuda, m, k, dtype):
    import turbodiffusion_b200.ops as ops
    x = _mk(m, k, 1000 + m + k, dtype)
    q_ref, s_ref = O.int8_quant(x)
    q, s = ops.int8_quant(x.to(cuda))
    torch.cuda.synchronize()
    assert torch.equal(s.cpu(), s_ref), "block scales must be bit-identical"
    assert torch.equal(q.cpu(), q_ref), f"int8 codes differ at {(q.cpu() != q_ref).sum().item()} positions"


def test_quant_zero_block_and_preallocated_outputs(cuda):
    from turbodiffusion_b200.turbo_diffusion_ops import quant_cuda
    x = torch.zeros(256, 256, dtype=torch.bfloat16)
    x[130:, 128:] = _mk(126, 128, 5)
    q_ref, s_ref = O.int8_quant(x)
    q = torch.full((256, 256), 77, dtype=torch.int8, device=cuda)
    s = torch.full((2, 2), -1.0, device=cuda)
    q2, s2 = quant_cuda(x.to(cuda), q, s)
    assert q2.data_ptr() == q.data_ptr() and s2.data_ptr() == s.data_ptr()
    assert torch.equal(q.cpu(), q_ref) and torch.equal(s.cpu(), s_ref)
    assert s_ref[0, 0].item() == pytest.approx(1e-8 / 128)  # amax clamp of an all-zero block


def test_quant_rejects_fp32(cuda):
    from turbodiffusion_b200.turbo_diffusion_ops import quant_cuda
    with pytest.raises(RuntimeError):
        quant_cuda(torch.zeros(128, 128, device=cuda))


GEMM_SHAPES = [
    (128, 256, 128),     # one tile, one K-block
    (128, 256, 512),     # K pipeline wraps the 4-stage ring
    (256, 512, 1536),    # several tiles
    (120, 256, 256),     # ragged M (Wan tail: 32760 % 128 = 120)
    (300, 384, 640),     # ragged M, N not a multiple of the 256 tile
    (129, 136, 128),     # N % 128 != 0 (n % 8 == 0)
    (1, 128, 128),
    (2048, 1536, 1536),  # more tiles (192) than the H100's 132 SMs: more than one wave of CTAs
]


@pytest.mark.parametrize("m,n,k", GEMM_SHAPES)
def test_gemm_bit_exact_vs_oracle(cuda, m, n, k):
    from turbodiffusion_b200.turbo_diffusion_ops import gemm_cuda
    x = _mk(m, k, 11 * m + k)
    w = _mk(n, k, 13 * n + k, outliers=False) * 0.05
    a_q, a_s = O.int8_quant(x)
    b_q, b_s = O.int8_quant(w.to(torch.bfloat16))
    ref = O.int8_gemm(a_q, a_s, b_q, b_s, torch.bfloat16)
    c = torch.full((m, n), float("nan"), dtype=torch.bfloat16, device=cuda)
    gemm_cuda(a_q.to(cuda), a_s.to(cuda), b_q.to(cuda), b_s.to(cuda), c)
    torch.cuda.synchronize()
    got = c.cpu()
    assert not torch.isnan(got.float()).any(), "some outputs were never written"
    neq = (got.view(torch.int16) != ref.view(torch.int16))
    assert not neq.any(), (f"{neq.sum().item()} / {neq.numel()} outputs differ; max abs "
                           f"{(got.float() - ref.float()).abs().max().item():.4g}; first rows {neq.nonzero()[:5].tolist()}")


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_int8_linear_with_bias_matches_module_semantics(cuda, dtype):
    import turbodiffusion_b200.ops as ops
    m, n, k = 200, 384, 256
    x = _mk(m, k, 3, dtype)
    w = (_mk(n, k, 4, dtype, outliers=False).float() * 0.05).to(dtype)
    bias = _mk(1, n, 5, dtype, outliers=False)[0]
    w_q, w_s = O.int8_quant(w)
    ref = O.int8_linear(x, w_q, w_s, bias)
    lin = ops.Int8Linear(k, n, bias=True, dtype=dtype).to(cuda)
    lin.int8_weight.copy_(w_q)
    lin.scale.copy_(w_s)
    lin.bias.copy_(bias)
    got = lin(x.to(cuda).reshape(2, 100, k)).reshape(m, n).cpu()
    assert torch.equal(got.view(torch.int16), ref.view(torch.int16))
    assert sorted(lin.state_dict().keys()) == ["bias", "int8_weight", "scale"]


def test_gemm_unsupported_k_raises(cuda):
    from turbodiffusion_b200.turbo_diffusion_ops import gemm_cuda
    from turbodiffusion_b200._lib import Tdb200Error
    a = torch.zeros(128, 100, dtype=torch.int8, device=cuda)
    s = torch.ones(1, 1, device=cuda)
    c = torch.zeros(128, 128, dtype=torch.bfloat16, device=cuda)
    with pytest.raises(Tdb200Error):
        gemm_cuda(a, s, a, s, c)


def test_gemm_linearity_at_full_wan_shape(cuda):
    """Size-independent property at the BASELINE shape (M=32760, Wan-1.3B q-projection): with unit scales the GEMM is
    an exact integer matmul, so C(A, B1 + B2) == C(A, B1) + C(A, B2) exactly while sums stay below 2^8 (bf16-exact)."""
    from turbodiffusion_b200.turbo_diffusion_ops import gemm_cuda
    m, n, k = 32760, 1536, 1536
    g = torch.Generator(device="cuda").manual_seed(0)
    a = torch.randint(-1, 2, (m, k), generator=g, device=cuda, dtype=torch.int8)
    # sparse +-1 weights keep |dot| small enough to be exactly representable in bf16
    b1 = (torch.rand(n, k, generator=g, device=cuda) < 0.01).to(torch.int8)
    b2 = -(torch.rand(n, k, generator=g, device=cuda) < 0.01).to(torch.int8)
    ones_a = torch.ones((m + 127) // 128, k // 128, device=cuda)
    ones_b = torch.ones(n // 128, k // 128, device=cuda)
    outs = []
    for b in (b1, b2, b1 + b2):
        c = torch.empty(m, n, dtype=torch.bfloat16, device=cuda)
        gemm_cuda(a, ones_a, b.contiguous(), ones_b, c)
        outs.append(c.float())
    assert outs[0].abs().max() < 128
    assert torch.equal(outs[0] + outs[1], outs[2])
    # spot-check 64 random rows against an exact integer matmul
    rows = torch.randint(0, m, (64,), device=cuda)
    ref = (a[rows].float() @ (b1 + b2).float().t())
    assert torch.equal(outs[2][rows], ref)


@pytest.mark.parametrize("m,n,k,gelu", [(300, 512, 256, True), (128, 256, 128, False), (1000, 1280, 384, True)])
def test_gemm_with_fused_quantised_output_is_bit_exact(cuda, m, n, k, gelu):
    """(q, s) from the fused epilogue == quant_cuda(act(gemm + bias)) of the unfused kernels, and == the oracle."""
    from turbodiffusion_b200.turbo_diffusion_ops import (gemm_cuda_bias_gelu, gemm_cuda_quant_out, gemm_cuda_swizzle_bias,
                                                         quant_cuda)
    x = _mk(m, k, 21 * m + k)
    w = (_mk(n, k, 23 * n + k, outliers=False).float() * 0.05).to(torch.bfloat16)
    bias = _mk(1, n, 9, outliers=False)[0]
    a_q, a_s = O.int8_quant(x)
    b_q, b_s = O.int8_quant(w)
    dev = [t.to(cuda) for t in (a_q, a_s, b_q, b_s, bias)]
    q, s = gemm_cuda_quant_out(*dev, torch.bfloat16, gelu=gelu)
    c = torch.empty(m, n, dtype=torch.bfloat16, device=cuda)
    (gemm_cuda_bias_gelu if gelu else gemm_cuda_swizzle_bias)(dev[0], dev[1], dev[2], dev[3], c, dev[4])
    q2, s2 = quant_cuda(c)
    torch.cuda.synchronize()
    if gelu:
        # the quantised-output epilogue evaluates tanh with one MUFU (absolute error 2^-11, far below the int8 step), the
        # 16-bit epilogue uses the 1-ulp sigmoid form: codes may differ by one on a small fraction of the elements
        dq = (q.to(torch.int16) - q2.to(torch.int16)).abs()
        assert dq.max().item() <= 1 and (dq > 0).float().mean().item() < 2e-2
        assert ((s - s2).abs() <= 2.0 ** -7 * s2).all()
    else:
        assert torch.equal(s, s2) and torch.equal(q, q2)
    if not gelu:  # the oracle's GELU uses the exact tanh; the plain path is bit-exact end to end
        y = O.int8_gemm(a_q, a_s, b_q, b_s, torch.bfloat16, bias)
        q_ref, s_ref = O.int8_quant(y)
        assert torch.equal(s.cpu(), s_ref) and torch.equal(q.cpu(), q_ref)


@pytest.mark.parametrize("m,n,k", [(300, 512, 256), (1000, 1280, 384)])
def test_gelu_epilogue_vs_oracle_gelu(cuda, m, n, k):
    """The fused GELU(tanh) epilogue against the ORACLE's GELU (torch's fp32 tanh on the bf16 pre-activation, the value
    nn.GELU(approximate="tanh") produces for a bf16 tensor, rcm/networks/wan2pt1.py:375).  The 16-bit epilogue evaluates
    x * sigmoid(2u): every output is within ONE bf16 ulp of the oracle (or 1e-6 absolute in the cancelling negative tail),
    more than 99 % of the non-tiny values are bit-identical.  The quantised-output epilogue uses the one-MUFU tanh: its int8
    codes differ by at most one code on a small fraction of the elements and the block scales are within one bf16 ulp of
    the oracle's (the scale is amax/128 of bf16 values).  The one-pass gelu_quant kernel is held to the same bound."""
    import torch.nn.functional as F
    from turbodiffusion_b200.turbo_diffusion_ops import gemm_cuda_bias_gelu, gemm_cuda_quant_out
    x = _mk(m, k, 31 * m + k)
    w = (_mk(n, k, 37 * n + k, outliers=False).float() * 0.05).to(torch.bfloat16)
    bias = _mk(1, n, 11, outliers=False)[0]
    a_q, a_s = O.int8_quant(x)
    b_q, b_s = O.int8_quant(w)
    dev = [t.to(cuda) for t in (a_q, a_s, b_q, b_s, bias)]
    c = torch.empty(m, n, dtype=torch.bfloat16, device=cuda)
    gemm_cuda_bias_gelu(dev[0], dev[1], dev[2], dev[3], c, dev[4])
    pre = O.int8_gemm(a_q, a_s, b_q, b_s, torch.bfloat16, bias)           # bit-exact pre-activation (tested above)
    ref = F.gelu(pre, approximate="tanh")                                   # bf16 in, fp32 opmath, bf16 out
    got = c.cpu()
    # torch evaluates 0.5 x (1 + tanh(u)) in fp32: in the negative tail 1 + tanh(u) cancels and torch's own result is only
    # good to ~1e-7 absolute; the kernel evaluates x * sigmoid(2u) (no cancellation).  So: one ulp of T (<= 2^-7 relative for
    # an 8-bit significand), or 1e-6 absolute.
    diff = (got.float() - ref.float()).abs()
    ok = diff <= torch.maximum(2.0 ** -7 * ref.float().abs(), torch.tensor(1e-6))
    assert ok.all(), (diff[~ok].max().item(), (~ok).sum().item())
    big = ref.float().abs() > 1e-3
    same = got.view(torch.int16)[big] == ref.view(torch.int16)[big]
    assert same.float().mean().item() > 0.99
    q, s = gemm_cuda_quant_out(*dev, torch.bfloat16, gelu=True)
    q_ref, s_ref = O.int8_quant(ref)
    torch.cuda.synchronize()
    assert ((s.cpu() - s_ref).abs() <= 2.0 ** -7 * s_ref).all()
    dq = (q.cpu().to(torch.int16) - q_ref.to(torch.int16)).abs()
    assert dq.max().item() <= 1 and (dq > 0).float().mean().item() < 2e-2, (dq.max().item(), (dq > 0).float().mean().item())
    # the split path: T(acc + bias) from the GEMM, then GELU + quantisation in one pass
    from turbodiffusion_b200.turbo_diffusion_ops import gelu_quant_cuda, gemm_cuda_swizzle_bias
    c2 = torch.empty(m, n, dtype=torch.bfloat16, device=cuda)
    gemm_cuda_swizzle_bias(dev[0], dev[1], dev[2], dev[3], c2, dev[4])
    assert torch.equal(c2.cpu().view(torch.int16), pre.view(torch.int16))
    q3, s3 = gelu_quant_cuda(c2)
    dq3 = (q3.cpu().to(torch.int16) - q_ref.to(torch.int16)).abs()
    assert dq3.max().item() <= 1 and (dq3 > 0).float().mean().item() < 2e-2, (dq3.max().item(), (dq3 > 0).float().mean().item())
    assert ((s3.cpu() - s_ref).abs() <= 2.0 ** -7 * s_ref).all()


@pytest.mark.parametrize("m,n_part,k,parts,dtype", [(1000, 256, 384, 3, torch.bfloat16), (130, 512, 128, 2, torch.float16),
                                                   (32760, 1536, 1536, 3, torch.bfloat16)])
def test_split_output_gemm_equals_the_separate_gemms(cuda, m, n_part, k, parts, dtype):
    """f2: one GEMM against row-concatenated projection weights, outputs as `parts` contiguous matrices (the fused q/k/v of
    block.py; packing of acceleration.py:836-860) == the projections' own GEMMs bit for bit, including the ragged last row
    tile of every part (the 3-D store map clips rows past m per part)."""
    from turbodiffusion_b200 import ops
    from turbodiffusion_b200.turbo_diffusion_ops import gemm_cuda_split, gemm_cuda_swizzle_bias
    g = torch.Generator().manual_seed(m + parts)
    x = torch.randn(m, k, generator=g).to(dtype).to(cuda)
    xq, xs = ops.int8_quant(x)
    ws = [ops.int8_quant((torch.randn(n_part, k, generator=g) * k ** -0.5).to(dtype).to(cuda)) for _ in range(parts)]
    bs = [(torch.randn(n_part, generator=g) * 0.1).to(dtype).to(cuda) for _ in range(parts)]
    guard = torch.full((parts + 1, m, n_part), 7.0, dtype=dtype, device=cuda)       # detects writes past the last part
    fused = gemm_cuda_split(xq, xs, torch.cat([w[0] for w in ws]), torch.cat([w[1] for w in ws]), torch.cat(bs), dtype, parts)
    assert fused.shape == (parts, m, n_part) and fused.is_contiguous()
    for i in range(parts):
        y = torch.empty(m, n_part, dtype=dtype, device=cuda)
        gemm_cuda_swizzle_bias(xq, xs, ws[i][0], ws[i][1], y, bs[i])
        assert torch.equal(fused[i], y), i
    assert (guard == 7.0).all()
    with pytest.raises(RuntimeError):
        gemm_cuda_split(xq, xs, torch.cat([w[0] for w in ws])[: parts * n_part - 128], torch.cat([w[1] for w in ws])[:-1],
                        None, dtype, parts)       # parts must be equal multiples of 256 columns
