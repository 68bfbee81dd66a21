"""GPU: the W8A8 GEMM's 128x256 output tile at its edges, bit for bit against the CPU oracle.

Each CTA computes 128 rows x 256 columns as two 128-column halves with their own weight block scales.  The cases cover
odd and even counts of 128-row tiles, a last 256-column tile that is partial or holds only one half, the split q/k/v
output, the quantised output with an odd number of 128-column blocks, one and many K-blocks, and CUDA-graph replay.
"""
import pytest
import torch

from oracle import td_oracle as O

pytestmark = pytest.mark.gpu


def _operands(m, n, k, seed, dtype):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(m, k, generator=g)
    x[:, :: max(1, k // 7)] *= 20.0                      # outlier channels: the per-block scales differ
    w = torch.randn(n, k, generator=g) * k ** -0.5
    w[:: 97] *= 8.0                                       # and differ between the two halves of a tile
    bias = torch.randn(n, generator=g).to(dtype)
    a_q, a_s = O.int8_quant(x.to(dtype))
    b_q, b_s = O.int8_quant(w.to(dtype))
    return a_q, a_s, b_q, b_s, bias


def _assert_same_bits(got, ref):
    neq = got.view(torch.int16) != ref.view(torch.int16)
    assert not neq.any(), (f"{neq.sum().item()} / {neq.numel()} outputs differ; max abs "
                           f"{(got.float() - ref.float()).abs().max().item():.4g}; first {neq.nonzero()[:5].tolist()}")


@pytest.mark.parametrize("m,n,k", [
    (384, 384, 256),      # 3 row tiles; the last 256-column tile holds one half
    (4096, 1664, 256),    # 32 row tiles; 13 weight blocks: the last tile holds one half
    (9472, 136, 128),     # 74 row tiles; one K-block; the second half holds 8 columns
    (32760, 256, 384),    # 256 row tiles, ragged last one (32760 % 128 = 120)
    (1, 384, 128),        # one row
    (512, 1536, 256),     # the cross k/v row count
    (256, 384, 8960),     # the FFN-down depth: 70 K-blocks wrap the stage ring many times
])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("with_bias", [False, True])
def test_wide_tile_bit_exact(cuda, m, n, k, dtype, with_bias):
    from turbodiffusion_b200.turbo_diffusion_ops import gemm_cuda, gemm_cuda_swizzle_bias
    a_q, a_s, b_q, b_s, bias = _operands(m, n, k, 7 * m + 3 * n + k, dtype)
    ref = O.int8_gemm(a_q, a_s, b_q, b_s, dtype, bias if with_bias else None)
    c = torch.full((m, n), float("nan"), dtype=dtype, device=cuda)
    dev = [t.to(cuda) for t in (a_q, a_s, b_q, b_s)]
    if with_bias:
        gemm_cuda_swizzle_bias(*dev, c, bias.to(cuda))
    else:
        gemm_cuda(*dev, c)
    torch.cuda.synchronize()
    _assert_same_bits(c.cpu(), ref)


@pytest.mark.parametrize("m,n_part,parts,dtype", [(384, 256, 2, torch.bfloat16), (1000, 256, 3, torch.float16),
                                                 (4096, 512, 3, torch.bfloat16)])
def test_wide_tile_split_output(cuda, m, n_part, parts, dtype):
    from turbodiffusion_b200.turbo_diffusion_ops import gemm_cuda_split
    k = 256
    a_q, a_s, b_q, b_s, bias = _operands(m, parts * n_part, k, 11 * m + parts, dtype)
    ref = O.int8_gemm(a_q, a_s, b_q, b_s, dtype, bias)
    out = gemm_cuda_split(*[t.to(cuda) for t in (a_q, a_s, b_q, b_s, bias)], dtype, parts)
    torch.cuda.synchronize()
    for i in range(parts):
        _assert_same_bits(out[i].cpu(), ref[:, i * n_part:(i + 1) * n_part])


@pytest.mark.parametrize("m,n,k", [(384, 384, 256), (300, 640, 128), (4096, 1664, 384)])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_wide_tile_quantised_output_odd_blocks(cuda, m, n, k, dtype):
    """n = 128 x odd: the last tile's second half is empty, its scale column must still be the first half's alone."""
    from turbodiffusion_b200.turbo_diffusion_ops import gemm_cuda_quant_out
    a_q, a_s, b_q, b_s, bias = _operands(m, n, k, 13 * m + n, dtype)
    q_ref, s_ref = O.int8_quant(O.int8_gemm(a_q, a_s, b_q, b_s, dtype, bias))
    q, s = gemm_cuda_quant_out(*[t.to(cuda) for t in (a_q, a_s, b_q, b_s, bias)], dtype, gelu=False)
    torch.cuda.synchronize()
    assert torch.equal(s.cpu(), s_ref)
    assert torch.equal(q.cpu(), q_ref)


def test_wide_tile_cuda_graph_replay(cuda):
    from turbodiffusion_b200.turbo_diffusion_ops import gemm_cuda_swizzle_bias
    m, n, k = 384, 640, 256
    a_q, a_s, b_q, b_s, bias = _operands(m, n, k, 5, torch.bfloat16)
    dev = [t.to(cuda) for t in (a_q, a_s, b_q, b_s, bias)]
    c = torch.empty(m, n, dtype=torch.bfloat16, device=cuda)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        gemm_cuda_swizzle_bias(*dev[:4], c, dev[4])      # warm-up outside the capture (sets the shared-memory attribute)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        gemm_cuda_swizzle_bias(*dev[:4], c, dev[4])
    c.fill_(float("nan"))
    a_q2, a_s2 = O.int8_quant((torch.randn(m, k) * 3.0).to(torch.bfloat16))
    dev[0].copy_(a_q2.to(cuda))
    dev[1].copy_(a_s2.to(cuda))
    graph.replay()
    torch.cuda.synchronize()
    _assert_same_bits(c.cpu(), O.int8_gemm(a_q2, a_s2, b_q, b_s, torch.bfloat16, bias))
