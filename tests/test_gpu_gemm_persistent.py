"""GPU: the W8A8 GEMM's persistent tile loop, bit for bit against the CPU oracle.

The kernel launches min(tiles, SMs) CTAs and CTA b works through tiles b, b + grid, b + 2 grid, ... of 128 x 256 outputs
with the operand ring, its barrier phases and the quantised epilogue's amax exchange slots carried from tile to tile.
Every case below gives a CTA several different tiles (more tiles than the device has SMs, and not a multiple of them),
which no launch did while a CTA computed one tile and retired: the carried state these cases exercise (ring slot and
phase continuing across tiles, the row-scale variant releasing its last slot, exchange slots reused by a later tile) did
not exist then.  The row count that needed more than 65535 row tiles was refused outright.
"""
import pytest
import torch

from oracle import td_oracle as O

pytestmark = pytest.mark.gpu


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _operands(m, n, k, seed, dtype=torch.bfloat16):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(m, k, generator=g)
    x[:, :: max(1, k // 7)] *= 20.0                      # outlier channels: the per-block scales differ
    x[:: 131] *= 5.0                                      # and differ from row tile to row tile
    w = torch.randn(n, k, generator=g) * k ** -0.5
    w[:: 97] *= 8.0                                       # and between the two halves of a tile
    bias = torch.randn(n, generator=g).to(dtype)
    a_q, a_s = O.int8_quant(x.to(dtype))
    b_q, b_s = O.int8_quant(w.to(dtype))
    return a_q, a_s, b_q, b_s, bias


def _assert_same_bits(got, ref):
    neq = got.view(torch.int16) != ref.view(torch.int16)
    assert not neq.any(), (f"{neq.sum().item()} / {neq.numel()} outputs differ; max abs "
                           f"{(got.float() - ref.float()).abs().max().item():.4g}; first {neq.nonzero()[:5].tolist()}")


def _ragged_rows(row_tiles):
    return 128 * row_tiles - 37


@pytest.mark.parametrize("k_blocks", [1, 5, 70])
def test_several_tiles_per_cta_full_and_half_tiles(cuda, k_blocks):
    """(SMs + 1) ragged row tiles x 3 column tiles of n = 640 (1, 5 K-blocks) or SMs / 2 + 1 row tiles x 2 column tiles of
    n = 384 (70 K-blocks): the tile count exceeds the SM count without being a multiple of it, so a CTA alternates between
    full tiles and tiles whose second half lies past n.  1, 5 and 70 K-blocks are not multiples of the four ring stages,
    so every tile after a CTA's first starts at a ring slot and phase left by the one before."""
    from turbodiffusion_b200.turbo_diffusion_ops import gemm_cuda_swizzle_bias
    sms = _sms()
    m, n = (_ragged_rows(sms + 1), 640) if k_blocks < 70 else (_ragged_rows(sms // 2 + 1), 384)
    assert ((m + 127) // 128) * ((n + 255) // 256) > sms
    a_q, a_s, b_q, b_s, bias = _operands(m, n, 128 * k_blocks, 3 * k_blocks + 1)
    ref = O.int8_gemm(a_q, a_s, b_q, b_s, torch.bfloat16, bias)
    c = torch.full((m, n), float("nan"), dtype=torch.bfloat16, device=cuda)
    gemm_cuda_swizzle_bias(*[t.to(cuda) for t in (a_q, a_s, b_q, b_s)], c, bias.to(cuda))
    torch.cuda.synchronize()
    _assert_same_bits(c.cpu(), ref)


def test_several_tiles_per_cta_split_output(cuda):
    """The q/k/v form: three 256-column parts written as separate matrices, each CTA's tiles falling into different parts."""
    from turbodiffusion_b200.turbo_diffusion_ops import gemm_cuda_split
    m, n_part, parts, k = _ragged_rows(_sms() // 2 + 3), 256, 3, 640
    a_q, a_s, b_q, b_s, bias = _operands(m, parts * n_part, k, 17, torch.float16)
    ref = O.int8_gemm(a_q, a_s, b_q, b_s, torch.float16, bias)
    out = gemm_cuda_split(*[t.to(cuda) for t in (a_q, a_s, b_q, b_s, bias)], torch.float16, parts)
    torch.cuda.synchronize()
    for i in range(parts):
        _assert_same_bits(out[i].cpu(), ref[:, i * n_part:(i + 1) * n_part])


@pytest.mark.parametrize("gelu", [False, True])
def test_several_tiles_per_cta_quantised_output(cuda, gelu):
    """n = 128 x 5: every third tile of a CTA's sequence has one half and so one amax exchange, the case in which a set of
    exchange slots shared by consecutive tiles could be overwritten while a slow warp still reads it.  Without GELU the
    scales and codes equal the oracle's; with it the epilogue's one-MUFU tanh keeps the codes within one of the oracle's
    on under 2 % of the elements (as tests/test_gpu_quant_gemm.py holds it), which a stale amax would break."""
    import torch.nn.functional as F
    from turbodiffusion_b200.turbo_diffusion_ops import gemm_cuda_quant_out
    m, n, k = _ragged_rows(_sms() + 1), 640, 384
    a_q, a_s, b_q, b_s, bias = _operands(m, n, k, 29)
    y = O.int8_gemm(a_q, a_s, b_q, b_s, torch.bfloat16, bias)
    q_ref, s_ref = O.int8_quant(F.gelu(y, approximate="tanh") if gelu else y)
    q, s = gemm_cuda_quant_out(*[t.to(cuda) for t in (a_q, a_s, b_q, b_s, bias)], torch.bfloat16, gelu=gelu)
    torch.cuda.synchronize()
    if gelu:
        assert ((s.cpu() - s_ref).abs() <= 2.0 ** -7 * s_ref).all()
        dq = (q.cpu().to(torch.int16) - q_ref.to(torch.int16)).abs()
        assert dq.max().item() <= 1 and (dq > 0).float().mean().item() < 2e-2, (dq.max().item(), (dq > 0).float().mean().item())
    else:
        assert torch.equal(s.cpu(), s_ref)
        assert torch.equal(q.cpu(), q_ref)


@pytest.mark.parametrize("k", [128, 640])
def test_several_tiles_per_cta_row_scale(cuda, k):
    """The LTX row-scale entry point: its K loop frees a ring slot one K-block late, so the last slot of a tile is freed
    after the loop; a CTA's second tile would wait for ever on a slot that was not."""
    from turbodiffusion_b200 import ltx
    m, n = _ragged_rows(_sms() + 1), 640
    g = torch.Generator().manual_seed(k)
    x = (torch.randn(m, k, generator=g) * 2).bfloat16()
    x[:, ::61] *= 12
    w = (torch.randn(n, k, generator=g) * 0.05).bfloat16()
    bias = torch.randn(n, generator=g).bfloat16()
    xq, xs = O.ltx_row_quant_int8(x)
    wq, ws = O.ltx_row_quant_int8(w)
    ref = O.ltx_gemm_post_scale(xq, xs, wq, ws, bias)
    got = ltx.gemm_int8_post_scale_bias(*[t.to(cuda) for t in (xq, xs, wq, ws, bias)]).cpu()
    _assert_same_bits(got, ref)


def test_several_tiles_per_cta_cuda_graph_replay(cuda):
    from turbodiffusion_b200.turbo_diffusion_ops import gemm_cuda_swizzle_bias
    m, n, k = _ragged_rows(_sms() + 1), 640, 640
    a_q, a_s, b_q, b_s, bias = _operands(m, n, k, 5)
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


def test_more_than_65535_row_tiles(cuda):
    """m = 65537 x 128 - 37 rows used to be refused (the row tiles were a grid dimension); the 1-D persistent grid serves
    it.  The oracle is evaluated on the first, a middle and the last (ragged) row tiles: row tiles are independent."""
    from turbodiffusion_b200.turbo_diffusion_ops import gemm_cuda_swizzle_bias
    row_tiles, n, k = 65537, 8, 128
    m = _ragged_rows(row_tiles)
    g = torch.Generator(device=cuda).manual_seed(1)
    a_q = torch.randint(-128, 128, (m, k), device=cuda, dtype=torch.int8, generator=g)
    a_s = torch.rand(row_tiles, 1, device=cuda, generator=g) * 1e-2 + 1e-3
    b_q = torch.randint(-128, 128, (n, k), device=cuda, dtype=torch.int8, generator=g)
    b_s = torch.rand(1, 1, device=cuda, generator=g) * 1e-2 + 1e-3
    bias = torch.randn(n, device=cuda, generator=g).bfloat16()
    c = torch.full((m, n), float("nan"), dtype=torch.bfloat16, device=cuda)
    gemm_cuda_swizzle_bias(a_q, a_s, b_q, b_s, c, bias)
    torch.cuda.synchronize()
    assert not c.isnan().any()
    for t0, t1 in ((0, 2), (40000, 40003), (row_tiles - 2, row_tiles)):
        rows = slice(128 * t0, min(128 * t1, m))
        ref = O.int8_gemm(a_q[rows].cpu(), a_s[t0:t1].cpu(), b_q.cpu(), b_s.cpu(), torch.bfloat16, bias.cpu())
        _assert_same_bits(c[rows].cpu(), ref)
