"""GPU: where the W8A8 GEMM's epilogue writes, and where it must not.

The epilogue stages each warpgroup's 64 rows of a 128-column half in shared memory and stores them with TMA through a
tensor map over the output: the map, not a per-element predicate, keeps rows >= m, columns >= n and a split output's
ragged last rows out of memory that is not the output's.  Every case here places the output inside a larger buffer
filled with a sentinel byte, checks that no byte outside the output changed, and checks the output itself against the
CPU oracle: bit for bit, except where the oracle's exact tanh stands in for the epilogue's GELU (held to the bounds of
tests/test_gpu_quant_gemm.py).  The staging buffer is reused by a warpgroup's second half and by its next tile; the
cases with one K-block and several tiles per CTA put those epilogues back to back.
"""
import pytest
import torch
import torch.nn.functional as F

from oracle import td_oracle as O

pytestmark = pytest.mark.gpu

PAD = 4096          # sentinel bytes on each side of the output
SENTINEL = 0x5A
GELU = 1            # TDB200_EPILOGUE_GELU_TANH


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _lib():
    from turbodiffusion_b200._lib import DTYPE_TAG, check, lib, ptr, stream_ptr
    return DTYPE_TAG, check, lib(), ptr, stream_ptr


def _inside_sentinel(cuda, shape, dtype):
    """(buffer, output): a contiguous output of `shape` with PAD sentinel bytes before and after it"""
    numel = 1
    for s in shape:
        numel *= s
    nbytes = numel * torch.empty((), dtype=dtype).element_size()
    buf = torch.full((2 * PAD + nbytes,), SENTINEL, dtype=torch.uint8, device=cuda)
    return buf, buf[PAD:PAD + nbytes].view(dtype).view(shape)


def _assert_untouched_outside(buf):
    b = buf.cpu()
    before, after = (b[:PAD] != SENTINEL), (b[-PAD:] != SENTINEL)
    assert not before.any() and not after.any(), (
        f"{before.sum().item()} bytes before and {after.sum().item()} bytes after the output were written")


def _assert_same_bits(got, ref):
    neq = got.view(torch.int16) != ref.view(torch.int16)
    assert not neq.any(), (f"{neq.sum().item()} / {neq.numel()} outputs differ; max abs "
                           f"{(got.float() - ref.float()).abs().max().item():.4g}; first {neq.nonzero()[:5].tolist()}")


def _assert_gelu_close(got, ref):
    """one ulp of T, or 1e-6 absolute where torch's 0.5 x (1 + tanh u) cancels (tests/test_gpu_quant_gemm.py)"""
    diff = (got.float() - ref.float()).abs()
    ok = diff <= torch.maximum(2.0 ** -7 * ref.float().abs(), torch.tensor(1e-6))
    assert ok.all(), (diff[~ok].max().item(), (~ok).sum().item(), (~ok).nonzero()[:5].tolist())


def _assert_codes_close(q, s, q_ref, s_ref):
    assert ((s - s_ref).abs() <= 2.0 ** -7 * s_ref).all()
    dq = (q.to(torch.int16) - q_ref.to(torch.int16)).abs()
    assert dq.max().item() <= 1 and (dq > 0).float().mean().item() < 2e-2, (dq.max().item(), (dq > 0).float().mean().item())


def _block_operands(m, n, k, seed, dtype):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(m, k, generator=g)
    x[:, :: max(1, k // 5)] *= 16.0
    w = torch.randn(n, k, generator=g) * k ** -0.5
    w[:: 53] *= 6.0
    bias = torch.randn(n, generator=g).to(dtype)
    a_q, a_s = O.int8_quant(x.to(dtype))
    b_q, b_s = O.int8_quant(w.to(dtype))
    return a_q, a_s, b_q, b_s, bias


def _run_16bit(cuda, m, n, k, dtype, with_bias, gelu, seed):
    DTYPE_TAG, check, lib, ptr, stream_ptr = _lib()
    a_q, a_s, b_q, b_s, bias = _block_operands(m, n, k, seed, dtype)
    bias = bias if with_bias else None
    dev = [t.to(cuda) for t in (a_q, a_s, b_q, b_s)]
    buf, c = _inside_sentinel(cuda, (m, n), dtype)
    check(lib.tdb200_gemm_w8a8_ex(*[ptr(t) for t in dev], ptr(None if bias is None else bias.to(cuda)), ptr(c),
                                  DTYPE_TAG[dtype], m, n, k, GELU if gelu else 0, stream_ptr(c.device)), "gemm_cuda")
    torch.cuda.synchronize()
    _assert_untouched_outside(buf)
    ref = O.int8_gemm(a_q, a_s, b_q, b_s, dtype, bias)
    if gelu:
        _assert_gelu_close(c.cpu(), F.gelu(ref, approximate="tanh"))
    else:
        _assert_same_bits(c.cpu(), ref)


def _run_quant(cuda, m, n, k, dtype, gelu, seed):
    DTYPE_TAG, check, lib, ptr, stream_ptr = _lib()
    a_q, a_s, b_q, b_s, bias = _block_operands(m, n, k, seed, dtype)
    dev = [t.to(cuda) for t in (a_q, a_s, b_q, b_s, bias)]
    buf, q = _inside_sentinel(cuda, (m, n), torch.int8)
    s = torch.empty((m + 127) // 128, n // 128, dtype=torch.float32, device=cuda)
    check(lib.tdb200_gemm_w8a8_quant_out(*[ptr(t) for t in dev], ptr(q), ptr(s), DTYPE_TAG[dtype], m, n, k,
                                         GELU if gelu else 0, stream_ptr(q.device)), "gemm_cuda_quant_out")
    torch.cuda.synchronize()
    _assert_untouched_outside(buf)
    y = O.int8_gemm(a_q, a_s, b_q, b_s, dtype, bias)
    q_ref, s_ref = O.int8_quant(F.gelu(y, approximate="tanh") if gelu else y)
    if gelu:
        _assert_codes_close(q.cpu(), s.cpu(), q_ref, s_ref)
    else:
        assert torch.equal(s.cpu(), s_ref)
        assert torch.equal(q.cpu(), q_ref)


def _run_row_scale(cuda, m, n, k, dtype, seed):
    DTYPE_TAG, check, lib, ptr, stream_ptr = _lib()
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(m, k, generator=g) * 2).to(dtype)
    x[:, ::61] *= 12
    w = (torch.randn(n, k, generator=g) * 0.05).to(dtype)
    bias = torch.randn(n, generator=g).to(dtype)
    xq, xs = O.ltx_row_quant_int8(x)
    wq, ws = O.ltx_row_quant_int8(w)
    dev = [t.to(cuda) for t in (xq, xs, wq, ws, bias)]
    buf, y = _inside_sentinel(cuda, (m, n), dtype)
    check(lib.tdb200_gemm_w8a8_rowwise(*[ptr(t) for t in dev], ptr(y), DTYPE_TAG[dtype], m, n, k, stream_ptr(y.device)),
          "gemm_w8a8_rowwise")
    torch.cuda.synchronize()
    _assert_untouched_outside(buf)
    _assert_same_bits(y.cpu(), O.ltx_gemm_post_scale(xq, xs, wq, ws, bias, dtype))


# n = 648: the last tile's second half holds 8 columns, so its first 64-column box is clipped and its second lies past n;
# n = 376: the last tile's first half is clipped inside its second box and its second half lies wholly past n
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("n", [376, 648])
@pytest.mark.parametrize("m_rem", [1, 63, 127])
@pytest.mark.parametrize("kind", ["plain", "bias", "gelu", "row_scale"])
def test_ragged_rows_and_columns_16bit(cuda, kind, m_rem, n, dtype):
    m, k = 2 * 128 + m_rem, 256
    if kind == "row_scale":
        _run_row_scale(cuda, m, n, k, dtype, m_rem + n)
    else:
        _run_16bit(cuda, m, n, k, dtype, kind != "plain", kind == "gelu", m_rem + n)


# n = 640: the last tile's second half lies wholly past n (the quantised output needs n % 128 == 0)
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("m_rem", [1, 63, 127])
@pytest.mark.parametrize("gelu", [False, True])
def test_ragged_rows_quantised(cuda, gelu, m_rem, dtype):
    _run_quant(cuda, 2 * 128 + m_rem, 640, 256, dtype, gelu, 7 * m_rem)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("m_rem", [1, 63, 127])
def test_split_output_parts_stay_apart(cuda, m_rem, dtype):
    """Three 256-column parts as separate [m, 256] matrices with ragged m: a part's last row tile must not reach into the
    next part's first rows, nor the last part past the end of the output."""
    DTYPE_TAG, check, lib, ptr, stream_ptr = _lib()
    m, n_part, parts, k = 3 * 128 + m_rem, 256, 3, 384
    a_q, a_s, b_q, b_s, bias = _block_operands(m, parts * n_part, k, 11 + m_rem, dtype)
    dev = [t.to(cuda) for t in (a_q, a_s, b_q, b_s, bias)]
    buf, out = _inside_sentinel(cuda, (parts, m, n_part), dtype)
    check(lib.tdb200_gemm_w8a8_split(*[ptr(t) for t in dev], ptr(out), DTYPE_TAG[dtype], m, parts * n_part, k, parts,
                                     stream_ptr(out.device)), "gemm_cuda_split")
    torch.cuda.synchronize()
    _assert_untouched_outside(buf)
    ref = O.int8_gemm(a_q, a_s, b_q, b_s, dtype, bias)
    for i in range(parts):
        _assert_same_bits(out[i].cpu(), ref[:, i * n_part:(i + 1) * n_part])


@pytest.mark.parametrize("kind", ["bias", "quant", "row_scale"])
def test_back_to_back_epilogues_one_k_block(cuda, kind):
    """One K-block per tile and a little more than 3 x SMs tiles: every CTA runs three tiles (a few run four), each
    epilogue following the last on the same staging buffer after a single K-block, with ragged rows in the last tiles."""
    sms = _sms()
    n, k = 512, 128
    m = 128 * ((3 * sms + 1 + 1) // 2) - 37            # 2 column tiles per row tile
    assert (m + 127) // 128 * 2 >= 3 * sms + 1
    if kind == "bias":
        _run_16bit(cuda, m, n, k, torch.bfloat16, True, False, 1)
    elif kind == "quant":
        _run_quant(cuda, m, n, k, torch.bfloat16, False, 2)
    else:
        _run_row_scale(cuda, m, n, k, torch.float16, 3)


def test_cuda_graph_replay_into_sentinel_buffer(cuda):
    DTYPE_TAG, check, lib, ptr, stream_ptr = _lib()
    m, n, k = 128 * (_sms() + 1) - 63, 648, 256
    a_q, a_s, b_q, b_s, bias = _block_operands(m, n, k, 5, torch.bfloat16)
    dev = [t.to(cuda) for t in (a_q, a_s, b_q, b_s, bias)]
    buf, c = _inside_sentinel(cuda, (m, n), torch.bfloat16)

    def call():
        check(lib.tdb200_gemm_w8a8_ex(*[ptr(t) for t in dev], ptr(c), DTYPE_TAG[torch.bfloat16], m, n, k, 0,
                                      stream_ptr(c.device)), "gemm_cuda")

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        call()                                          # outside the capture: sets the shared-memory attribute
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        call()
    buf.fill_(SENTINEL)
    a_q2, a_s2 = O.int8_quant((torch.randn(m, k, generator=torch.Generator().manual_seed(9)) * 3.0).to(torch.bfloat16))
    dev[0].copy_(a_q2.to(cuda))
    dev[1].copy_(a_s2.to(cuda))
    graph.replay()
    torch.cuda.synchronize()
    _assert_untouched_outside(buf)
    _assert_same_bits(c.cpu(), O.int8_gemm(a_q2, a_s2, b_q, b_s, torch.bfloat16, bias))
