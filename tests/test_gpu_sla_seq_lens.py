"""SparseLinearAttention / SageSparseLinearAttention with per-entry lengths (forward(..., seq_lens=...)) on the GPU.

Entry i's rows below n_i must be byte-identical to the same module called on entry i alone with q, k and v cut to n_i rows, and
its rows past n_i zero, at every served geometry (SageSLA (128, 64) and (64, 128), SLA (128, 64) and (64, 64)), every feature
map and both 16-bit dtypes, with the lengths 0, 1, 63, 64, 65, 127, 128, 129, L - 1 and L in one batch.  The same holds with the
padding filled with large values, NaN and +-inf; full lengths give the bytes of the call without lengths; the LUT and the moments
of the _vl entry points equal the trimmed call's; the padded call without lengths is not the trimmed call (the fault the lengths
remove); device lengths past L are clamped to L, output and reported sparsity alike; a CUDA graph captured with device lengths
replays with new lengths; the padded Wan pair (32760 and 20280 tokens, 12 heads of 128) matches its trimmed calls; and one entry
per module meets the float64 oracle bars of tests/test_gpu_sla.py."""
import pytest
import torch

pytestmark = pytest.mark.gpu

L = 320
LENS = [0, 1, 63, 64, 65, 127, 128, 129, L - 1, L]
GEOMETRIES = [("sage", (128, 64)), ("sage", (64, 128)), ("sla", (128, 64)), ("sla", (64, 64))]


@pytest.fixture(scope="module", autouse=True)
def _built():
    from turbodiffusion_b200 import _build
    _build.build()


def _module(kind, blocks, feature, dtype, topk=0.3, seed=0):
    from turbodiffusion_b200.SLA import core, utils
    if kind == "sage":
        utils.set_served_arch("sm100" if blocks == (128, 64) else "sm90")
        m = core.SageSparseLinearAttention(128, topk, feature, use_bf16=dtype == torch.bfloat16)
    else:
        m = core.SparseLinearAttention(128, topk, feature, BLKQ=blocks[0], BLKK=blocks[1], use_bf16=dtype == torch.bfloat16)
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():   # a live linear branch: proj_l is zero-initialised
        m.proj_l.weight.copy_(torch.randn(128, 128, generator=g) * 0.05)
        m.proj_l.bias.copy_(torch.randn(128, generator=g) * 0.05)
    return m.cuda()


@pytest.fixture(autouse=True)
def _restore_arch():
    from turbodiffusion_b200.SLA import utils
    prev = utils.SERVED_ARCH
    yield
    utils.set_served_arch(prev)


def _inputs(b, l, h, dtype, seed=1):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return [torch.randn(b, l, h, 128, device="cuda", dtype=dtype, generator=g) * s for s in (1.0, 1.0, 1.0)]


def _poison(ts, lens, value):
    out = []
    for t in ts:
        t = t.clone()
        for i, n in enumerate(lens):
            if value == "naninf":
                t[i, n:, :, 0::3] = float("nan")
                t[i, n:, :, 1::3] = float("inf")
                t[i, n:, :, 2::3] = float("-inf")
            else:
                t[i, n:] = value
        out.append(t)
    return out


def _check_against_trimmed(m, q, k, v, lens, out):
    for i, n in enumerate(lens):
        assert torch.all(out[i, n:] == 0), f"entry {i}: rows past {n} are not zero"
        if n == 0:
            continue
        ref = m(q[i:i + 1, :n].contiguous(), k[i:i + 1, :n].contiguous(), v[i:i + 1, :n].contiguous())
        assert torch.equal(out[i:i + 1, :n].view(torch.int16), ref.view(torch.int16)), f"entry {i} (n = {n}) differs"


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("feature", ["softmax", "elu", "relu"])
@pytest.mark.parametrize("kind,blocks", GEOMETRIES)
def test_entries_equal_their_trimmed_calls(kind, blocks, feature, dtype):
    m = _module(kind, blocks, feature, dtype)
    q, k, v = _inputs(len(LENS), L, 2, dtype)
    lens = torch.tensor(LENS, device="cuda")
    with torch.no_grad():
        out, sparsity = m(q, k, v, return_sparsity=True, seq_lens=lens)
        _check_against_trimmed(m, q, k, v, LENS, out)
        for value in (3.0e4, "naninf"):
            qp, kp, vp = _poison((q, k, v), LENS, value)
            assert torch.equal(m(qp, kp, vp, seq_lens=lens).view(torch.int16), out.view(torch.int16)), f"padding {value}"
        mask = torch.arange(L, device="cuda")[None, :] < lens[:, None]
        assert torch.equal(m(q, k, v, seq_lens=mask).view(torch.int16), out.view(torch.int16))
        assert torch.equal(m(q, k, v, seq_lens=lens.cpu()).view(torch.int16), out.view(torch.int16))
    blkk = m.block_sizes(0)[1]
    for i, n in enumerate(LENS):
        nblk = -(-n // blkk)
        want = 0.0 if n == 0 else max(1, min(nblk, int(m.topk * nblk))) / nblk
        assert sparsity.dtype == torch.float64 and sparsity[i].item() == want


@pytest.mark.parametrize("kind,blocks", GEOMETRIES)
def test_full_lengths_give_the_call_without_lengths(kind, blocks):
    m = _module(kind, blocks, "softmax", torch.bfloat16)
    q, k, v = _inputs(3, L, 2, torch.bfloat16)
    with torch.no_grad():
        ref, ref_sparsity = m(q, k, v, return_sparsity=True)
        out = m(q, k, v, seq_lens=torch.full((3,), L, device="cuda"))
        # int32 device lengths past L are clamped to L on the device: the output and the reported sparsity are those of L
        over, over_sparsity = m(q, k, v, return_sparsity=True,
                                seq_lens=torch.tensor([L + 1, 10 * L, 2 ** 31 - 1], device="cuda", dtype=torch.int32))
    assert torch.equal(out.view(torch.int16), ref.view(torch.int16))
    assert torch.equal(over.view(torch.int16), ref.view(torch.int16))
    assert over_sparsity.tolist() == [ref_sparsity] * 3


@pytest.mark.parametrize("kind,blocks", GEOMETRIES)
def test_the_padded_call_without_lengths_is_wrong(kind, blocks):
    m = _module(kind, blocks, "softmax", torch.bfloat16)
    lens = [129, 200]
    q, k, v = _poison(_inputs(2, L, 2, torch.bfloat16), lens, 0.0)   # zero padding: still not harmless
    with torch.no_grad():
        padded = m(q, k, v)
        for i, n in enumerate(lens):
            ref = m(q[i:i + 1, :n].contiguous(), k[i:i + 1, :n].contiguous(), v[i:i + 1, :n].contiguous())
            assert not torch.equal(padded[i:i + 1, :n], ref)


@pytest.mark.parametrize("kind,blocks", GEOMETRIES)
def test_lut_and_moments_equal_the_trimmed_calls(kind, blocks):
    from turbodiffusion_b200.SLA import core, utils
    m = _module(kind, blocks, "softmax", torch.float16)
    blkq, blkk = m.block_sizes(0)
    q, k, v = _poison(_inputs(len(LENS), L, 2, torch.float16), LENS, float("nan"))
    lens = torch.tensor(LENS, device="cuda", dtype=torch.int32)
    nblk = -(-L // blkk)
    topk = max(1, min(nblk, int(m.topk * nblk)))
    topks = utils.seq_topks(lens, m.topk, blkk)
    with torch.no_grad():
        prep = utils.quant_qk_vl(q, k, lens, blkq, blkk)
        smap, lut = utils.block_map_vl(prep.q_pool, prep.k_pool, topk, lens, topks, blkq, blkk)
        kv, ksum = core.linear_moments_vl(k, v, lens, m.feature)
        for i, n in enumerate(LENS):
            mb, nb, tk = -(-n // blkq), -(-n // blkk), int(topks[i])
            assert torch.all(lut[i, :, mb:] == -1) and torch.all(lut[i, :, :mb, tk:] == -1)
            assert torch.all(smap[i, :, mb:] == 0) and torch.all(smap[i, :, :, nb:] == 0)
            if n == 0:
                assert torch.all(kv[i] == 0) and torch.all(ksum[i] == 0)
                continue
            qi, ki, vi = (t[i:i + 1, :n].contiguous() for t in (q, k, v))
            p1 = core.select_prep(qi, ki, blkq, blkk)
            s1, l1 = utils.block_map_from_pools(p1.q_pool, p1.k_pool, tk)
            assert torch.equal(lut[i, :, :mb, :tk], l1[0]) and torch.equal(smap[i, :, :mb, :nb], s1[0])
            kv1, ks1 = core.linear_moments(ki, vi, m.feature)
            assert torch.equal(kv[i], kv1[0]) and torch.equal(ksum[i], ks1[0])


@pytest.mark.parametrize("kind,blocks", [("sage", (128, 64)), ("sla", (64, 64))])
def test_a_captured_graph_replays_with_new_lengths(kind, blocks):
    m = _module(kind, blocks, "softmax", torch.bfloat16)
    q, k, v = _inputs(3, L, 2, torch.bfloat16)
    lens = torch.tensor([L, 100, 1], device="cuda", dtype=torch.int32)
    with torch.no_grad():
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            m(q, k, v, seq_lens=lens)   # warm-up outside the capture
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out = m(q, k, v, seq_lens=lens)
        for new in ([65, L - 1, 0], [1, 129, 256]):
            lens.copy_(torch.tensor(new, dtype=torch.int32))
            graph.replay()
            torch.cuda.synchronize()
            ref = m(q, k, v, seq_lens=torch.tensor(new, device="cuda"))
            assert torch.equal(out.view(torch.int16), ref.view(torch.int16))


@pytest.mark.parametrize("kind,blocks", [("sage", (128, 64)), ("sage", (64, 128)), ("sla", (128, 64))])
def test_the_wan_pair_at_full_size(kind, blocks):
    m = _module(kind, blocks, "softmax", torch.bfloat16, topk=0.1)
    lens = [32760, 20280]
    q, k, v = _poison(_inputs(2, 32760, 12, torch.bfloat16), lens, float("nan"))
    with torch.no_grad():
        out = m(q, k, v, seq_lens=torch.tensor(lens, device="cuda"))
        _check_against_trimmed(m, q, k, v, lens, out)


@pytest.mark.parametrize("kind,blocks", GEOMETRIES)
def test_one_entry_per_module_meets_the_float64_oracle_bars(kind, blocks):
    """Entry 1 of a padded pair (333 of 600 rows, NaN padding) against the CPU oracle in float64 on the kernels' own block
    selection for that entry, with the bars of tests/test_gpu_sla.py: the INT8 modules cos >= 0.999 and rel-L2 <= 2e-2
    against the exact oracle and rel-L2 <= 1e-2 against its Sage INT8 restatement; the 16-bit ones cos >= 0.9999 and rel-L2
    <= 5e-3 against the exact oracle and against its restatement of the Triton path."""
    from oracle import td_oracle as O
    ratio, lens, l, h = 0.25, [600, 333], 600, 2
    m = _module(kind, blocks, "softmax", torch.bfloat16, topk=ratio)
    g = torch.Generator().manual_seed(1333)
    q = torch.randn(2, l, h, 128, generator=g)
    k = torch.randn(2, l, h, 128, generator=g) + torch.randn(1, 1, h, 128, generator=g) * 2.0
    v = torch.randn(2, l, h, 128, generator=g)
    q, k, v = (t.bfloat16() for t in (q, k, v))
    qp, kp, vp = _poison([t.cuda() for t in (q, k, v)], lens, float("nan"))
    m._keep_selection = {}
    try:
        with torch.no_grad():
            out = m(qp, kp, vp, seq_lens=torch.tensor(lens, device="cuda"))
        sel = m._keep_selection
    finally:
        m._keep_selection = None
    blkq, blkk = m.block_sizes(0)
    n = lens[1]
    mb, tk = -(-n // blkq), int(sel["topks"][1])
    lut = sel["lut"][1:2, :, :mb, :tk].cpu()
    qi, ki, vi = (t[1:2, :n].contiguous() for t in (q, k, v))
    w, bias = m.proj_l.weight.detach().cpu(), m.proj_l.bias.detach().cpu()
    got = out[1:2, :n].cpu()
    exact = O.sla_forward(qi, ki, vi, w, bias, ratio, mode="exact", lut=lut, blkq=blkq, blkk=blkk)
    s_exact = O.stats(got, exact)
    if kind == "sage":
        s_emu = O.stats(got, O.sla_forward(qi, ki, vi, w, bias, ratio, mode="sage", lut=lut, blkq=blkq, blkk=blkk))
        assert s_exact["cos"] >= 0.999 and s_exact["rel_l2"] <= 2e-2, (s_exact, s_emu)
        assert s_emu["rel_l2"] <= 1e-2, (s_exact, s_emu)
    else:
        s_emu = O.stats(got, O.sla_forward(qi, ki, vi, w, bias, ratio, mode="triton", lut=lut, blkq=blkq, blkk=blkk))
        assert s_exact["cos"] >= 0.9999 and s_exact["rel_l2"] <= 5e-3, (s_exact, s_emu)
        assert s_emu["rel_l2"] <= 5e-3, (s_exact, s_emu)
