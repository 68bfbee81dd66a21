"""GPU checks of SparseLinearAttention at its default block sizes, BLKQ = 64 and BLKK = 64, with 128-wide heads: the block
map, the fused inference forward for every feature map, and the training path (forward with lse, gradients against fp32
autograd of the oracle, hand-made block selections, determinism, CUDA-graph capture, path selection, a full-size run).

Bars are the ones the (128, 64) path meets: block map equal to the oracle's as a set except at entries within rounding of
the selection threshold (test_gpu_blockmap_golden.py); forward cos >= 0.9999 and rel-L2 <= 5e-3 against the fp32 oracle
and the Triton restatement (test_gpu_sla.py); lse within 1e-3 in log2 units, gradients cos >= 0.999 and rel-L2 <= 2e-2,
proj_l rel-L2 <= 2e-2 (test_gpu_sla_backward.py).  No reference golden exists at (64, 64): parity is pinned through the
oracle alone."""
import pytest
import torch
import torch.nn.functional as F

from oracle import td_oracle as O

import sla_backward_oracle as B

pytestmark = pytest.mark.gpu
BQ, BK = 64, 64


def _qkv(b, l, h, d, seed, dtype=torch.bfloat16):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(b, l, h, d, generator=g)
    k = torch.randn(b, l, h, d, generator=g) + torch.randn(1, 1, h, d, generator=g) * 2.0
    v = torch.randn(b, l, h, d, generator=g)
    return q.to(dtype), k.to(dtype), v.to(dtype)


def _module(ratio, seed=5, **kw):
    from turbodiffusion_b200.SLA import SparseLinearAttention
    mod = SparseLinearAttention(128, ratio, **kw).cuda()     # the constructor's default blocks: (64, 64)
    assert mod.block_sizes(0) == (BQ, BK)
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        mod.proj_l.weight.copy_(torch.randn(128, 128, generator=g) * 0.05)
        mod.proj_l.bias.copy_(torch.randn(128, generator=g) * 0.05)
    return mod


def _bars(got, want, cos=0.999, rel=2e-2, what=""):
    s = O.stats(got.float().cpu(), want.float().cpu())
    assert s["cos"] >= cos and s["rel_l2"] <= rel, (what, s)
    return s


@pytest.mark.parametrize("b,l,h,ratio", [(1, 1000, 2, 0.25), (2, 1280, 3, 0.1), (1, 4096, 2, 0.2)])
def test_block_map_vs_oracle(cuda, b, l, h, ratio):
    """64-row query pools, 64-row pools of the smoothed keys, top-k: the oracle's get_block_map(blkq=64, blkk=64) as a set,
    except at entries whose score is within rounding of the row's selection threshold."""
    q, k, v = _qkv(b, l, h, 128, 50 + l)
    mod = _module(ratio)
    _, sel = mod.forward_with_lut(q.cuda(), k.cuda(), v.cuda())
    qh, kh = (t.transpose(1, 2).contiguous() for t in (q, k))
    ref_map, _, topk = O.get_block_map(qh, kh, ratio, BQ, BK)
    assert sel["topk"] == max(1, topk) and sel["lut"].shape == (b, h, (l + BQ - 1) // BQ, sel["topk"])
    ours = sel["sparse_map"].cpu().bool()
    score = O.pooled_scores(qh, kh, BQ, BK).float()
    srt = torch.sort(score, dim=-1, descending=True).values
    thr = srt[..., topk - 1]
    diff = ours ^ ref_map.bool()
    near = (score - thr[..., None]).abs() <= 2.0 ** -6 * thr[..., None].abs() + 2.0 ** -6 * score.abs().amax(-1, keepdim=True)
    assert (near | ~diff).all(), "block map differs away from the selection threshold"
    assert diff.float().mean() < 2e-3
    assert torch.equal(ours, torch.zeros_like(ours).scatter_(-1, sel["lut"].cpu().long(), True))


def _linear_exact(qh, kh, vh, w, bias, feature):
    fq, fk = O.feature_maps(feature)
    pq, pk = fq(qh), fk(kh)
    kv = pk.transpose(-1, -2) @ vh
    ks = pk.sum(-2, keepdim=True)
    return ((pq @ kv) / (1e-5 + (pq * ks).sum(-1, keepdim=True))) @ w.t() + bias


FWD_CASES = [
    # b, l, h, ratio, dtype, feature
    (1, 1000, 2, 0.25, torch.bfloat16, "softmax"),   # ragged: 1000 = 15*64 + 40
    (2, 1280, 3, 0.1, torch.bfloat16, "softmax"),    # exact multiples, B = 2, H = 3
    (1, 700, 1, 1.0, torch.bfloat16, "softmax"),     # dense
    (1, 1000, 2, 0.25, torch.float16, "softmax"),
    (2, 1000, 3, 0.25, torch.bfloat16, "elu"),
    (1, 1280, 2, 0.3, torch.float16, "elu"),
    (1, 1000, 2, 0.25, torch.bfloat16, "relu"),
    (2, 1280, 3, 0.2, torch.float16, "relu"),
]


@pytest.mark.parametrize("b,l,h,ratio,dtype,feature", FWD_CASES)
def test_inference_forward_vs_oracle(cuda, b, l, h, ratio, dtype, feature):
    """The fused forward (no grad) against the fp32 oracle (exact sparse attention at blkq = blkk = 64 on the module's own
    LUT + the exact linear branch with the module's feature map) and, for softmax, the Triton restatement (P rounded)."""
    q, k, v = _qkv(b, l, h, 128, 2000 + l + h, dtype)
    if feature != "softmax":
        q = (q.float() * 0.5).to(dtype)          # keep elu / relu features in a range where the linear branch matters
    mod = _module(ratio, feature_map=feature, use_bf16=dtype == torch.bfloat16)
    with torch.no_grad():
        out, sel = mod.forward_with_lut(q.cuda(), k.cuda(), v.cuda())
    assert out.dtype == dtype and out.shape == q.shape
    lut = sel["lut"].cpu()
    w, bias = mod.proj_l.weight.detach().cpu(), mod.proj_l.bias.detach().cpu()
    qh, kh, vh = (t.transpose(1, 2).float() for t in (q, k, v))
    exact = (O.sparse_attention(qh, kh, vh, lut, BQ, BK) + _linear_exact(qh, kh, vh, w, bias, feature)).transpose(1, 2)
    s_exact = _bars(out, exact, 0.9999, 5e-3, ("exact", feature, dtype))
    if feature == "softmax":
        tri = O.sla_forward(q, k, v, w, bias, ratio, BQ, BK, dtype=dtype, mode="triton", lut=lut)
        s_tri = O.stats(out.float().cpu(), tri.float())
        assert s_tri["rel_l2"] <= 5e-3, (s_exact, s_tri)


def _oracle_grads(q, k, v, w, bias, lut, feature, gout):
    """fp32 autograd of O.sparse_attention(blkq = blkk = 64) + the exact linear branch -> (dq, dk, dv, dw, db), [B,L,H,D]."""
    leaves = [t.float().clone().requires_grad_() for t in (q, k, v)] + [w.float().clone().requires_grad_(),
                                                                        bias.float().clone().requires_grad_()]
    qf, kf, vf, wf, bf = leaves
    qh, kh, vh = (t.transpose(1, 2) for t in (qf, kf, vf))
    o = O.sparse_attention(qh, kh, vh, lut, BQ, BK) + _linear_exact(qh, kh, vh, wf, bf, feature)
    (o.transpose(1, 2) * gout.float()).sum().backward()
    return [t.grad for t in leaves]


GRAD_CASES = [
    # b, l, h, ratio, dtype, feature  (the case list of test_gpu_sla_backward.py's gradient test, golden input aside)
    (1, 1000, 2, 0.25, torch.bfloat16, "softmax"),     # ragged tails: 1000 = 15*64 + 40
    (1, 1280, 2, 0.1, torch.bfloat16, "softmax"),      # exact multiples
    (1, 700, 1, 1.0, torch.bfloat16, "softmax"),       # dense
    (1, 256, 2, 0.3, torch.bfloat16, "softmax"),       # one key block per query block
    (2, 333, 3, 0.5, torch.bfloat16, "softmax"),
    (1, 600, 2, 0.25, torch.float16, "softmax"),
    (1, 600, 2, 0.25, torch.bfloat16, "elu"),
    (1, 600, 2, 0.25, torch.bfloat16, "relu"),
]


@pytest.mark.parametrize("b,l,h,ratio,dtype,feature", GRAD_CASES)
def test_gradients_vs_fp32_oracle(cuda, b, l, h, ratio, dtype, feature):
    q, k, v = _qkv(b, l, h, 128, 300 + l, dtype)
    mod = _module(ratio, feature_map=feature, use_bf16=dtype == torch.bfloat16)
    qg, kg, vg = (t.cuda().requires_grad_() for t in (q, k, v))
    out, sel = mod.forward_with_lut(qg, kg, vg)
    assert sel["lut"].shape[2] == (l + BQ - 1) // BQ
    gout = torch.randn(out.shape, generator=torch.Generator().manual_seed(9)).to(dtype)
    out.backward(gout.cuda())
    lut = sel["lut"].cpu()
    w, bias = mod.proj_l.weight.detach().cpu(), mod.proj_l.bias.detach().cpu()
    want = _oracle_grads(q, k, v, w, bias, lut, feature, gout)
    got = [qg.grad, kg.grad, vg.grad, mod.proj_l.weight.grad, mod.proj_l.bias.grad]
    for name, gt, wt in zip(("dq", "dk", "dv", "dW", "db"), got, want):
        if name in ("dW", "db"):
            s = O.stats(gt.float().cpu(), wt)
            assert s["rel_l2"] <= 2e-2, (name, s)
        else:
            s = _bars(gt, wt, what=name)
        print(f"{name}: rel-L2 {s['rel_l2']:.2e} (cos {s['cos']:.6f})")


def _direct(q, k, v, lut, topk, seed=1):
    from turbodiffusion_b200.SLA.core import attn_bwd_qk16, attn_fwd_qk16_lse
    o_s, lse = attn_fwd_qk16_lse(q, k, v, lut, topk, 128 ** -0.5, blkq=BQ)
    d_o = torch.randn(q.shape, generator=torch.Generator().manual_seed(seed)).to(q.dtype).cuda()
    return o_s, lse, d_o, attn_bwd_qk16(q, k, v, o_s, d_o, lse, lut, topk, 128 ** -0.5, blkq=BQ)


def _check_blocks(q, k, v, lut, o_s, lse, d_o, grads, heads, q_blocks, k_blocks, b=0):
    """Sampled blocks against the closed-form backward at blkq = 64, given the kernel's lse and delta = rowsum(dO * o_s)."""
    qh, kh, vh, gh = (t.transpose(1, 2).cpu() for t in (q, k, v, d_o))
    delta = (o_s.float() * d_o.float()).sum(-1).transpose(1, 2).cpu()
    lse_c, lut_c = lse.cpu(), lut.cpu()
    dq, dk, dv = (t.transpose(1, 2).cpu() for t in grads)
    l = q.shape[1]
    for hi in heads:
        for mi in q_blocks:
            want = B.sparse_attention_bwd_dq(qh, kh, vh, gh, lut_c, lse_c, delta, b, hi, mi, blkq=BQ)
            _bars(dq[b, hi, mi * BQ:(mi + 1) * BQ], want, what=("dq", hi, mi))
        for ni in k_blocks:
            wk, wv = B.sparse_attention_bwd_dkdv(qh, kh, vh, gh, lut_c, lse_c, delta, b, hi, ni, blkq=BQ)
            gk, gv = dk[b, hi, ni * BK:min(l, (ni + 1) * BK)], dv[b, hi, ni * BK:min(l, (ni + 1) * BK)]
            if not wk.any():
                assert not gk.any() and not gv.any(), ("unselected key block", hi, ni)
                continue
            _bars(gk, wk, what=("dk", hi, ni))
            _bars(gv, wv, what=("dv", hi, ni))


def test_training_forward_lse_and_o_s(cuda):
    from turbodiffusion_b200.SLA.core import attn_fwd_qk16_lse
    b, l, h = 2, 1000, 3
    q, k, v = _qkv(b, l, h, 128, 41)
    mod = _module(0.25)
    _, sel = mod.forward_with_lut(q.cuda(), k.cuda(), v.cuda())
    o_s, lse = attn_fwd_qk16_lse(q.cuda(), k.cuda(), v.cuda(), sel["lut"], sel["topk"], 128 ** -0.5, blkq=BQ)
    qh, kh, vh = (t.transpose(1, 2).contiguous() for t in (q, k, v))
    lut = sel["lut"].cpu()
    _bars(o_s.transpose(1, 2), O.sparse_attention(qh, kh, vh, lut, BQ, BK), 0.9999, 5e-3, "o_s")
    assert (lse.cpu().double() - B.sparse_attention_lse(qh, kh, lut, BQ, BK)).abs().max() <= 1e-3


def test_hand_made_luts(cuda):
    """Key block 0 is selected by every query block (the key-major index at its longest list: 16 entries, both warpgroups
    take eight); key blocks 5 and 9 by none, so their dk / dv rows must be exactly zero.  Ragged tails on both sides."""
    b, l, h, topk = 1, 1000, 2, 3
    mblk, nblk = 16, 16
    q, k, v = (t.cuda() for t in _qkv(b, l, h, 128, 77))
    g = torch.Generator().manual_seed(4)
    others = torch.tensor([n for n in range(1, nblk) if n not in (5, 9)])
    lut = torch.empty(b, h, mblk, topk, dtype=torch.int32)
    for hi in range(h):
        for mi in range(mblk):
            lut[0, hi, mi, 0] = 0
            lut[0, hi, mi, 1:] = others[torch.randperm(len(others), generator=g)[:topk - 1]].sort().values
    lut = lut.cuda()
    o_s, lse, d_o, grads = _direct(q, k, v, lut, topk)
    _, dk, dv = grads
    for n in (5, 9):
        assert not dk[:, n * BK:(n + 1) * BK].any() and not dv[:, n * BK:(n + 1) * BK].any()
    _check_blocks(q, k, v, lut, o_s, lse, d_o, grads, range(h), range(mblk), range(nblk))


def test_backward_is_deterministic_and_graph_capturable(cuda):
    from turbodiffusion_b200.SLA.core import attn_bwd_qk16
    b, l, h = 1, 2100, 3
    q, k, v = (t.cuda() for t in _qkv(b, l, h, 128, 11))
    mod = _module(0.2)
    _, sel = mod.forward_with_lut(q, k, v)
    lut, topk = sel["lut"], sel["topk"]
    o_s, lse, d_o, first = _direct(q, k, v, lut, topk)
    second = attn_bwd_qk16(q, k, v, o_s, d_o, lse, lut, topk, 128 ** -0.5, blkq=BQ)
    for a, c in zip(first, second):
        assert torch.equal(a, c)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        attn_bwd_qk16(q, k, v, o_s, d_o, lse, lut, topk, 128 ** -0.5, blkq=BQ)   # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = attn_bwd_qk16(q, k, v, o_s, d_o, lse, lut, topk, 128 ** -0.5, blkq=BQ)
    for t in captured:
        t.zero_()
    graph.replay()
    torch.cuda.synchronize()
    for a, c in zip(first, captured):
        assert torch.equal(a, c)


def test_path_selection(cuda, monkeypatch):
    """No-grad calls run the fused 16-bit kernel at (64, 64); grad-requiring inputs take the training path on the same LUT."""
    import turbodiffusion_b200.SLA.core as core
    fused_calls = []
    real = core.attn_fwd_qk16
    monkeypatch.setattr(core, "attn_fwd_qk16", lambda *a, **kw: fused_calls.append(kw.get("blkq")) or real(*a, **kw))
    mod = _module(0.25)
    q, k, v = (t.cuda() for t in _qkv(1, 1000, 2, 128, 21))
    fused, sel_inf = mod.forward_with_lut(q, k, v)
    assert fused_calls == [BQ] and fused.grad_fn is None
    qg, kg, vg = (t.clone().requires_grad_() for t in (q, k, v))
    out, sel_train = mod.forward_with_lut(qg, kg, vg)
    assert fused_calls == [BQ]
    assert out.grad_fn is not None
    assert torch.equal(sel_train["lut"], sel_inf["lut"]) and sel_train["topk"] == sel_inf["topk"]
    _bars(out, fused, 0.9999, 5e-3, "training vs fused output")
    out.float().square().mean().backward()
    for t in (qg.grad, kg.grad, vg.grad, mod.proj_l.weight.grad, mod.proj_l.bias.grad):
        assert t is not None and torch.isfinite(t).all() and t.abs().sum() > 0


def test_full_size_shape_a(cuda):
    """L = 32760, 12 x 128, top-k 0.1 (Mblk = 512, last query block 56 rows): one forward and backward, then sampled blocks
    against the closed-form backward: dQ of the first and the ragged last query block, dK / dV of a selected key block and
    of the ragged last one (56 rows)."""
    b, l, h = 1, 32760, 12
    q, k, v = (t.cuda() for t in _qkv(b, l, h, 128, 123))
    mod = _module(0.1)
    qg, kg, vg = (t.clone().requires_grad_() for t in (q, k, v))
    out, sel = mod.forward_with_lut(qg, kg, vg)
    out.float().square().mean().backward()
    for t in (qg.grad, kg.grad, vg.grad, mod.proj_l.weight.grad):
        assert torch.isfinite(t).all()
    lut, topk = sel["lut"], sel["topk"]
    mblk, nblk = (l + BQ - 1) // BQ, (l + BK - 1) // BK
    assert lut.shape == (b, h, mblk, topk) and mblk == 512
    o_s, lse, d_o, grads = _direct(q, k, v, lut, topk)
    selected = lut[0, 3].flatten().unique().tolist()
    _check_blocks(q, k, v, lut, o_s, lse, d_o, grads, heads=(0, 7), q_blocks=(0, mblk - 1), k_blocks=(selected[0], nblk - 1))
