"""GPU checks of the SparseLinearAttention training path: the forward with log-sum-exp, gradients of q, k, v and proj_l against
fp32 autograd of the oracle, hand-made block selections, determinism, CUDA-graph capture, path selection and a full-size run.

Bars: o_s and the module output against the reference's goldens cos >= 0.9999, rel-L2 <= 5e-3; lse within 1e-3 (log2 units);
gradients cos >= 0.999 and rel-L2 <= 2e-2 (proj_l: rel-L2 <= 2e-2).  Each gradient case also prints how far a bf16 torch
restatement of the same computation is from the oracle, for context."""
import os

import pytest
import torch
import torch.nn.functional as F

from oracle import td_oracle as O

import sla_backward_oracle as B

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")


def _qkv(b, l, h, d, seed, dtype=torch.bfloat16):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(b, l, h, d, generator=g)
    k = torch.randn(b, l, h, d, generator=g) + torch.randn(1, 1, h, d, generator=g) * 2.0
    v = torch.randn(b, l, h, d, generator=g)
    return q.to(dtype), k.to(dtype), v.to(dtype)


def _module(d, ratio, seed=5, **kw):
    from turbodiffusion_b200.SLA import SparseLinearAttention
    mod = SparseLinearAttention(d, ratio, BLKQ=128, BLKK=64, **kw).cuda()
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        mod.proj_l.weight.copy_(torch.randn(d, d, generator=g) * 0.05)
        mod.proj_l.bias.copy_(torch.randn(d, generator=g) * 0.05)
    return mod


def _bars(got, want, cos=0.999, rel=2e-2, what=""):
    s = O.stats(got.float().cpu(), want.float().cpu())
    assert s["cos"] >= cos and s["rel_l2"] <= rel, (what, s)
    return s


def test_forward_lse_vs_reference_golden(cuda):
    from turbodiffusion_b200.SLA.core import attn_fwd_qk16_lse
    g = torch.load(os.path.join(GOLD, "sla_a.pt"))
    d = g["q"].shape[-1]
    mod = _module(d, g["topk_ratio"])
    with torch.no_grad():
        mod.proj_l.weight.copy_(g["proj_w"])
        mod.proj_l.bias.copy_(g["proj_b"])
    q, k, v = (g[n].cuda() for n in ("q", "k", "v"))
    _, sel = mod.forward_with_lut(q, k, v)
    o_s, lse = attn_fwd_qk16_lse(q, k, v, sel["lut"], sel["topk"], d ** -0.5)
    _bars(o_s.transpose(1, 2), g["o_s"], 0.9999, 5e-3, "o_s")
    qh, kh = (t.transpose(1, 2).contiguous() for t in (g["q"], g["k"]))
    lse_ref = B.sparse_attention_lse(qh, kh, sel["lut"].cpu())
    assert (lse.cpu().double() - lse_ref).abs().max() <= 1e-3
    qg = q.clone().requires_grad_()
    out, sel2 = mod.forward_with_lut(qg, k, v)
    assert out.requires_grad and torch.equal(sel2["lut"], sel["lut"])
    _bars(out, g["out"], 0.9999, 5e-3, "training-path output")


def _linear_exact(qh, kh, vh, w, bias, feature):
    fq, fk = O.feature_maps(feature)
    pq, pk = fq(qh), fk(kh)
    kv = pk.transpose(-1, -2) @ vh
    ks = pk.sum(-2, keepdim=True)
    return ((pq @ kv) / (1e-5 + (pq * ks).sum(-1, keepdim=True))) @ w.t() + bias


def _oracle_grads(q, k, v, w, bias, lut, feature, gout, restate_dtype=None):
    """fp32 autograd of O.sparse_attention + the exact linear branch (restate_dtype: P rounded to that dtype and the linear
    branch at the reference's 16-bit rounding points, on CPU) -> (dq, dk, dv, dw, db) in [B,L,H,D]."""
    leaves = [t.float().clone().requires_grad_() for t in (q, k, v)] + [w.float().clone().requires_grad_(),
                                                                        bias.float().clone().requires_grad_()]
    qf, kf, vf, wf, bf = leaves
    qh, kh, vh = (t.transpose(1, 2) for t in (qf, kf, vf))
    if restate_dtype is None:
        o = O.sparse_attention(qh, kh, vh, lut) + _linear_exact(qh, kh, vh, wf, bf, feature)
    else:
        fq, fk = O.feature_maps(feature)
        qd, kd, vd = (t.to(restate_dtype) for t in (qh, kh, vh))
        o_s = O.sparse_attention(qd, kd, vd, lut, p_dtype=restate_dtype)
        cq, ck = fq(qd).to(restate_dtype), fk(kd).to(restate_dtype)
        o_l = (cq @ (ck.transpose(-1, -2) @ vd)) / (1e-5 + (cq * ck.sum(-2, keepdim=True)).sum(-1, keepdim=True))
        o = o_s + F.linear(o_l, wf.to(restate_dtype), bf.to(restate_dtype)).float()
    (o.transpose(1, 2) * gout.float()).sum().backward()
    return [t.grad for t in leaves]


GRAD_CASES = [
    # b, l, h, ratio, dtype, feature
    ("golden", None, None, None, torch.bfloat16, "softmax"),
    (1, 1000, 2, 0.25, torch.bfloat16, "softmax"),     # ragged tails: 1000 = 7*128 + 104 = 15*64 + 40
    (1, 1280, 2, 0.1, torch.bfloat16, "softmax"),      # exact multiples
    (1, 700, 1, 1.0, torch.bfloat16, "softmax"),       # dense
    (1, 256, 2, 0.3, torch.bfloat16, "softmax"),       # exactly one key block per query block
    (2, 333, 3, 0.5, torch.bfloat16, "softmax"),
    (1, 600, 2, 0.25, torch.float16, "softmax"),
    (1, 600, 2, 0.25, torch.bfloat16, "elu"),
    (1, 600, 2, 0.25, torch.bfloat16, "relu"),
]


@pytest.mark.parametrize("b,l,h,ratio,dtype,feature", GRAD_CASES)
def test_gradients_vs_fp32_oracle(cuda, b, l, h, ratio, dtype, feature):
    d = 128
    if b == "golden":
        gd = torch.load(os.path.join(GOLD, "sla_a.pt"))
        q, k, v, ratio = gd["q"], gd["k"], gd["v"], gd["topk_ratio"]
    else:
        q, k, v = _qkv(b, l, h, d, 300 + l, dtype)
    mod = _module(d, ratio, feature_map=feature, use_bf16=dtype == torch.bfloat16)
    qg, kg, vg = (t.cuda().requires_grad_() for t in (q, k, v))
    out, sel = mod.forward_with_lut(qg, kg, vg)
    gout = torch.randn(out.shape, generator=torch.Generator().manual_seed(9)).to(dtype)
    out.backward(gout.cuda())
    lut = sel["lut"].cpu()
    w, bias = mod.proj_l.weight.detach().cpu(), mod.proj_l.bias.detach().cpu()
    want = _oracle_grads(q, k, v, w, bias, lut, feature, gout)
    restated = _oracle_grads(q, k, v, w, bias, lut, feature, gout, restate_dtype=dtype)
    got = [qg.grad, kg.grad, vg.grad, mod.proj_l.weight.grad, mod.proj_l.bias.grad]
    for name, gt, wt, rs in zip(("dq", "dk", "dv", "dW", "db"), got, want, restated):
        ctx = O.stats(rs, wt)
        if name in ("dW", "db"):
            s = O.stats(gt.float().cpu(), wt)
            assert s["rel_l2"] <= 2e-2, (name, s, "bf16 restatement:", ctx)
        else:
            s = _bars(gt, wt, what=(name, "bf16 restatement:", ctx))
        print(f"{name}: kernel {s['rel_l2']:.2e} (cos {s['cos']:.6f}), restatement {ctx['rel_l2']:.2e}")


def _direct(q, k, v, lut, topk, seed=1):
    from turbodiffusion_b200.SLA.core import attn_bwd_qk16, attn_fwd_qk16_lse
    d = q.shape[-1]
    o_s, lse = attn_fwd_qk16_lse(q, k, v, lut, topk, d ** -0.5)
    d_o = torch.randn(q.shape, generator=torch.Generator().manual_seed(seed)).to(q.dtype).cuda()
    return o_s, lse, d_o, attn_bwd_qk16(q, k, v, o_s, d_o, lse, lut, topk, d ** -0.5)


def _check_blocks(q, k, v, lut, o_s, lse, d_o, grads, heads, q_blocks, k_blocks, b=0):
    """Sampled blocks against the closed-form oracle, given the kernel's lse and delta = rowsum(dO * o_s)."""
    qh, kh, vh, gh = (t.transpose(1, 2).cpu() for t in (q, k, v, d_o))
    delta = (o_s.float() * d_o.float()).sum(-1).transpose(1, 2).cpu()
    lse_c, lut_c = lse.cpu(), lut.cpu()
    dq, dk, dv = (t.transpose(1, 2).cpu() for t in grads)
    l = q.shape[1]
    for hi in heads:
        for mi in q_blocks:
            want = B.sparse_attention_bwd_dq(qh, kh, vh, gh, lut_c, lse_c, delta, b, hi, mi)
            _bars(dq[b, hi, mi * 128:(mi + 1) * 128], want, what=("dq", hi, mi))
        for ni in k_blocks:
            wk, wv = B.sparse_attention_bwd_dkdv(qh, kh, vh, gh, lut_c, lse_c, delta, b, hi, ni)
            gk, gv = dk[b, hi, ni * 64:min(l, (ni + 1) * 64)], dv[b, hi, ni * 64:min(l, (ni + 1) * 64)]
            if not wk.any():
                assert not gk.any() and not gv.any(), ("unselected key block", hi, ni)
                continue
            _bars(gk, wk, what=("dk", hi, ni))
            _bars(gv, wv, what=("dv", hi, ni))


def test_hand_made_luts(cuda):
    """Key block 0 is selected by every query block (the key-major index at its longest list); key blocks 5 and 9 by none,
    so their dk / dv rows must be exactly zero."""
    b, l, h, topk = 1, 1000, 2, 3
    mblk, nblk = 8, 16
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
        assert not dk[:, n * 64:(n + 1) * 64].any() and not dv[:, n * 64:(n + 1) * 64].any()
    _check_blocks(q, k, v, lut, o_s, lse, d_o, grads, range(h), range(mblk), range(nblk))


def test_backward_is_deterministic_and_graph_capturable(cuda):
    from turbodiffusion_b200.SLA.core import attn_bwd_qk16
    b, l, h = 1, 2100, 3
    q, k, v = (t.cuda() for t in _qkv(b, l, h, 128, 11))
    mod = _module(128, 0.2)
    _, sel = mod.forward_with_lut(q, k, v)
    lut, topk = sel["lut"], sel["topk"]
    o_s, lse, d_o, first = _direct(q, k, v, lut, topk)
    second = attn_bwd_qk16(q, k, v, o_s, d_o, lse, lut, topk, 128 ** -0.5)
    for a, c in zip(first, second):
        assert torch.equal(a, c)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        attn_bwd_qk16(q, k, v, o_s, d_o, lse, lut, topk, 128 ** -0.5)   # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = attn_bwd_qk16(q, k, v, o_s, d_o, lse, lut, topk, 128 ** -0.5)
    for t in captured:
        t.zero_()
    graph.replay()
    torch.cuda.synchronize()
    for a, c in zip(first, captured):
        assert torch.equal(a, c)


def test_path_selection(cuda, monkeypatch):
    """Inputs without grad, or grad disabled, run the fused kernel (its linear moments use float atomics, so two fused calls
    are compared for the path taken, not bit for bit); grad-requiring inputs take the training path on the same LUT."""
    import turbodiffusion_b200.SLA.core as core
    fused_calls = []
    real = core.attn_fwd_qk16
    monkeypatch.setattr(core, "attn_fwd_qk16", lambda *a, **kw: fused_calls.append(1) or real(*a, **kw))
    mod = _module(128, 0.25)
    q, k, v = (t.cuda() for t in _qkv(1, 1000, 2, 128, 21))
    fused, sel_inf = mod.forward_with_lut(q, k, v)
    assert fused_calls == [1] and fused.grad_fn is None
    qg, kg, vg = (t.clone().requires_grad_() for t in (q, k, v))
    with torch.no_grad():
        again = mod(qg, kg, vg)
    assert fused_calls == [1, 1] and again.grad_fn is None
    _bars(again, fused, 0.99999, 1e-3, "two fused calls")
    out, sel_train = mod.forward_with_lut(qg, kg, vg)
    assert fused_calls == [1, 1]
    assert out.grad_fn is not None and not torch.equal(out, fused)
    assert torch.equal(sel_train["lut"], sel_inf["lut"]) and sel_train["topk"] == sel_inf["topk"]
    _bars(out, fused, 0.9999, 5e-3, "training vs fused output")
    out.float().square().mean().backward()
    for t in (qg.grad, kg.grad, vg.grad, mod.proj_l.weight.grad, mod.proj_l.bias.grad):
        assert t is not None and torch.isfinite(t).all() and t.abs().sum() > 0


def test_full_size_shape_a(cuda):
    """L = 32760, 12 x 128, top-k 0.1: one forward and backward, then sampled blocks against the closed-form oracle: dQ of the
    first query block and of the ragged last one (120 rows), dK / dV of a key block and of the ragged last one (56 rows)."""
    b, l, h = 1, 32760, 12
    q, k, v = (t.cuda() for t in _qkv(b, l, h, 128, 123))
    mod = _module(128, 0.1)
    qg, kg, vg = (t.clone().requires_grad_() for t in (q, k, v))
    out, sel = mod.forward_with_lut(qg, kg, vg)
    out.float().square().mean().backward()
    for t in (qg.grad, kg.grad, vg.grad, mod.proj_l.weight.grad):
        assert torch.isfinite(t).all()
    lut, topk = sel["lut"], sel["topk"]
    o_s, lse, d_o, grads = _direct(q, k, v, lut, topk)
    mblk, nblk = (l + 127) // 128, (l + 63) // 64
    selected = lut[0, 3].flatten().unique().tolist()
    _check_blocks(q, k, v, lut, o_s, lse, d_o, grads, heads=(0, 7), q_blocks=(0, mblk - 1), k_blocks=(selected[0], nblk - 1))
