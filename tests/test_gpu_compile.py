"""The tdb200:: custom operators on the H100: torch.library.opcheck of every op (the sparse attention's autograd formula
included), and torch.compile'd modules against their eager runs."""
import pytest
import torch

from oracle import td_oracle as O

from test_gpu_sla_backward import _bars, _linear_exact, _oracle_grads, _qkv
from test_gpu_sla_q64_16bit import _oracle_grads as _oracle_grads_q64

pytestmark = pytest.mark.gpu


def _r(*shape, dtype=torch.bfloat16, scale=1.0, seed=0):
    g = torch.Generator().manual_seed(seed + sum(shape))
    return (torch.randn(*shape, generator=g) * scale).to(dtype).cuda()


def _opcheck_samples():
    from turbodiffusion_b200 import _ops
    f32 = torch.float32
    m, k, n = 300, 256, 384
    x = _r(m, k)
    a_q, a_s = _ops.quant_int8_block128(x)
    w_q, w_s = _ops.quant_int8_block128(_r(n, k, scale=0.05))
    w3_q, w3_s = _ops.quant_int8_block128(_r(3 * 256, k, scale=0.05, seed=1))
    bias = _r(n, scale=0.02)
    vec = lambda s: _r(k, dtype=f32, scale=0.1, seed=s)  # noqa: E731
    xs, xf = _r(m, k, seed=3), _r(m, k, dtype=f32)
    _, stats = _ops.gate_residual_stats(x, xs, None, 1e-6)
    ang = _r(m, 64, dtype=f32)
    table = torch.stack((ang.cos(), ang.sin()), -1).contiguous()
    lx, tab, ts = _r(2, 37, 256), _r(6, 256, dtype=f32, scale=0.1), _r(2, 1, 6 * 256, scale=0.1)
    cs = _r(2, 4, 37, 32, scale=0.5)
    r_q, r_s = _ops.quant_int8_rowwise(x)
    rw_q, rw_s = _ops.quant_int8_rowwise(_r(n, k, scale=0.05))
    s = [
        (_ops.quant_int8_block128, (x,)),
        (_ops.quant_int8_block128_out, (x, torch.empty_like(a_q), torch.empty_like(a_s))),
        (_ops.gelu_quant_int8_block128, (x,)),
        (_ops.gemm_w8a8, (a_q, a_s, w_q, w_s, bias, 0, torch.empty(m, n, dtype=torch.bfloat16, device="cuda"))),
        (_ops.gemm_w8a8, (a_q, a_s, w_q, w_s, bias, 1, torch.empty(m, n, dtype=torch.bfloat16, device="cuda"))),
        (_ops.gemm_w8a8, (a_q, a_s, w_q, w_s, None, 0, torch.empty(m, n, dtype=torch.float16, device="cuda"))),
        (_ops.gemm_w8a8_split, (a_q, a_s, w3_q[:512].contiguous(), w3_s[:4].contiguous(), None, torch.bfloat16, 2)),
        (_ops.gemm_w8a8_split, (a_q, a_s, w3_q, w3_s, _r(768, scale=0.02), torch.bfloat16, 3)),
        (_ops.gemm_w8a8_quant_out, (a_q, a_s, w_q, w_s, bias, torch.bfloat16, True)),
        (_ops.rms_norm_f32, (xf, vec(1), 1e-6, torch.empty_like(xf))),
        (_ops.layer_norm_f32, (xf, vec(1), vec(2), 1e-6, torch.empty_like(xf))),
        (_ops.rms_norm, (x, vec(1), 1e-6)),
        (_ops.layer_norm, (x, vec(1), vec(2), 1e-6)),
        (_ops.layer_norm_modulate, (x, vec(1), vec(2), 1e-6)),
        (_ops.layer_norm_modulate_quant, (x, vec(1), vec(2), 1e-6)),
        (_ops.layer_norm_modulate_quant_stats, (x, stats, vec(1), vec(2))),
        (_ops.gate_residual, (x, xs, vec(3))),
        (_ops.gate_residual_stats, (x, xs, vec(3), 1e-6)),
        (_ops.rope_interleaved, (_r(m, 2, 128), ang)),
        (_ops.rms_norm_rope, (x, vec(4), ang, 1e-6, 2)),
        (_ops.rms_norm_rope_table, (x, vec(4), table, 1e-6, 2)),
        (_ops.ltx_modulated_rms_norm_ada, (lx, tab, ts, 1, 0, 6, 1e-6)),
        (_ops.ltx_modulate_ada, (lx, tab, ts, 4, 3, 6)),
        (_ops.ltx_gated_residual_ada, (lx, _r(2, 37, 256, seed=5), tab, ts, 2, 6)),
        (_ops.ltx_split_rope, (lx, cs, _r(2, 4, 37, 32, scale=0.5, seed=6))),
        (_ops.quant_int8_rowwise, (x,)),
        (_ops.quant_int8_rowwise_out, (x, torch.empty_like(r_q), torch.empty_like(r_s))),
        (_ops.gemm_w8a8_rowwise, (r_q, r_s, rw_q, rw_s, bias, torch.bfloat16)),
    ]
    b, l, h = 1, 1000, 2
    for d in (64, 128):
        q, kk, v = _r(b, l, h, d, seed=7), _r(b, l, h, d, seed=8), _r(b, l, h, d, seed=9)
        for blkq, blkk in ((128, 64), (64, 128)):
            prep = _ops.sla_quant_qk(q, kk, l, blkq, blkk)
            kmean, q_i8, q_scale, k_i8, k_scale, q_pool, k_pool = prep
            topk = 3
            sm, lut = _ops.sla_block_map(q_pool, k_pool, topk)
            buf = _ops.sla_linear_moments(kk, v, 0)
            kv, ksum = buf[: b * h * d * d].view(b, h, d, d), buf[b * h * d * d:].view(b, h, d)
            kvw = _ops.sla_project_moments(_r(d, d, dtype=f32, scale=0.05), kv, torch.bfloat16)
            s += [(_ops.sla_quant_qk, (q, kk, l, blkq, blkk)), (_ops.sla_quant_q, (q, blkq)), (_ops.sla_quant_k, (kk, l, blkk)),
                  (_ops.sla_block_map, (q_pool, k_pool, topk)),
                  (_ops.sla_attn_fwd, (q_i8, q_scale, k_i8, k_scale, v, q, lut, topk, kvw, ksum, _r(d, dtype=f32), d ** -0.5, l,
                                       0, blkq, blkk, False))]
        s += [(_ops.sla_linear_moments, (kk, v, 1)), (_ops.sla_project_moments, (_r(d, d, dtype=f32), kv, torch.bfloat16))]
    d = 128
    for blkq in (128, 64):
        q_i8, q_scale, q_pool = _ops.sla_quant_q(q, blkq)
        _, _, _, k_pool = _ops.sla_quant_k(kk, l, 64)
        _, lut = _ops.sla_block_map(q_pool, k_pool, 4)
        s.append((_ops.sla_attn16_fwd, (q, kk, v, lut, 4, kvw, ksum, _r(d, dtype=f32), d ** -0.5, l, 0, blkq)))
        qg, kg, vg = (t.clone().requires_grad_() for t in (q, kk, v))
        s.append((_ops.sla_attn16_fwd_lse, (qg, kg, vg, lut, 4, d ** -0.5, blkq)))
        o_s, lse = _ops.sla_attn16_fwd_lse(q, kk, v, lut, 4, d ** -0.5, blkq)
        s.append((_ops.sla_attn16_bwd, (q, kk, v, o_s, _r(b, l, h, d, seed=10), lse, lut, 4, d ** -0.5, blkq)))
    return s


def test_opcheck_every_op(cuda):
    samples = _opcheck_samples()
    assert {op._schema.name for op, _ in samples} == {f"tdb200::{n}" for n in dir(torch.ops.tdb200)
                                                      if isinstance(getattr(torch.ops.tdb200, n), torch._ops.OpOverloadPacket)}
    for op, args in samples:
        if op is torch.ops.tdb200.sla_linear_moments.default:
            # the moments are accumulated with floating-point atomics: two runs differ in the last bits, which the AOT
            # dispatch test's exact output comparison would report; schema, fake kernel and autograd checks still run
            torch.library.opcheck(op, args, test_utils=("test_schema", "test_autograd_registration", "test_faketensor"))
        else:
            torch.library.opcheck(op, args)


# ------------------------------------------------------------------------------------------------ compiled vs eager
def _same(a, b):
    if a.dtype in (torch.bfloat16, torch.float16):
        return torch.equal(a.view(torch.int16), b.view(torch.int16))
    return torch.equal(a, b)


def _close(a, b, rel=1e-3):
    return ((a.float() - b.float()).norm() / b.float().norm()).item() <= rel


def _breaks(fn, *args):
    torch._dynamo.reset()
    return torch._dynamo.explain(fn)(*args).graph_break_count


# The linear-attention moments are accumulated with floating-point atomics (csrc/sla_moments.cu), so with a nonzero
# proj_l.weight two eager runs differ in the last bits too.  With proj_l.weight = 0 (the modules' initialisation) the linear
# branch is exactly proj_l.bias and every other kernel is deterministic: compiled and eager must then agree bit for bit.
@pytest.mark.parametrize("proj_w", ["zero", "random"])
def test_wan_block_compiled_matches_eager_at_a_ragged_length(cuda, proj_w):
    from turbodiffusion_b200.block import WanBlockB200, random_block_state
    dim, heads, l, lc = 512, 4, 1000, 77
    check = _same if proj_w == "zero" else _close
    for attention in ("sagesla", "sla"):
        blk = WanBlockB200(random_block_state(dim, 1024, heads, seed=3, device=cuda), dim, heads, topk=0.3, attention=attention)
        if proj_w == "zero":
            with torch.no_grad():
                blk.sla.proj_l.weight.zero_()
        x, e0, ctx = _r(l, dim, seed=1), _r(6, dim, dtype=torch.float32, scale=0.1), _r(lc, dim, seed=2)
        ang = O.wan_rope_angles(4, 10, 25, dim // heads).cuda()
        ref = blk(x, e0, ang, ctx)
        assert _breaks(blk.forward, x, e0, ang, ctx) == 0
        torch._dynamo.reset()
        got = torch.compile(blk.forward, fullgraph=True)(x, e0, ang, ctx)
        assert check(got, ref), attention
        ro = torch.compile(blk.forward, mode="reduce-overhead", fullgraph=True)
        for _ in range(3):
            out = ro(x, e0, ang, ctx)
            assert check(out, ref), (attention, "reduce-overhead replay")


def test_linear_and_norm_modules_compiled_are_bit_identical(cuda):
    import turbodiffusion_b200.ops as ops
    from turbodiffusion_b200.ltx import PostScaleInt8Linear
    lin = torch.nn.Linear(512, 768).cuda().bfloat16()
    ln = torch.nn.LayerNorm(512).cuda()
    with torch.no_grad():
        ln.weight.normal_(1, 0.1), ln.bias.normal_(0, 0.1)
    rms = ops.FastRMSNorm(512).cuda()
    with torch.no_grad():
        rms.weight.normal_(1, 0.1)
    mods = [ops.Int8Linear.from_linear(lin), rms, ops.FastLayerNorm.from_layernorm(ln).cuda(), ops.FastLayerNorm(512).cuda(),
            PostScaleInt8Linear.from_linear(lin)]
    x = _r(2, 333, 512)
    for m in mods:
        for inp in (x, x.float()) if not isinstance(m, (ops.Int8Linear, PostScaleInt8Linear)) else (x,):
            ref = m(inp)
            assert _breaks(m, inp) == 0, type(m).__name__
            torch._dynamo.reset()
            assert _same(torch.compile(m, fullgraph=True)(inp), ref), type(m).__name__


SLA_CASES = [("sla", dict(BLKQ=128, BLKK=64), d, fm) for d in (64, 128) for fm in ("softmax", "elu", "relu")]
SLA_CASES += [("sla", dict(BLKQ=64, BLKK=64), 128, fm) for fm in ("softmax", "elu", "relu")]
SLA_CASES += [("sagesla-" + arch, {}, d, "softmax") for arch in ("sm100", "sm90") for d in (64, 128)]


@pytest.mark.parametrize("kind,kw,d,fm", SLA_CASES)
def test_sla_inference_compiled_matches_eager(cuda, kind, kw, d, fm):
    from turbodiffusion_b200.SLA import SageSparseLinearAttention, SparseLinearAttention
    from turbodiffusion_b200.SLA.utils import set_served_arch
    prev = set_served_arch(kind.split("-")[1] if kind.startswith("sagesla") else "sm100")
    try:
        cls = SparseLinearAttention if kind == "sla" else SageSparseLinearAttention
        m = cls(d, 0.25, feature_map=fm, **kw).cuda()
        q, k, v = (t.cuda() for t in _qkv(1, 1000, 2, d, 11))
        with torch.no_grad():
            m.proj_l.bias.normal_(0, 0.05)                 # proj_l.weight stays 0: bit-identical (see above)
            ref = m(q, k, v)
            assert _breaks(m, q, k, v) == 0
            torch._dynamo.reset()
            cm = torch.compile(m, fullgraph=True)
            assert _same(cm(q, k, v), ref)
            m.proj_l.weight.normal_(0, 0.05)
            assert _close(cm(q, k, v), m(q, k, v))
    finally:
        set_served_arch(prev)


@pytest.mark.parametrize("blkq", [128, 64])
def test_sparse_branch_compiled_is_bit_identical_with_gradients(cuda, blkq):
    from turbodiffusion_b200.SLA.core import attn_fwd_qk16_lse
    from turbodiffusion_b200.SLA import SparseLinearAttention
    q, k, v = (t.cuda() for t in _qkv(1, 1000, 2, 128, 13))
    _, sel = SparseLinearAttention(128, 0.25, BLKQ=blkq, BLKK=64).cuda().forward_with_lut(q, k, v)
    gout = _r(1, 1000, 2, 128, seed=21)

    def f(q, k, v, lut):
        o_s, lse = attn_fwd_qk16_lse(q, k, v, lut, sel["topk"], 128 ** -0.5, blkq)
        return o_s, lse

    results = []
    torch._dynamo.reset()
    for fn in (f, torch.compile(f, fullgraph=True)):
        qg, kg, vg = (t.clone().requires_grad_() for t in (q, k, v))
        o_s, lse = fn(qg, kg, vg, sel["lut"])
        o_s.backward(gout)
        results.append([o_s.detach(), lse.detach(), qg.grad, kg.grad, vg.grad])
    for name, a, b in zip(("o_s", "lse", "dq", "dk", "dv"), *results):
        assert _same(a, b), name


@pytest.mark.parametrize("blk", [dict(BLKQ=128, BLKK=64), dict(BLKQ=64, BLKK=64)])
@pytest.mark.parametrize("feature", ["softmax", "elu"])
def test_sla_training_compiled_within_the_training_bars(cuda, blk, feature):
    from turbodiffusion_b200.SLA import SparseLinearAttention
    d, ratio = 128, 0.25
    q, k, v = _qkv(1, 1000, 2, d, 1300)
    mod = SparseLinearAttention(d, ratio, feature_map=feature, **blk).cuda()
    g = torch.Generator().manual_seed(5)
    with torch.no_grad():
        mod.proj_l.weight.copy_(torch.randn(d, d, generator=g) * 0.05)
        mod.proj_l.bias.copy_(torch.randn(d, generator=g) * 0.05)
    with torch.no_grad():
        _, sel = mod.forward_with_lut(q.cuda(), k.cuda(), v.cuda())       # the selection: eager side channel
    qg, kg, vg = (t.cuda().requires_grad_() for t in (q, k, v))
    assert _breaks(mod, qg, kg, vg) == 0
    torch._dynamo.reset()
    out = torch.compile(mod, fullgraph=True)(qg, kg, vg)
    gout = torch.randn(out.shape, generator=torch.Generator().manual_seed(9)).to(out.dtype)
    out.backward(gout.cuda())
    lut = sel["lut"].cpu()
    w, bias = mod.proj_l.weight.detach().cpu(), mod.proj_l.bias.detach().cpu()
    blkq = blk["BLKQ"]
    want = (_oracle_grads if blkq == 128 else _oracle_grads_q64)(q, k, v, w, bias, lut, feature, gout)
    for name, gt, wt in zip(("dq", "dk", "dv", "dW", "db"), [qg.grad, kg.grad, vg.grad, mod.proj_l.weight.grad,
                                                              mod.proj_l.bias.grad], want):
        if name in ("dW", "db"):
            assert O.stats(gt.float().cpu(), wt)["rel_l2"] <= 2e-2, name
        else:
            _bars(gt, wt, what=name)
    qh, kh, vh = (t.float().transpose(1, 2) for t in (q, k, v))
    ref = (O.sparse_attention(qh, kh, vh, lut, blkq, 64) + _linear_exact(qh, kh, vh, w, bias, feature)).transpose(1, 2)
    _bars(out.detach(), ref, what="output")


def test_d64_training_is_refused_before_any_kernel_under_compile(cuda):
    from turbodiffusion_b200 import _lib
    from turbodiffusion_b200.SLA import SparseLinearAttention
    m = SparseLinearAttention(64, 0.2, BLKQ=128, BLKK=64).cuda()
    q, k, v = (t.cuda().requires_grad_() for t in _qkv(1, 512, 2, 64, 3))
    before = _lib.LAUNCHES
    torch._dynamo.reset()
    with pytest.raises(NotImplementedError):          # the compiled region falls back at the raise: the user's exception
        torch.compile(m)(q, k, v)
    torch._dynamo.reset()
    with pytest.raises(Exception) as info:            # fullgraph: Dynamo reports the refusal it traced
        torch.compile(m, fullgraph=True)(q, k, v)
    chain, e = [], info.value
    while e is not None:
        chain.append(e)
        e = e.__cause__ or e.__context__
    assert any("NotImplementedError" in repr(x) for x in chain), chain
    assert _lib.LAUNCHES == before
