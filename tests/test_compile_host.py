"""The tdb200:: custom operators without a GPU: fake (meta) kernels against the C ABI's documented shapes (include/tdb200.h),
and whole modules traced by TorchDynamo with fullgraph=True on fake CUDA tensors."""
import pytest
import torch
from torch._subclasses.fake_tensor import FakeTensorMode

import turbodiffusion_b200.ops as ops
from turbodiffusion_b200 import _ops, ltx
from turbodiffusion_b200.block import WanBlockB200
from turbodiffusion_b200.SLA.core import SageSparseLinearAttention, SparseLinearAttention

BF, F32, I8, I32 = torch.bfloat16, torch.float32, torch.int8, torch.int32


def cdiv(a, b):
    return (a + b - 1) // b


def _t(shape, dtype=BF):
    return torch.empty(shape, dtype=dtype, device="cuda")


def _cases():
    """(id, op, args builder, expected outputs [(shape, dtype)], mutated argument names)."""
    m, k, n = 300, 256, 384                      # ragged M: scales cover ceil(m/128) row blocks
    sc = lambda r, c: (cdiv(r, 128), cdiv(c, 128))  # noqa: E731
    gemm_in = lambda nn: (_t((m, k), I8), _t(sc(m, k), F32), _t((nn, k), I8), _t(sc(nn, k), F32))  # noqa: E731
    c = [
        ("quant", _ops.quant_int8_block128, lambda: (_t((m, k)),), [((m, k), I8), (sc(m, k), F32)], set()),
        ("quant_out", _ops.quant_int8_block128_out, lambda: (_t((m, k)), _t((m, k), I8), _t(sc(m, k), F32)), [],
         {"out_q", "out_s"}),
        ("gelu_quant", _ops.gelu_quant_int8_block128, lambda: (_t((m, k)),), [((m, k), I8), (sc(m, k), F32)], set()),
        ("gemm", _ops.gemm_w8a8, lambda: (*gemm_in(n), _t((n,)), 0, _t((m, n))), [], {"c"}),
        ("gemm_no_bias", _ops.gemm_w8a8, lambda: (*gemm_in(n), None, 1, _t((m, n), torch.float16)), [], {"c"}),
        ("gemm_quant_out", _ops.gemm_w8a8_quant_out, lambda: (*gemm_in(n), _t((n,)), BF, True),
         [((m, n), I8), (sc(m, n), F32)], set()),
        ("rms_norm_f32", _ops.rms_norm_f32, lambda: (_t((m, k), F32), _t((k,), F32), 1e-6, _t((m, k), F32)), [], {"out"}),
        ("layer_norm_f32", _ops.layer_norm_f32, lambda: (_t((m, k), F32), None, None, 1e-6, _t((m, k), F32)), [], {"out"}),
        ("rms_norm", _ops.rms_norm, lambda: (_t((m, k)), _t((k,), F32), 1e-6), [((m, k), BF)], set()),
        ("layer_norm", _ops.layer_norm, lambda: (_t((m, k)), _t((k,), F32), _t((k,), F32), 1e-6), [((m, k), BF)], set()),
        ("layer_norm_modulate", _ops.layer_norm_modulate, lambda: (_t((m, k)), _t((k,), F32), _t((k,), F32), 1e-6),
         [((m, k), BF)], set()),
        ("layer_norm_modulate_quant", _ops.layer_norm_modulate_quant,
         lambda: (_t((m, k)), _t((k,), F32), _t((k,), F32), 1e-6), [((m, k), I8), (sc(m, k), F32)], set()),
        ("layer_norm_modulate_quant_stats", _ops.layer_norm_modulate_quant_stats,
         lambda: (_t((m, k)), _t((2 * m,), F32), _t((k,), F32), _t((k,), F32)), [((m, k), I8), (sc(m, k), F32)], set()),
        ("gate_residual", _ops.gate_residual, lambda: (_t((m, k)), _t((m, k)), _t((k,), F32)), [((m, k), BF)], set()),
        ("gate_residual_stats", _ops.gate_residual_stats, lambda: (_t((m, k)), _t((m, k)), None, 1e-6),
         [((m, k), BF), ((2 * m,), F32)], set()),
        ("rope_interleaved", _ops.rope_interleaved, lambda: (_t((m, 2, 128)), _t((m, 64), F32)), [((m, 2, 128), BF)], set()),
        ("rms_norm_rope", _ops.rms_norm_rope, lambda: (_t((m, 256)), _t((256,), F32), _t((m, 64), F32), 1e-6, 2),
         [((m, 256), BF)], set()),
        ("rms_norm_rope_table", _ops.rms_norm_rope_table,
         lambda: (_t((m, 256)), _t((256,), F32), _t((m, 64, 2), F32), 1e-6, 2), [((m, 256), BF)], set()),
        ("ltx_modulated_rms_norm_ada", _ops.ltx_modulated_rms_norm_ada,
         lambda: (_t((2, 37, 64)), _t((6, 64), F32), _t((2, 1, 384)), 1, 0, 6, 1e-6), [((2, 37, 64), BF)], set()),
        ("ltx_modulate_ada", _ops.ltx_modulate_ada, lambda: (_t((2, 37, 64)), _t((6, 64), F32), _t((2, 37, 384)), 1, 0, 6),
         [((2, 37, 64), BF)], set()),
        ("ltx_gated_residual_ada", _ops.ltx_gated_residual_ada,
         lambda: (_t((2, 37, 64)), _t((2, 37, 64)), _t((6, 64), F32), _t((2, 1, 384)), 2, 6), [((2, 37, 64), BF)], set()),
        ("ltx_split_rope", _ops.ltx_split_rope, lambda: (_t((2, 37, 256)), _t((2, 4, 37, 32)), _t((2, 4, 37, 32))),
         [((2, 37, 256), BF)], set()),
        ("quant_int8_rowwise", _ops.quant_int8_rowwise, lambda: (_t((m, k)),), [((m, k), I8), ((m,), F32)], set()),
        ("quant_int8_rowwise_out", _ops.quant_int8_rowwise_out, lambda: (_t((m, k)), _t((m, k), I8), _t((m,), F32)), [],
         {"out_q", "out_s"}),
        ("gemm_w8a8_rowwise", _ops.gemm_w8a8_rowwise,
         lambda: (_t((m, k), I8), _t((m,), F32), _t((n, k), I8), _t((n,), F32), None, torch.float16),
         [((m, n), torch.float16)], set()),
    ]
    for parts in (2, 3):
        c.append((f"gemm_split_parts{parts}", _ops.gemm_w8a8_split, lambda p=parts: (*gemm_in(p * 256), _t((p * 256,)), BF, p),
                  [((parts, m, 256), BF)], set()))
    # SLA: ragged L, both INT8 geometries / the 16-bit query blocks, d = 64 and 128
    b, h, lq, lk = 2, 3, 1000, 1182
    for d in (64, 128):
        for blkq, blkk in ((128, 64), (64, 128), (64, 64)):
            mb, nb = cdiv(lq, blkq), cdiv(lk, blkk)
            tag = f"d{d}_q{blkq}_k{blkk}"
            if (blkq, blkk) != (64, 64):
                c.append((f"sla_quant_qk_{tag}", _ops.sla_quant_qk,
                          lambda d=d, blkq=blkq, blkk=blkk: (_t((b, lq, h, d)), _t((b, lk, h, d)), lk, blkq, blkk),
                          [((b, h, d), F32), ((b, h, lq, d), I8), ((b, h, mb), F32), ((b, h, lk, d), I8), ((b, h, nb), F32),
                           ((b, h, mb, d), BF), ((b, h, nb, d), BF)], set()))
                c.append((f"sla_attn_fwd_{tag}", _ops.sla_attn_fwd,
                          lambda d=d, blkq=blkq, blkk=blkk, mb=mb: (
                              _t((b, h, lq, d), I8), _t((b, h, mb), F32), _t((b, h, lk, d), I8), _t((b, h, cdiv(lk, blkk)), F32),
                              _t((b, lk, h, d)), _t((b, lq, h, d)), _t((b, h, mb, 3), I32), 3, _t((b, h, d, d)),
                              _t((b, h, d), F32), _t((d,), F32), d ** -0.5, lk, 0, blkq, blkk, False),
                          [((b, lq, h, d), BF)], set()))
            c.append((f"sla_quant_q_{tag}", _ops.sla_quant_q, lambda d=d, blkq=blkq: (_t((b, lq, h, d)), blkq),
                      [((b, h, lq, d), I8), ((b, h, mb), F32), ((b, h, mb, d), BF)], set()))
            c.append((f"sla_quant_k_{tag}", _ops.sla_quant_k, lambda d=d, blkk=blkk: (_t((b, lk, h, d)), lk, blkk),
                      [((b, h, d), F32), ((b, h, lk, d), I8), ((b, h, nb), F32), ((b, h, nb, d), BF)], set()))
            c.append((f"sla_block_map_{tag}", _ops.sla_block_map,
                      lambda d=d, mb=mb, nb=nb: (_t((b, h, mb, d)), _t((b, h, nb, d)), 5),
                      [((b, h, mb, nb), I8), ((b, h, mb, 5), I32)], set()))
        c.append((f"sla_linear_moments_d{d}", _ops.sla_linear_moments, lambda d=d: (_t((b, lk, h, d)), _t((b, lk, h, d)), 1),
                  [((b * h * d * (d + 1),), F32)], set()))
        c.append((f"sla_project_moments_d{d}", _ops.sla_project_moments, lambda d=d: (_t((d, d), F32), _t((b, h, d, d), F32), BF),
                  [((b, h, d, d), BF)], set()))
    d, l = 128, 1000
    for blkq in (128, 64):
        lut = lambda blkq=blkq: _t((b, h, cdiv(l, blkq), 4), I32)  # noqa: E731
        c.append((f"sla_attn16_fwd_q{blkq}", _ops.sla_attn16_fwd,
                  lambda lut=lut, blkq=blkq: (_t((b, l, h, d)), _t((b, l, h, d)), _t((b, l, h, d)), lut(), 4, _t((b, h, d, d)),
                                              _t((b, h, d), F32), _t((d,), F32), d ** -0.5, l, 0, blkq),
                  [((b, l, h, d), BF)], set()))
        c.append((f"sla_attn16_fwd_lse_q{blkq}", _ops.sla_attn16_fwd_lse,
                  lambda lut=lut, blkq=blkq: (_t((b, l, h, d)), _t((b, l, h, d)), _t((b, l, h, d)), lut(), 4, d ** -0.5, blkq),
                  [((b, l, h, d), BF), ((b, h, l), F32)], set()))
        c.append((f"sla_attn16_bwd_q{blkq}", _ops.sla_attn16_bwd,
                  lambda lut=lut, blkq=blkq: (*[_t((b, l, h, d)) for _ in range(5)], _t((b, h, l), F32), lut(), 4, d ** -0.5,
                                              blkq),
                  [((b, l, h, d), BF)] * 3, set()))
    return c


CASES = _cases()


def test_every_registered_op_has_a_fake_case():
    registered = {name for name in dir(torch.ops.tdb200) if isinstance(getattr(torch.ops.tdb200, name),
                                                                      torch._ops.OpOverloadPacket)}
    covered = {case[1]._schema.name.split("::")[1] for case in CASES}
    assert registered == covered


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_fake_kernel_matches_the_abi_shapes(case):
    _, op, args, expect, mutated = case
    with FakeTensorMode():
        out = op(*args())
    outs = [] if out is None else list(out) if isinstance(out, (tuple, list)) else [out]
    assert [(tuple(t.shape), t.dtype) for t in outs] == [(tuple(s), dt) for s, dt in expect]
    for t in outs:
        assert t.is_contiguous() and t.device.type == "cuda"
    writes = {a.name for a in op._schema.arguments if a.alias_info is not None and a.alias_info.is_write}
    assert writes == mutated


# ------------------------------------------------------------------------------------------------ tracing whole modules
def _trace(fn, *args):
    """Compile `fn` with fullgraph=True on fake CUDA inputs; return the FX graphs Dynamo produced."""
    graphs = []

    def backend(gm, example_inputs):
        graphs.append(gm)
        return gm.forward

    torch._dynamo.reset()
    out = torch.compile(fn, backend=backend, fullgraph=True, dynamic=False)(*args)
    return graphs, out


def _only_tdb200_and_aten(graphs):
    """Every call in the traced graphs is a tdb200:: op, an aten op / torch function, or Python glue (getitem, arithmetic)."""
    seen = set()
    for gm in graphs:
        for node in gm.graph.nodes:
            if node.op == "call_function":
                t = node.target
                if isinstance(t, (torch._ops.OpOverload, torch._ops.OpOverloadPacket)):
                    ns = t.namespace if isinstance(t, torch._ops.OpOverload) else t._qualified_op_name.split("::")[0]
                    assert ns in ("tdb200", "aten"), t
                    seen.add(ns)
                else:
                    mod = getattr(t, "__module__", "") or ""
                    assert mod.startswith(("torch", "_operator")) or t.__name__ in dir(__builtins__), t
            elif node.op == "call_module":
                raise AssertionError(f"unexpected submodule call {node.target}")
    assert "tdb200" in seen
    return seen


@pytest.fixture
def hopper(monkeypatch):
    """SageSLA asks the device for its compute capability while it is traced; a GPU-less host answers for an H100."""
    monkeypatch.setattr(torch.cuda, "get_device_capability", lambda device=None: (9, 0))


def _qkv(b, l, h, d, requires_grad=False):
    return [_t((b, l, h, d)).requires_grad_(requires_grad) for _ in range(3)]


SLA_CONFIGS = [(SparseLinearAttention, dict(BLKQ=128, BLKK=64), d, fm) for d in (64, 128) for fm in ("softmax", "elu", "relu")]
SLA_CONFIGS += [(SparseLinearAttention, dict(BLKQ=64, BLKK=64), 128, fm) for fm in ("softmax", "elu", "relu")]
SLA_CONFIGS += [(SageSparseLinearAttention, {}, d, "softmax") for d in (64, 128)]


@pytest.mark.parametrize("arch", ["sm100", "sm90"])
@pytest.mark.parametrize("cls,kw,d,fm", SLA_CONFIGS, ids=[f"{c.__name__}-{kw}-d{d}-{fm}" for c, kw, d, fm in SLA_CONFIGS])
def test_sla_inference_forward_traces_without_a_break(hopper, cls, kw, d, fm, arch):
    from turbodiffusion_b200.SLA.utils import set_served_arch
    if arch == "sm90" and cls is not SageSparseLinearAttention:
        pytest.skip("the served arch only selects SageSLA's block family")
    prev = set_served_arch(arch)
    try:
        with FakeTensorMode():
            with torch.device("cuda"):
                m = cls(d, 0.2, feature_map=fm, **kw)
            graphs, out = _trace(m, *_qkv(1, 1000, 3, d))
        assert tuple(out.shape) == (1, 1000, 3, d)
        assert len(graphs) == 1
        _only_tdb200_and_aten(graphs)
    finally:
        set_served_arch(prev)


@pytest.mark.parametrize("blk", [dict(BLKQ=128, BLKK=64), dict(BLKQ=64, BLKK=64)])
@pytest.mark.parametrize("fm", ["softmax", "elu", "relu"])
def test_sla_training_forward_traces_without_a_break(blk, fm):
    with FakeTensorMode():
        with torch.device("cuda"):
            m = SparseLinearAttention(128, 0.2, feature_map=fm, **blk)
        graphs, out = _trace(m, *_qkv(1, 1000, 2, 128, requires_grad=True))
    assert len(graphs) == 1 and out.requires_grad
    targets = {n.target for gm in graphs for n in gm.graph.nodes}
    assert torch.ops.tdb200.sla_attn16_fwd_lse.default in targets
    _only_tdb200_and_aten(graphs)


def test_d64_training_is_refused_at_trace_time():
    with FakeTensorMode():
        with torch.device("cuda"):
            m = SparseLinearAttention(64, 0.2, BLKQ=128, BLKK=64)
        with pytest.raises(Exception) as info:
            _trace(m, *_qkv(1, 512, 2, 64, requires_grad=True))
    chain, e = [], info.value
    while e is not None:
        chain.append(e)
        e = e.__cause__ or e.__context__
    assert any(isinstance(x, NotImplementedError) for x in chain) or "NotImplementedError" in str(info.value)


def test_sla_topk_is_a_guard():
    """The LTX client sets `.topk` before every call: a new value recompiles, the same value reuses the graph."""
    with FakeTensorMode():
        with torch.device("cuda"):
            m = SparseLinearAttention(128, 0.2, BLKQ=128, BLKK=64)
        q, k, v = _qkv(1, 1000, 2, 128)
        graphs = []

        def backend(gm, ex):
            graphs.append(gm)
            return gm.forward

        torch._dynamo.reset()
        cm = torch.compile(m, backend=backend, fullgraph=True, dynamic=False)
        cm(q, k, v)
        cm(q, k, v)
        m.topk = 0.5
        cm(q, k, v)
    luts = [[n.args[2] for n in gm.graph.nodes if n.target == torch.ops.tdb200.sla_block_map.default] for gm in graphs]
    assert luts == [[3], [8]]    # nblk = 16 key blocks: int(0.2 * 16), int(0.5 * 16)


def _linear_modules():
    yield "Int8Linear", ops.Int8Linear(256, 384), _t((2, 150, 256))
    yield "Int8Linear_nobias", ops.Int8Linear(256, 384, bias=False), _t((300, 256))
    yield "FastRMSNorm", ops.FastRMSNorm(256), _t((2, 150, 256))
    yield "FastRMSNorm_fp32", ops.FastRMSNorm(256), _t((2, 150, 256), F32)
    yield "FastLayerNorm", ops.FastLayerNorm(256, elementwise_affine=True), _t((2, 150, 256))
    yield "FastLayerNorm_noaffine", ops.FastLayerNorm(256), _t((300, 256))
    yield "FastLayerNorm_fp32", ops.FastLayerNorm(256, elementwise_affine=True), _t((300, 256), F32)
    yield "PostScaleInt8Linear", ltx.PostScaleInt8Linear(256, 384), _t((2, 150, 256))


@pytest.mark.parametrize("name", ["Int8Linear", "Int8Linear_nobias", "FastRMSNorm", "FastRMSNorm_fp32", "FastLayerNorm",
                                  "FastLayerNorm_noaffine", "FastLayerNorm_fp32", "PostScaleInt8Linear"])
def test_linear_and_norm_modules_trace_without_a_break(name):
    with FakeTensorMode():
        with torch.device("cuda"):
            m, x = next((m, x) for n, m, x in _linear_modules() if n == name)
        graphs, out = _trace(m, x)
    assert len(graphs) == 1 and out.shape[:-1] == x.shape[:-1]
    _only_tdb200_and_aten(graphs)


def test_ltx_prologue_operators_trace_without_a_break():
    def f(x, res, table, ts, cos, sin):
        y = ltx.modulated_rms_norm_from_ada(x, table, ts, 1, 0, 6, 1e-6)
        y = ltx.modulate_from_ada(y, table, ts, 4, 3, 6)
        y = ltx.gated_residual_from_ada(y, res, table, ts, 2, 6)
        return ltx.apply_split_rotary_emb(y, cos, sin)

    with FakeTensorMode():
        graphs, out = _trace(f, _t((2, 37, 256)), _t((2, 37, 256)), _t((6, 256), F32), _t((2, 1, 1536)), _t((2, 4, 37, 32), F32),
                             _t((2, 4, 37, 32), F32))
    assert len(graphs) == 1 and tuple(out.shape) == (2, 37, 256)
    _only_tdb200_and_aten(graphs)


def _fake_block_state(dim, ffn, heads):
    """The layout of block.random_block_state, as empty fake tensors."""
    sd = {}
    for name, (n, k) in {"self_attn.q": (dim, dim), "self_attn.k": (dim, dim), "self_attn.v": (dim, dim),
                         "self_attn.o": (dim, dim), "cross_attn.q": (dim, dim), "cross_attn.k": (dim, dim),
                         "cross_attn.v": (dim, dim), "cross_attn.o": (dim, dim), "ffn.0": (ffn, dim),
                         "ffn.2": (dim, ffn)}.items():
        sd[name + ".int8_weight"], sd[name + ".scale"], sd[name + ".bias"] = _t((n, k), I8), _t((cdiv(n, 128), cdiv(k, 128)), F32), _t((n,))
    for name in ("self_attn.norm_q", "self_attn.norm_k", "cross_attn.norm_q", "cross_attn.norm_k", "norm3"):
        sd[name + ".weight"] = _t((dim,), F32)
    sd["norm3.bias"] = _t((dim,), F32)
    sd["modulation"] = _t((1, 6, dim), F32)
    d = dim // heads
    sd["self_attn.attn_op.local_attn.proj_l.weight"] = _t((d, d), F32)
    sd["self_attn.attn_op.local_attn.proj_l.bias"] = _t((d,), F32)
    return sd


@pytest.mark.parametrize("attention", ["sagesla", "sla"])
@pytest.mark.parametrize("ffn_mode", ["fused", "split"])
def test_wan_block_forward_traces_without_a_break(hopper, monkeypatch, ffn_mode, attention):
    from turbodiffusion_b200 import block as B
    monkeypatch.setattr(B, "FFN_ACT_MODE", ffn_mode)
    dim, heads, l, lc = 256, 2, 600, 77
    with FakeTensorMode():
        with torch.device("cuda"):
            blk = WanBlockB200(_fake_block_state(dim, 512, heads), dim, heads, topk=0.3, attention=attention)
        args = (_t((l, dim)), _t((6, dim), F32), _t((l, 64), F32), _t((lc, dim)))
        graphs, out = _trace(lambda *a: blk.forward(*a), *args)
        assert len(graphs) == 1 and tuple(out.shape) == (l, dim)
        # with the row statistics carried in and out, as WanHotPath chains blocks
        graphs2, (out2, stats) = _trace(lambda x, e0, ang, ctx, st: blk.forward(x, e0, ang, ctx, st, want_stats=True),
                                        *args, _t((2 * l,), F32))
        assert len(graphs2) == 1 and tuple(stats.shape) == (2 * l,)
    _only_tdb200_and_aten(graphs + graphs2)
    names = {n.target for gm in graphs for n in gm.graph.nodes}
    assert (torch.ops.tdb200.gemm_w8a8_quant_out.default in names) == (ffn_mode == "fused")
