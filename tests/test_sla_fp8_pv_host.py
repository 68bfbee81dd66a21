"""CPU checks of SageSLA's FP8 P.V option: the C entry points' validation (tdb200_sla_quant_v_fp8, tdb200_sla_attn_fwd_fp8v), the
selection switch (SLA.utils.set_sage_pv, TDB200_SAGE_PV, install) and where it routes SageSparseLinearAttention, the LTX
adapters and sequence parallelism, the tdb200_fp8:: fake kernels, and fullgraph tracing of both Sage block families."""
import ctypes
import os
import subprocess
import sys

import pytest
import torch

INVALID, UNSUPPORTED = -1, -2
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _p(v=4096):
    return ctypes.c_void_p(v)


@pytest.fixture(scope="module")
def lib():
    from turbodiffusion_b200 import _build, _lib
    _build.build()
    return _lib.lib()


def _quant(lib, v=_p(), dtype=0, b=1, l=300, h=2, d=128, blkk=128, v_fp8=_p(), v_scale=_p()):
    return lib.tdb200_sla_quant_v_fp8(v, dtype, b, l, h, d, blkk, v_fp8, v_scale, None)


def _attn(lib, q_i8=_p(), v_fp8=_p(), v_scale=_p(), dtype=0, topk=2, b=1, l=256, lk=256, h=2, d=128, feature=0, blkq=128,
          blkk=64, seq=0):
    return lib.tdb200_sla_attn_fwd_fp8v(q_i8, _p(), _p(), _p(), v_fp8, v_scale, _p(), dtype, _p(), topk, _p(), _p(), _p(), _p(), b, l,
                                        lk, h, d, 0.088, feature, blkq, blkk, seq, None)


def test_argument_validation(lib):
    cases = [
        ("quant block", lambda: _quant(lib, blkk=96), UNSUPPORTED, b"key block size"),
        ("quant null v", lambda: _quant(lib, v=None), INVALID, b"null"),
        ("quant null scale", lambda: _quant(lib, v_scale=None), INVALID, b"null"),
        ("quant shape", lambda: _quant(lib, l=0), INVALID, b"bad shape"),
        ("quant head dim", lambda: _quant(lib, d=64), UNSUPPORTED, b"head dim"),
        ("quant dtype", lambda: _quant(lib, dtype=3), UNSUPPORTED, b"dtype"),
        ("quant grid", lambda: _quant(lib, h=70000), UNSUPPORTED, b"too large"),
        ("quant size", lambda: _quant(lib, l=1 << 33, h=64), UNSUPPORTED, b"too large"),
        ("quant misaligned", lambda: _quant(lib, v_fp8=_p(4097)), INVALID, b"aligned"),
        ("attn blocks", lambda: _attn(lib, blkq=64, blkk=64), UNSUPPORTED, b"block sizes"),
        ("attn blocks 128x128", lambda: _attn(lib, blkq=128, blkk=128), UNSUPPORTED, b"block sizes"),
        ("attn null", lambda: _attn(lib, q_i8=None), INVALID, b"null"),
        ("attn null v", lambda: _attn(lib, v_fp8=None), INVALID, b"null"),
        ("attn null scale", lambda: _attn(lib, v_scale=None), INVALID, b"null"),
        ("attn shape", lambda: _attn(lib, lk=0), INVALID, b"bad shape"),
        ("attn misaligned", lambda: _attn(lib, v_scale=_p(4100)), INVALID, b"aligned"),
        ("attn head dim", lambda: _attn(lib, d=64), UNSUPPORTED, b"head dim"),
        ("attn hopper head dim", lambda: _attn(lib, d=64, blkq=64, blkk=128), UNSUPPORTED, b"head dim"),
        ("attn feature", lambda: _attn(lib, feature=3), INVALID, b"feature"),
        ("attn seq-major feature", lambda: _attn(lib, feature=1, seq=1), UNSUPPORTED, b"sequence-major"),
        ("attn seq-major batch", lambda: _attn(lib, b=2, seq=1), UNSUPPORTED, b"batch"),
        ("attn topk", lambda: _attn(lib, topk=9), INVALID, b"topk"),
        ("attn dtype", lambda: _attn(lib, dtype=7), UNSUPPORTED, b"dtype"),
        ("attn grid", lambda: _attn(lib, h=70000), UNSUPPORTED, b"too large"),
    ]
    for name, call, code, needle in cases:
        rc = call()
        msg = lib.tdb200_last_error() or b""
        assert rc == code, (name, rc, msg)
        assert needle in msg, (name, msg)


def test_valid_calls_without_a_gpu_report_an_error_code(lib):
    if torch.cuda.is_available():
        pytest.skip("this check is for hosts without a GPU")
    assert _quant(lib) in (-3, -4) and lib.tdb200_last_error()
    assert _attn(lib, blkq=64, blkk=128) in (-3, -4) and lib.tdb200_last_error()


def test_set_sage_pv_and_install():
    import turbodiffusion_b200
    from turbodiffusion_b200.SLA import utils
    assert utils.SAGE_PV == "bf16"
    with pytest.raises(ValueError):
        utils.set_sage_pv("fp16")
    assert utils.set_sage_pv("fp8") == "bf16"
    try:
        assert utils.SAGE_PV == "fp8"
        turbodiffusion_b200.install()            # leaves the setting as it is
        assert utils.SAGE_PV == "fp8"
        turbodiffusion_b200.install(sage_pv="bf16")
        assert utils.SAGE_PV == "bf16"
        with pytest.raises(ValueError):
            turbodiffusion_b200.install(sage_pv="e4m3")
        turbodiffusion_b200.install(sage_pv="fp8")
        assert utils.SAGE_PV == "fp8"
    finally:
        utils.set_sage_pv("bf16")
        turbodiffusion_b200.install()


@pytest.mark.parametrize("env,want", [(None, "bf16"), ("", "bf16"), ("bf16", "bf16"), ("fp8", "fp8"), ("int4", "ValueError")])
def test_environment_default(env, want):
    e = {k: v for k, v in os.environ.items() if k != "TDB200_SAGE_PV"}
    if env is not None:
        e["TDB200_SAGE_PV"] = env
    r = subprocess.run([sys.executable, "-c", "from turbodiffusion_b200.SLA import utils; print(utils.SAGE_PV)"],
                       capture_output=True, text=True, env=e, cwd=ROOT)
    if want == "ValueError":
        assert r.returncode != 0 and "ValueError" in r.stderr and "TDB200_SAGE_PV" in r.stderr
    else:
        assert r.returncode == 0 and r.stdout.strip() == want, r.stderr


class _Recorder:
    """Stands in for the library: records the tdb200 / tdb200_fp8 operators SageSparseLinearAttention calls (module level
    `_ops` of SLA.core and SLA.utils), returning tensors of the right shapes."""

    def __init__(self, monkeypatch):
        from turbodiffusion_b200 import _ops
        from turbodiffusion_b200.SLA import core, utils
        self.calls = []
        monkeypatch.setattr(core, "require_cuda", lambda *a: None)
        monkeypatch.setattr(utils, "require_cuda", lambda *a: None)
        monkeypatch.setattr(core, "get_cuda_arch", lambda index: utils.SERVED_ARCH)   # no device to query

        def rec(name, fake):
            def f(*a):
                self.calls.append(name)
                return fake(*a)
            return f

        ns = type("Ops", (), {})()
        ns.sla_quant_qk = rec("sla_quant_qk", _ops._quant_qk_fake)
        ns.sla_block_map = rec("sla_block_map", _ops._block_map_fake)
        ns.sla_linear_moments = rec("sla_linear_moments", _ops._moments_fake)
        ns.sla_project_moments = rec("sla_project_moments", _ops._project_fake)
        ns.sla_attn_fwd = rec("sla_attn_fwd", lambda q_i8, q_scale, k_i8, k_scale, v, q, *r: torch.zeros_like(q))
        ns.sla_quant_v_fp8 = rec("sla_quant_v_fp8", _ops._quant_v_fp8_fake)
        ns.sla_attn_fwd_fp8v = rec("sla_attn_fwd_fp8v", lambda q_i8, q_scale, k_i8, k_scale, v_fp8, v_scale, q, *r:
                                   torch.zeros_like(q))
        monkeypatch.setattr(core, "_ops", ns)
        monkeypatch.setattr(utils, "_ops", ns)


@pytest.mark.parametrize("arch", ["sm100", "sm90"])
@pytest.mark.parametrize("feature_map", ["softmax", "elu", "relu"])
def test_the_module_calls_the_fp8_entry_points_only_under_fp8(monkeypatch, arch, feature_map):
    from turbodiffusion_b200.SLA import SageSparseLinearAttention, utils
    rec = _Recorder(monkeypatch)
    monkeypatch.setattr(utils, "SERVED_ARCH", arch)
    m = SageSparseLinearAttention(128, 0.3, feature_map=feature_map)
    x = torch.zeros(1, 600, 2, 128, dtype=torch.bfloat16)
    m(x, x, x)
    assert "sla_attn_fwd" in rec.calls and "sla_quant_v_fp8" not in rec.calls and "sla_attn_fwd_fp8v" not in rec.calls
    rec.calls.clear()
    monkeypatch.setattr(utils, "SAGE_PV", "fp8")
    m(x, x, x)
    assert rec.calls[-2:] == ["sla_quant_v_fp8", "sla_attn_fwd_fp8v"] and "sla_attn_fwd" not in rec.calls


def test_head_dim_64_is_refused_before_any_library_call(monkeypatch):
    from turbodiffusion_b200.SLA import SageSparseLinearAttention, utils
    rec = _Recorder(monkeypatch)
    monkeypatch.setattr(utils, "SAGE_PV", "fp8")
    x = torch.zeros(1, 600, 2, 64, dtype=torch.bfloat16)
    with pytest.raises(NotImplementedError, match="head dim 64"):
        SageSparseLinearAttention(64, 0.3)(x, x, x)
    assert rec.calls == []


def test_sparse_linear_attention_is_not_affected(monkeypatch):
    """SparseLinearAttention's INT8-QK calls (elu / relu at (128, 64), 64-wide heads) keep the 16-bit P.V under "fp8"."""
    from turbodiffusion_b200.SLA import SparseLinearAttention, utils
    rec = _Recorder(monkeypatch)
    monkeypatch.setattr(utils, "SAGE_PV", "fp8")
    x = torch.zeros(1, 600, 2, 64, dtype=torch.bfloat16)
    SparseLinearAttention(64, 0.3, BLKQ=128, BLKK=64)(x, x, x)
    assert "sla_attn_fwd" in rec.calls and "sla_attn_fwd_fp8v" not in rec.calls


@pytest.mark.parametrize("d", [128, 64])
def test_ltx_adapters_follow_the_setting(monkeypatch, d):
    from turbodiffusion_b200.SLA import core, utils
    rec = _Recorder(monkeypatch)
    monkeypatch.setattr(core.torch, "zeros", lambda *a, **kw: torch.empty(*a, dtype=kw.get("dtype")))
    monkeypatch.setattr(core.torch, "ones", lambda *a, **kw: torch.empty(*a, dtype=kw.get("dtype")))
    b, h, l = 1, 2, 300
    q8 = torch.zeros(b, h, l, d, dtype=torch.int8)
    v = torch.zeros(b, h, l, d, dtype=torch.bfloat16)
    v_fp8 = torch.empty(b, h, d, 320)
    core.fused.scale_fuse_quant_cuda(v, v_fp8, None, l)
    lut = torch.zeros(b, h, 3, 1, dtype=torch.int32)
    args = (q8, q8, v_fp8, torch.empty(b, h, l, d, dtype=torch.bfloat16), lut, None, None, torch.ones(b, h, 3),
            torch.ones(b, h, 5), None)
    monkeypatch.setattr(utils, "SAGE_PV", "fp8")
    if d == 64:
        with pytest.raises(NotImplementedError, match="head dim 64"):
            core.qk_int8_sv_f8_accum_f16_block_sparse_attn_inst_buf_fuse_v_scale_with_pv_threshold(*args)
        assert rec.calls == []
        return
    core.qk_int8_sv_f8_accum_f16_block_sparse_attn_inst_buf_fuse_v_scale_with_pv_threshold(*args)
    core.qattn.qk_int8_sv_f8_accum_f32_block_sparse_attn_inst_buf_fuse_v_scale_with_pv_threshold_sm90(*args)
    assert rec.calls == ["sla_quant_v_fp8", "sla_attn_fwd_fp8v"] * 2
    rec.calls.clear()
    monkeypatch.setattr(utils, "SAGE_PV", "bf16")
    core.qk_int8_sv_f8_accum_f16_block_sparse_attn_inst_buf_fuse_v_scale_with_pv_threshold(*args)
    assert rec.calls == ["sla_attn_fwd"]


def test_sequence_parallel_refuses_fp8_before_any_library_call(monkeypatch):
    from turbodiffusion_b200 import dist
    from turbodiffusion_b200.SLA import utils
    rec = _Recorder(monkeypatch)
    sp = dist.SequenceParallel.__new__(dist.SequenceParallel)
    monkeypatch.setattr(utils, "SAGE_PV", "fp8")
    with pytest.raises(NotImplementedError, match="FP8"):
        sp.install(object(), "allgather")
    with pytest.raises(NotImplementedError, match="FP8"):
        dist.require_served_arch("sm100")
    monkeypatch.setattr(utils, "SAGE_PV", "bf16")
    dist.require_served_arch("sm100")
    assert rec.calls == []


def test_fake_kernels_match_the_abi_shapes():
    from torch._subclasses.fake_tensor import FakeTensorMode
    from turbodiffusion_b200 import _ops
    b, l, h, d = 2, 333, 3, 128
    with FakeTensorMode(allow_non_fake_inputs=False):
        v = torch.empty(b, l, h, d, dtype=torch.float16, device="cuda")
        for blkk in (64, 128):
            v_fp8, v_scale = _ops.sla_quant_v_fp8(v, l, blkk)
            assert (v_fp8.shape, v_fp8.dtype) == ((b, h, d, (l + blkk - 1) // blkk * blkk), torch.uint8)
            assert (v_scale.shape, v_scale.dtype) == ((b, h, d), torch.float32)
        q8 = torch.empty(b, h, l, d, dtype=torch.int8, device="cuda")
        f = torch.empty(4, device="cuda")
        out = _ops.sla_attn_fwd_fp8v(q8, f, q8, f, v_fp8, v_scale, v, torch.empty(1, dtype=torch.int32, device="cuda"), 2, v, f, f,
                                     0.088, l, 0, 64, 128, False)
        assert (out.shape, out.dtype) == ((b, l, h, d), torch.float16)
    ops = {n for n in dir(torch.ops.tdb200_fp8) if isinstance(getattr(torch.ops.tdb200_fp8, n), torch._ops.OpOverloadPacket)}
    assert ops == {"sla_quant_v_fp8", "sla_attn_fwd_fp8v"}


@pytest.mark.parametrize("arch", ["sm100", "sm90"])
def test_sage_modules_trace_as_one_graph_under_fp8(monkeypatch, arch):
    from torch._subclasses.fake_tensor import FakeTensorMode
    from turbodiffusion_b200.SLA import SageSparseLinearAttention, utils
    graphs = []

    def backend(gm, example_inputs):
        graphs.append(gm)
        return gm.forward

    monkeypatch.setattr(torch.cuda, "get_device_capability", lambda device=None: (9, 0))   # a GPU-less host answers for an H100
    prev_pv, prev_arch = utils.set_sage_pv("fp8"), utils.set_served_arch(arch)
    try:
        torch._dynamo.reset()
        with FakeTensorMode():
            with torch.device("cuda"):
                m = SageSparseLinearAttention(128, 0.2)
            q, k, v = (torch.empty(1, 1000, 2, 128, dtype=torch.bfloat16, device="cuda") for _ in range(3))
            with torch.no_grad():
                torch.compile(m, backend=backend, fullgraph=True, dynamic=False)(q, k, v)
    finally:
        utils.set_sage_pv(prev_pv)
        utils.set_served_arch(prev_arch)
        torch._dynamo.reset()
    assert len(graphs) == 1
    targets = {n.target for gm in graphs for n in gm.graph.nodes}
    assert torch.ops.tdb200_fp8.sla_quant_v_fp8.default in targets and torch.ops.tdb200_fp8.sla_attn_fwd_fp8v.default in targets
    assert torch.ops.tdb200.sla_attn_fwd.default not in targets
