"""Host-side behaviour of the operator mirrors that does not need a GPU: there is no CPU / eager fallback (CPU tensors
and a missing library raise), constructors / buffers / signatures follow the reference's operator API
(turbodiffusion/ops/core.py, SLA/core.py, ops/bindings.cpp), and the host helpers (RoPE angle table, row sharding,
launch accounting) compute what the reference's callers expect."""
import inspect
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import td_oracle as O  # noqa: E402
from turbodiffusion_b200 import _lib, ops, turbo_diffusion_ops as tdo  # noqa: E402
from turbodiffusion_b200.SLA import SageSparseLinearAttention, SparseLinearAttention  # noqa: E402


def test_cpu_tensors_are_refused_not_computed():
    x = torch.randn(128, 128).bfloat16()
    w = torch.ones(128)
    calls = [
        lambda: tdo.quant_cuda(x),
        lambda: ops.int8_quant(x),
        lambda: ops.rmsnorm(x.float(), w, 1e-6),
        lambda: ops.layernorm(x.float(), None, None, 1e-6, False),
        lambda: ops.fast_rmsnorm(x, w, 1e-6),
        lambda: ops.gate_residual(x, x, w),
    ]
    for f in calls:
        with pytest.raises(_lib.Tdb200Error, match="no CPU fallback"):
            f()
    q = torch.randn(1, 128, 1, 128).bfloat16()
    with pytest.raises(_lib.Tdb200Error, match="no CPU fallback"):
        SageSparseLinearAttention(128, 0.1)(q, q, q)
    with pytest.raises(_lib.Tdb200Error, match="no CPU fallback"):
        SparseLinearAttention(128, 0.1, BLKQ=128, BLKK=64)(q, q, q)


def test_missing_library_fails_loudly():
    """Importing the binding with the shared library absent must raise with build instructions (no silent fallback)."""
    code = ("import sys; sys.path.insert(0, %r)\n"
            "from turbodiffusion_b200 import _lib\n"
            "_lib.LIB_PATH = '/nonexistent/libtdb200.so'\n"
            "try:\n    _lib.lib()\nexcept _lib.Tdb200Error as e:\n    print('RAISED', 'no fallback' in str(e) and '_build' in str(e))\n") % ROOT
    p = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert p.returncode == 0 and "RAISED True" in p.stdout, p.stdout + p.stderr


def test_pybind_mirror_signatures_follow_bindings_cpp():
    """ops/bindings.cpp:11-16 + quant.cu:70 / gemm.cu:67 / rmsnorm.cu:57-59 / layernorm.cu:60-62 argument order."""
    assert list(inspect.signature(tdo.quant_cuda).parameters) == ["x", "out_q", "out_s"]
    assert list(inspect.signature(tdo.gemm_cuda).parameters) == ["a_q", "a_s", "b_q", "b_s", "c"]
    assert list(inspect.signature(tdo.rms_norm_cuda).parameters)[:3] == ["x", "eps", "w"]
    assert list(inspect.signature(tdo.layer_norm_cuda).parameters)[:4] == ["x", "eps", "w", "b"]
    # the two entry points TurboT2AV looks up with getattr (acceleration.py:695-701)
    assert list(inspect.signature(tdo.gemm_cuda_swizzle).parameters)[:5] == ["a_q", "a_s", "b_q", "b_s", "c"]
    assert list(inspect.signature(tdo.gemm_cuda_swizzle_bias).parameters)[:6] == ["a_q", "a_s", "b_q", "b_s", "c", "bias"]


def test_int8_linear_module_buffers_and_keys():
    """ops/core.py:391-412: buffers int8_weight [out,in] int8, scale [ceil(out/128), ceil(in/128)] fp32, bias [out]."""
    m = ops.Int8Linear(1536, 8960)
    sd = m.state_dict()
    assert list(sd) == ["int8_weight", "scale", "bias"]
    assert sd["int8_weight"].shape == (8960, 1536) and sd["int8_weight"].dtype == torch.int8
    assert sd["scale"].shape == (70, 12) and sd["scale"].dtype == torch.float32
    assert sd["bias"].shape == (8960,) and sd["bias"].dtype == torch.bfloat16
    assert "bias" not in ops.Int8Linear(256, 300, bias=False).state_dict() or ops.Int8Linear(256, 300, bias=False).bias is None
    lin = torch.nn.Linear(256, 384)
    q = ops.Int8Linear.from_linear(lin, quantize=False)          # structure only (like the reference, nothing is copied);
    assert q.int8_weight.shape == (384, 256) and q.scale.shape == (3, 2)      # quantize=True runs quant_cuda on the GPU
    assert q.bias.shape == (384,) and q.bias.dtype == lin.weight.dtype


def test_fast_norm_modules_take_over_parameters():
    class WanRMSNormLike(torch.nn.Module):                        # rcm/networks/wan2pt1.py WanRMSNorm: .dim, .eps, .weight
        def __init__(self, dim, eps):
            super().__init__()
            self.dim, self.eps = dim, eps
            self.weight = torch.nn.Parameter(torch.rand(dim) + 0.5)

    rms = WanRMSNormLike(96, 1e-6)
    f = ops.FastRMSNorm.from_rmsnorm(rms)
    assert f.eps == 1e-6 and torch.equal(f.weight, rms.weight)
    ln = torch.nn.LayerNorm(96, eps=1e-6, elementwise_affine=True)
    g = ops.FastLayerNorm.from_layernorm(ln)
    assert g.eps == 1e-6 and torch.equal(g.weight, ln.weight) and torch.equal(g.bias, ln.bias)
    h = ops.FastLayerNorm.from_layernorm(torch.nn.LayerNorm(96, eps=1e-6, elementwise_affine=False))
    assert h.weight is None and h.bias is None


def test_sla_modules_constructor_and_zero_init():
    """SLA/core.py:38-66,122-166: proj_l = Linear(head_dim, head_dim) fp32, zero-initialised; topk mutable; dtype flag."""
    for cls, kw in ((SageSparseLinearAttention, {}), (SparseLinearAttention, {"BLKQ": 128, "BLKK": 64})):
        m = cls(128, 0.1, **kw)
        assert sorted(m.state_dict()) == ["proj_l.bias", "proj_l.weight"]
        assert m.proj_l.weight.dtype == torch.float32 and not m.proj_l.weight.any() and not m.proj_l.bias.any()
        assert m.topk == 0.1 and m.dtype == torch.bfloat16
        m.topk = 0.3                                                  # acceleration.py:400-409 mutates it per call
        assert cls(64, 0.2, use_bf16=False, **kw).dtype == torch.float16
    with pytest.raises(Exception):
        SageSparseLinearAttention(128, 0.1, feature_map="nope")


def test_wan_rope_angle_table_matches_oracle():
    """rcm/networks/wan2pt1.py:86-137: per-axis frequency split 44/42/42 of D=128 (22+21+21 angles), t/h/w raster."""
    a = ops.wan_rope_angles(3, 4, 5, 128, torch.device("cpu"))
    b = O.wan_rope_angles(3, 4, 5, 128)
    assert a.shape == (60, 64) and a.dtype == torch.float32
    assert torch.equal(a, b)
    assert (a[0] == 0).all() and (a[1, :22] == 0).all() and (a[1, 43:] != 0).any()   # w is the fastest axis


def test_launch_accounting_counts_every_abi_call():
    before = _lib.LAUNCHES
    _lib.check(0, "gemm_w8a8")
    _lib.check(0, "sla_quant_qk")
    _lib.check(0, "anything", launches=3)
    assert _lib.LAUNCHES - before == 1 + 4 + 3
    with pytest.raises(_lib.Tdb200Error, match=r"boom failed \(code -1\)"):
        _lib.check(-1, "boom")

