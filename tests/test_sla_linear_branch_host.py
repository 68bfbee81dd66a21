"""CPU checks of the linear-branch kernels' C entry points (argument validation, workspace size), of the selection switch
(SLA.utils.set_linear_branch, install) and of which branch SparseLinearAttention's training forward takes."""
import ctypes

import pytest
import torch

INVALID, UNSUPPORTED, WORKSPACE = -1, -2, -5


def _p(v=4096):
    return ctypes.c_void_p(v)


@pytest.fixture(scope="module")
def lib():
    from turbodiffusion_b200 import _build, _lib
    _build.build()
    return _lib.lib()


def _fwd(lib, q=_p(), d=128, dtype=0, feature=0, b=1, l=256, h=2):
    return lib.tdb200_sla_linear_fwd(q, _p(), _p(), _p(), _p(), dtype, feature, _p(), b, l, h, d, None)


def _bwd(lib, ws=_p(), ws_bytes=1 << 40, d=128, dtype=0, feature=0, dw=_p(), l=256):
    return lib.tdb200_sla_linear_bwd(_p(), _p(), _p(), _p(), _p(), _p(), _p(), dtype, feature, _p(), _p(), _p(), dw, _p(), ws,
                                     ws_bytes, 1, l, 2, d, None)


def _tan(lib, q=_p(), ws_bytes=1 << 40, d=128, dtype=0, feature=0):
    return lib.tdb200_sla_linear_tangent(q, _p(), _p(), _p(), _p(), _p(), _p(), _p(), _p(), dtype, feature, _p(), _p(), ws_bytes,
                                         1, 256, 2, d, None)


def test_argument_validation(lib):
    cases = [
        ("fwd null", lambda: _fwd(lib, q=None), INVALID, b"null"),
        ("fwd misaligned", lambda: _fwd(lib, q=_p(4098)), INVALID, b"aligned"),
        ("fwd head dim", lambda: _fwd(lib, d=64), UNSUPPORTED, b"head dim"),
        ("fwd dtype", lambda: _fwd(lib, dtype=5), UNSUPPORTED, b"dtype"),
        ("fwd feature", lambda: _fwd(lib, feature=3), UNSUPPORTED, b"feature"),
        ("fwd shape", lambda: _fwd(lib, l=0), INVALID, b"shape"),
        ("fwd grid", lambda: _fwd(lib, b=300, h=300), UNSUPPORTED, b"65535"),
        ("fwd size", lambda: _fwd(lib, l=1 << 33, h=64), UNSUPPORTED, b"2^39"),
        ("bwd null", lambda: _bwd(lib, dw=None), INVALID, b"null"),
        ("bwd null workspace", lambda: _bwd(lib, ws=None), INVALID, b"null"),
        ("bwd head dim", lambda: _bwd(lib, d=64), UNSUPPORTED, b"head dim"),
        ("bwd dtype", lambda: _bwd(lib, dtype=2), UNSUPPORTED, b"dtype"),
        ("bwd feature", lambda: _bwd(lib, feature=-1), UNSUPPORTED, b"feature"),
        ("bwd workspace", lambda: _bwd(lib, ws_bytes=lib.tdb200_sla_linear_bwd_workspace_bytes(1, 2, 256, 128) - 1), WORKSPACE,
         b"workspace"),
        ("tangent null", lambda: _tan(lib, q=None), INVALID, b"null"),
        ("tangent misaligned", lambda: _tan(lib, q=_p(4100)), INVALID, b"aligned"),
        ("tangent head dim", lambda: _tan(lib, d=64), UNSUPPORTED, b"head dim"),
        ("tangent dtype", lambda: _tan(lib, dtype=9), UNSUPPORTED, b"dtype"),
        ("tangent feature", lambda: _tan(lib, feature=4), UNSUPPORTED, b"feature"),
        ("tangent workspace", lambda: _tan(lib, ws_bytes=lib.tdb200_sla_linear_tangent_workspace_bytes(1, 2, 256, 128) - 1),
         WORKSPACE, b"workspace"),
    ]
    for name, call, code, needle in cases:
        rc = call()
        msg = lib.tdb200_last_error() or b""
        assert rc == code, (name, rc, msg)
        assert needle in msg, (name, msg)


def test_exact_workspace_passes_validation(lib):
    if torch.cuda.is_available():
        pytest.skip("this check is for hosts without a GPU")
    rc = _bwd(lib, ws_bytes=lib.tdb200_sla_linear_bwd_workspace_bytes(1, 2, 256, 128))
    assert rc in (-3, -4) and lib.tdb200_last_error()


@pytest.mark.parametrize("b,h,l", [(1, 2, 256), (2, 3, 333), (1, 12, 32760), (1, 40, 75600)])
def test_workspace_size_formula(lib, b, h, l):
    def a(x):
        return (x + 255) // 256 * 256
    tiles = (l + 63) // 64
    splits = min(tiles, 16)
    want = 3 * a(2 * b * l * h * 128) + 2 * a(4 * b * h * tiles * 128) + a(4 * b * h * splits * 128 * 128) \
        + a(4 * b * h * 128 * 128) + a(4 * b * h * 128)
    assert lib.tdb200_sla_linear_bwd_workspace_bytes(b, h, l, 128) == want
    assert lib.tdb200_sla_linear_tangent_workspace_bytes(b, h, l, 128) == \
        2 * a(2 * b * l * h * 128) + a(4 * b * h * tiles * 128) + a(4 * b * h * splits * 128 * 128) + a(4 * b * h * 128 * 128) \
        + a(4 * b * h * 128)
    assert lib.tdb200_sla_linear_bwd_workspace_bytes(0, h, l, 128) == INVALID
    assert lib.tdb200_sla_linear_bwd_workspace_bytes(b, h, l, 64) == UNSUPPORTED


def test_set_linear_branch_and_install():
    import turbodiffusion_b200
    from turbodiffusion_b200.SLA import utils
    assert utils.LINEAR_BRANCH == "reference"
    with pytest.raises(ValueError):
        utils.set_linear_branch("torch")
    assert utils.set_linear_branch("fused") == "reference"
    try:
        assert utils.LINEAR_BRANCH == "fused"
        with pytest.raises(ValueError):
            turbodiffusion_b200.install(sla_linear_branch="cuda")
        turbodiffusion_b200.install(sla_linear_branch="reference")
        assert utils.LINEAR_BRANCH == "reference"
        turbodiffusion_b200.install(sla_linear_branch="fused")
        assert utils.LINEAR_BRANCH == "fused"
    finally:
        utils.set_linear_branch("reference")
        turbodiffusion_b200.install()


def test_linear_branch_refusals():
    from turbodiffusion_b200.SLA.core import linear_branch
    w, b = torch.zeros(128, 128), torch.zeros(128)
    x64 = torch.zeros(1, 8, 1, 64, dtype=torch.bfloat16)
    with pytest.raises(NotImplementedError):
        linear_branch(x64, x64, x64, w, b)
    x = torch.zeros(1, 8, 1, 128, dtype=torch.bfloat16)
    with pytest.raises(ValueError):
        linear_branch(x, x.half(), x, w, b)
    with pytest.raises(RuntimeError):   # CPU tensors: no fallback
        linear_branch(x, x, x, w, b)


class _Recorder:
    """Stands in for the parts of the training forward that need a GPU, recording which linear branch runs."""

    def __init__(self, monkeypatch):
        from turbodiffusion_b200.SLA import core
        self.calls = []
        monkeypatch.setattr(core, "require_cuda", lambda *a: None)
        monkeypatch.setattr(core, "select_prep", lambda q, k, bq, bk: type("P", (), {"q_pool": None, "k_pool": None,
                                                                                      "nblk": 16})())
        monkeypatch.setattr(core, "block_map_from_pools", lambda *a: (None, None))
        monkeypatch.setattr(core, "sparse_attention16", lambda q, *a: torch.zeros_like(q))
        monkeypatch.setattr(core, "linear_branch", self._fused)
        monkeypatch.setattr(core._SLABase, "_linear_branch", self._torch)

    def _fused(self, q, k, v, w, b, feature):
        self.calls.append(("fused", feature))
        return torch.zeros_like(q)

    def _torch(self_, *a):   # noqa: N805  (bound as the module's method)
        raise AssertionError("replaced per instance")


def test_training_forward_takes_the_selected_branch(monkeypatch):
    from turbodiffusion_b200.SLA import core, utils
    rec = _Recorder(monkeypatch)
    seen = []
    monkeypatch.setattr(core._SLABase, "_linear_branch", lambda self, q, k, v: seen.append("reference") or torch.zeros_like(q))
    m = core.SparseLinearAttention(128, 0.1, "relu", BLKQ=128, BLKK=64)
    q = torch.zeros(1, 256, 2, 128, dtype=torch.bfloat16, requires_grad=True)
    m(q, q, q)
    assert seen == ["reference"] and rec.calls == []
    prev = utils.set_linear_branch("fused")
    try:
        m(q, q, q)
    finally:
        utils.set_linear_branch(prev)
    assert seen == ["reference"] and rec.calls == [("fused", 2)]


def test_fake_kernels_match_the_abi_shapes():
    """The two tdb200_linear:: operators on fake CUDA tensors: the shapes and dtypes include/tdb200.h documents."""
    from torch._subclasses.fake_tensor import FakeTensorMode
    from turbodiffusion_b200 import _ops
    b, l, h, d = 2, 333, 3, 128
    with FakeTensorMode(allow_non_fake_inputs=False):
        x = [torch.empty(b, l, h, d, dtype=torch.float16, device="cuda") for _ in range(4)]
        w, bias = torch.empty(d, d, device="cuda"), torch.empty(d, device="cuda")
        o, mom = _ops.sla_linear_fwd(x[0], x[1], x[2], w, bias, 1)
        assert (o.shape, o.dtype, mom.shape, mom.dtype) == ((b, l, h, d), torch.float16, (b * h * d * (d + 1),), torch.float32)
        outs = _ops.sla_linear_bwd(x[0], x[1], x[2], x[3], mom, w, 1)
        assert [(t.shape, t.dtype) for t in outs] == [((b, l, h, d), torch.float16)] * 3 + [((d, d), torch.float32),
                                                                                            ((d,), torch.float32)]
    ops = {n for n in dir(torch.ops.tdb200_linear) if isinstance(getattr(torch.ops.tdb200_linear, n), torch._ops.OpOverloadPacket)}
    assert ops == {"sla_linear_fwd", "sla_linear_bwd", "sla_linear_tangent"}


@pytest.mark.parametrize("blk", [dict(BLKQ=128, BLKK=64), dict(BLKQ=64, BLKK=64)])
def test_training_forward_traces_as_one_graph(blk):
    """The "fused" training forward under torch.compile(fullgraph=True) on fake CUDA tensors: one graph holding both kernels'
    operators, and no torch linear branch."""
    from torch._subclasses.fake_tensor import FakeTensorMode
    from turbodiffusion_b200.SLA import core, utils
    graphs = []

    def backend(gm, example_inputs):
        graphs.append(gm)
        return gm.forward

    prev = utils.set_linear_branch("fused")
    try:
        torch._dynamo.reset()
        with FakeTensorMode():
            with torch.device("cuda"):
                m = core.SparseLinearAttention(128, 0.2, feature_map="relu", **blk)
            q, k, v = (torch.empty(1, 1000, 2, 128, dtype=torch.bfloat16, device="cuda", requires_grad=True) for _ in range(3))
            out = torch.compile(m, backend=backend, fullgraph=True, dynamic=False)(q, k, v)
    finally:
        utils.set_linear_branch(prev)
        torch._dynamo.reset()
    assert len(graphs) == 1 and out.requires_grad
    targets = {n.target for gm in graphs for n in gm.graph.nodes}
    assert torch.ops.tdb200_linear.sla_linear_fwd.default in targets
    assert torch.ops.tdb200.sla_attn16_fwd_lse.default in targets
    assert torch.ops.aten.bmm.default not in targets and torch.matmul not in targets and torch.nn.functional.linear not in targets


def test_proj_l_tangent_falls_back_to_the_torch_branch(monkeypatch):
    """Under "fused", a call whose proj_l weight carries a forward-mode tangent takes the torch branch."""
    import torch.autograd.forward_ad as fwAD
    from turbodiffusion_b200.SLA import core, utils
    rec = _Recorder(monkeypatch)
    seen = []
    monkeypatch.setattr(core._SLABase, "_linear_branch", lambda self, q, k, v: seen.append("reference") or torch.zeros_like(q))
    m = core.SparseLinearAttention(128, 0.1, "relu", BLKQ=128, BLKK=64)
    q = torch.zeros(1, 256, 2, 128, dtype=torch.bfloat16, requires_grad=True)
    params = {n: p.detach() for n, p in m.named_parameters()}
    prev = utils.set_linear_branch("fused")
    try:
        with fwAD.dual_level():
            w = fwAD.make_dual(params["proj_l.weight"], torch.ones_like(params["proj_l.weight"]))
            torch.func.functional_call(m, {**params, "proj_l.weight": w}, (q, q, q))
        torch.func.functional_call(m, params, (q, q, q))
    finally:
        utils.set_linear_branch(prev)
    assert seen == ["reference"] and rec.calls == [("fused", 2)]


def test_linear_branch_refuses_a_proj_tangent():
    import torch.autograd.forward_ad as fwAD
    from turbodiffusion_b200.SLA.core import linear_branch
    x = torch.zeros(1, 8, 1, 128, dtype=torch.bfloat16)
    with fwAD.dual_level():
        w = fwAD.make_dual(torch.zeros(128, 128), torch.ones(128, 128))
        with pytest.raises(NotImplementedError):
            linear_branch(x, x, x, w, torch.zeros(128))
