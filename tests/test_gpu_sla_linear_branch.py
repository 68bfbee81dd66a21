"""SparseLinearAttention's linear branch on the CUDA kernels (SLA.core.linear_branch, tdb200_sla_linear_fwd / _bwd) against
float64, next to the reference torch composition (the module's _linear_branch) and a float32 restatement that rounds where the
kernels do (include/tdb200.h): o_l, dq, dk, dv, dW and db."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

DTYPES = {"bf16": torch.bfloat16, "fp16": torch.float16}
FEATURES = ("softmax", "elu", "relu")


@pytest.fixture(scope="module", autouse=True)
def _lib():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from turbodiffusion_b200 import _lib as L
    L.lib()


def _phi(x, feature):
    if feature == "softmax":
        return F.softmax(x, dim=-1)
    if feature == "elu":
        return F.elu(x) + 1
    return F.relu(x)


def _exact(q, k, v, w, b, feature):
    """The formula in float64 with autograd, q, k, v [B, L, H, D]."""
    qh, kh, vh = (t.transpose(1, 2) for t in (q, k, v))
    cq, ck = _phi(qh, feature), _phi(kh, feature)
    m = ck.transpose(-1, -2) @ vh
    s = ck.sum(-2, keepdim=True)
    u = (cq @ m) / (1e-5 + (cq * s).sum(-1, keepdim=True))
    return (u @ w.T + b).transpose(1, 2)


def _rnd(x, dt):
    return x.to(dt).float()


def _rnd_mat(x, dt):
    """x rounded to dt after a power-of-two scale putting the max of each trailing matrix near 2^14 (exact in fp32)."""
    m = x.abs().amax(dim=(-1, -2), keepdim=True).clamp_min(1e-30)
    sc = torch.exp2(14 - torch.floor(torch.log2(m)))
    return _rnd(x * sc, dt) / sc


def _rnd_rows(x, dt):
    m = x.abs().amax(dim=-1, keepdim=True).clamp_min(1e-30)
    sc = torch.exp2(-torch.floor(torch.log2(m)))
    return _rnd(x * sc, dt) / sc


def _vjp_phi(x, dc, feature):
    if feature == "softmax":
        c = F.softmax(x, dim=-1)
        return c * (dc - (c * dc).sum(-1, keepdim=True))
    if feature == "elu":
        return dc * torch.where(x > 0, torch.ones_like(x), torch.exp(x))
    return dc * (x > 0).float()


def _restated(q, k, v, w, b, g, feature):
    """Forward and backward in float32 at the kernels' rounding points: (o, dq, dk, dv, dW, db)."""
    dt = q.dtype
    qh, kh, vh, gh = (t.transpose(1, 2).float() for t in (q, k, v, g))
    cq, ck = _rnd(_phi(qh, feature), dt), _rnd(_phi(kh, feature), dt)
    m = ck.transpose(-1, -2) @ vh
    s = ck.sum(-2, keepdim=True)
    mt = _rnd_mat(m, dt)
    den = 1e-5 + (cq * s).sum(-1, keepdim=True)
    u = (cq @ mt) / den
    wt = _rnd(w, dt)
    o = _rnd(u, dt) @ wt.T + b
    du = gh @ wt
    e = (du * u).sum(-1, keepdim=True) / den
    dcq = (_rnd(du, dt) @ mt.transpose(-1, -2)) / den - e * s
    dm = cq.transpose(-1, -2) @ _rnd_rows(du / den, dt)
    ds = -(e * cq).sum(-2, keepdim=True)
    dmt = _rnd_mat(dm, dt)
    dck = vh @ dmt.transpose(-1, -2) + ds
    dv = ck @ dmt
    dq, dk = _vjp_phi(qh, dcq, feature), _vjp_phi(kh, dck, feature)
    dw = (gh.transpose(-1, -2) @ _rnd(u, dt)).sum((0, 1))
    db = gh.sum((0, 1, 2))
    tr = lambda t: _rnd(t.transpose(1, 2), dt)  # noqa: E731   outputs in T
    return tr(o), tr(dq), tr(dk), tr(dv), dw, db


def _rel(x, ref):
    return ((x.double() - ref).norm() / ref.norm().clamp_min(1e-300)).item()


def _inputs(b, l, h, dtype, seed, q_scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    q, k, v, do = (torch.randn(b, l, h, 128, generator=g, device="cuda").to(dtype) for _ in range(4))
    q = (q.float() * q_scale).to(dtype)
    w = torch.randn(128, 128, generator=g, device="cuda") * 128 ** -0.5
    bias = torch.randn(128, generator=g, device="cuda") * 0.1
    return q, k, v, do, w, bias


def _fused(q, k, v, do, w, bias, feature):
    from turbodiffusion_b200.SLA.core import linear_branch
    q, k, v = (t.detach().requires_grad_() for t in (q, k, v))
    w, bias = w.detach().requires_grad_(), bias.detach().requires_grad_()
    o = linear_branch(q, k, v, w, bias, feature)
    o.backward(do)
    return o.detach(), q.grad, k.grad, v.grad, w.grad, bias.grad


def _reference(q, k, v, do, w, bias, feature):
    from turbodiffusion_b200.SLA.core import SparseLinearAttention
    m = SparseLinearAttention(128, 0.1, feature, BLKQ=128, BLKK=64, use_bf16=q.dtype == torch.bfloat16).cuda()
    with torch.no_grad():
        m.proj_l.weight.copy_(w)
        m.proj_l.bias.copy_(bias)
    q, k, v = (t.detach().requires_grad_() for t in (q, k, v))
    o = m._linear_branch(q, k, v)
    o.backward(do)
    return o.detach(), q.grad, k.grad, v.grad, m.proj_l.weight.grad, m.proj_l.bias.grad


def _float64(q, k, v, do, w, bias, feature):
    q, k, v = (t.detach().double().requires_grad_() for t in (q, k, v))
    w, bias = w.detach().double().requires_grad_(), bias.detach().double().requires_grad_()
    o = _exact(q, k, v, w, bias, feature)
    o.backward(do.double())
    return o.detach(), q.grad, k.grad, v.grad, w.grad, bias.grad


NAMES = ("o_l", "dq", "dk", "dv", "dW", "db")


def _check_bars(q, k, v, do, w, bias, feature, label, ref_bar=True):
    got = _fused(q, k, v, do, w, bias, feature)
    ex = _float64(q, k, v, do, w, bias, feature)
    r32 = _restated(q, k, v, w, bias, do, feature)
    ref = _reference(q, k, v, do, w, bias, feature)
    for name, x, e, x32, xr in zip(NAMES, got, ex, r32, ref):
        assert torch.isfinite(x).all(), (label, name)
        err, err32, errr = _rel(x, e), _rel(x32, e), _rel(xr, e)
        print(f"{label} {name}: fused {err:.3e}  float32 restatement {err32:.3e}  reference torch {errr:.3e}")
        assert err <= 1.5 * err32 + 1e-6, (label, name, err, err32)
        if ref_bar:
            assert err <= errr, (label, name, err, errr)
    return got


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("feature", FEATURES)
@pytest.mark.parametrize("b,l,h", [(1, 1000, 2), (2, 333, 3), (1, 512, 2), (1, 40, 2)])
def test_operator_against_float64(dtype, feature, b, l, h):
    q, k, v, do, w, bias = _inputs(b, l, h, DTYPES[dtype], seed=l + 7 * h)
    _check_bars(q, k, v, do, w, bias, feature, f"{dtype} {feature} b={b} l={l} h={h}")


@pytest.mark.parametrize("dtype", list(DTYPES))
def test_dead_relu_channel(dtype):
    """relu: channel 5 is negative on every key, and the queries sit on it: den = 1e-5 + tiny, 1/den near 1e5."""
    q, k, v, do, w, bias = _inputs(1, 1000, 2, DTYPES[dtype], seed=3)
    k[..., 5] = -k[..., 5].abs() - 0.1
    q = q.float()
    q[..., 5] = 6.0
    q[:, ::2, :, :5] = -1.0
    q[:, ::2, :, 6:] = -1.0           # even rows: only the dead channel is live
    q = q.to(DTYPES[dtype])
    got = _check_bars(q, k, v, do, w, bias, "relu", f"{dtype} dead relu channel", ref_bar=False)
    ref = _reference(q, k, v, do, w, bias, "relu")
    print("reference path finite:", [bool(torch.isfinite(x).all()) for x in ref])
    assert all(torch.isfinite(x).all() for x in got)


@pytest.mark.parametrize("dtype", list(DTYPES))
def test_softmax_near_one_hot(dtype):
    q, k, v, do, w, bias = _inputs(1, 1000, 2, DTYPES[dtype], seed=5, q_scale=12.0)
    _check_bars(q, k, v, do, w, bias, "softmax", f"{dtype} softmax near one-hot", ref_bar=False)


def test_long_relu_fp16_moments_past_fp16_range():
    """relu at l = 32760 with mean 8 in v: M passes 65504, which the kernels scale into range."""
    q, k, v, do, w, bias = _inputs(1, 32760, 1, torch.float16, seed=9)
    v = (v.float() + 8).half()
    got = _check_bars(q, k, v, do, w, bias, "relu", "fp16 relu l=32760 v+8", ref_bar=False)
    ref = _reference(q, k, v, do, w, bias, "relu")
    print("reference path finite:", [bool(torch.isfinite(x).all()) for x in ref])


def test_deterministic_and_heads_independent():
    q, k, v, do, w, bias = _inputs(2, 1000, 3, torch.bfloat16, seed=11)
    a = _fused(q, k, v, do, w, bias, "softmax")
    b = _fused(q, k, v, do, w, bias, "softmax")
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    one = _fused(q[:, :, 1:2], k[:, :, 1:2], v[:, :, 1:2], do[:, :, 1:2], w, bias, "softmax")
    for x, y in zip(a[:4], one[:4]):
        assert torch.equal(x[:, :, 1:2], y)


def test_poisoned_tails_and_unwritten_rows():
    """Inputs are views into larger buffers whose rows past l hold NaN; outputs beyond l are not written."""
    from turbodiffusion_b200 import _ops
    b, l, h = 1, 333, 2
    q, k, v, do, w, bias = _inputs(b, l, h, torch.bfloat16, seed=13)
    clean = _fused(q, k, v, do, w, bias, "elu")

    def poisoned(t):
        big = torch.full((b, l + 64, h, 128), float("nan"), dtype=t.dtype, device="cuda")
        big[:, :l] = t
        return big[:, :l]    # contiguous prefix of the buffer: rows past l are NaN in memory

    qp, kp, vp, dop = (poisoned(t) for t in (q, k, v, do))
    o, mom = _ops.sla_linear_fwd(qp, kp, vp, w, bias, 1)
    assert torch.equal(o, clean[0])
    dq, dk, dv, dw, db = _ops.sla_linear_bwd(qp, kp, vp, dop, mom, w, 1)
    for x, y in zip((dq, dk, dv, dw, db), clean[1:]):
        assert torch.equal(x, y)
    # rows past l of the outputs: the kernels are handed views of sentinel-filled buffers
    from turbodiffusion_b200._lib import DTYPE_TAG, lib, ptr, stream_ptr
    out = torch.full((b, l + 64, h, 128), 7.0, dtype=torch.bfloat16, device="cuda")
    rc = lib().tdb200_sla_linear_fwd(ptr(q), ptr(mom), ptr(mom) + 4 * b * h * 128 * 128, ptr(w), ptr(bias), DTYPE_TAG[q.dtype],
                                     1, ptr(out), b, l, h, 128, stream_ptr(q.device))
    assert rc == 0
    assert torch.equal(out[:, :l], clean[0]) and (out[:, l:] == 7.0).all()


def test_cuda_graph_replays_eager_bits():
    from turbodiffusion_b200 import _ops
    q, k, v, do, w, bias = _inputs(1, 1000, 2, torch.float16, seed=17)
    eager_o, mom = _ops.sla_linear_fwd(q, k, v, w, bias, 2)
    eager_g = _ops.sla_linear_bwd(q, k, v, do, mom, w, 2)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _ops.sla_linear_fwd(q, k, v, w, bias, 2)
        _ops.sla_linear_bwd(q, k, v, do, mom, w, 2)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        go, gmom = _ops.sla_linear_fwd(q, k, v, w, bias, 2)
        gg = _ops.sla_linear_bwd(q, k, v, do, gmom, w, 2)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(go, eager_o) and torch.equal(gmom, mom)
    for x, y in zip(gg, eager_g):
        assert torch.equal(x, y)


def test_shape_a_sampled_rows():
    """Shape A (l = 32760, 12 heads): o_l and dq on sampled rows, dk / dv / dW against float64 on full tensors."""
    q, k, v, do, w, bias = _inputs(1, 32760, 12, torch.bfloat16, seed=19)
    got = _fused(q, k, v, do, w, bias, "softmax")
    ex = _float64(q, k, v, do, w, bias, "softmax")
    ref = _reference(q, k, v, do, w, bias, "softmax")
    rows = torch.arange(0, 32760, 97, device="cuda")
    for name, x, e, r in zip(NAMES, got, ex, ref):
        xs, es, rs = (t[:, rows] if t.dim() == 4 else t for t in (x, e, r))
        err, errr = _rel(xs, es), _rel(rs, es)
        print(f"shape A {name}: fused {err:.3e}  reference torch {errr:.3e}")
        assert err <= errr, (name, err, errr)


def _module(feature, blk, dtype, seed):
    from turbodiffusion_b200.SLA.core import SparseLinearAttention
    torch.manual_seed(seed)
    m = SparseLinearAttention(128, 0.2, feature, BLKQ=blk[0], BLKK=blk[1], use_bf16=dtype == torch.bfloat16).cuda()
    with torch.no_grad():
        m.proj_l.weight.normal_(0, 128 ** -0.5)
        m.proj_l.bias.normal_(0, 0.1)
    return m


def _train_step(m, q, k, v, do):
    q, k, v = (t.detach().requires_grad_() for t in (q, k, v))
    m.zero_grad()
    o = m(q, k, v)
    o.backward(do)
    return o.detach(), q.grad, k.grad, v.grad, m.proj_l.weight.grad.clone(), m.proj_l.bias.grad.clone()


@pytest.mark.parametrize("blk", [(128, 64), (64, 64)])
@pytest.mark.parametrize("feature", FEATURES)
def test_module_training_fused_matches_reference_path(blk, feature):
    """The fused training step against the default one: the sparse branch is the same kernels, so the difference is the
    linear branch's, which is checked above against float64; here the whole step must stay within the reference step's
    own bf16 distance from the fused linear branch (rel-L2 2e-2) and the default setting must be untouched."""
    from turbodiffusion_b200.SLA import utils
    q, k, v, do, _, _ = _inputs(1, 1000, 2, torch.bfloat16, seed=23)
    m = _module(feature, blk, torch.bfloat16, 1)
    base = _train_step(m, q, k, v, do)
    prev = utils.set_linear_branch("fused")
    try:
        fused = _train_step(m, q, k, v, do)
    finally:
        utils.set_linear_branch(prev)
    again = _train_step(m, q, k, v, do)
    for name, x, y, z in zip(NAMES, base, fused, again):
        assert torch.equal(x, z), name             # the default path is unchanged by having run the fused one
        assert torch.isfinite(y).all(), name
        err = _rel(y, x.double())
        print(f"module {feature} {blk} {name}: fused vs reference path {err:.3e}")
        assert err < 2e-2, (name, err)


def test_compiled_training_step_has_no_graph_breaks():
    from turbodiffusion_b200.SLA import utils
    q, k, v, do, _, _ = _inputs(1, 1000, 2, torch.bfloat16, seed=31)
    m = _module("elu", (128, 64), torch.bfloat16, 3)
    prev = utils.set_linear_branch("fused")
    try:
        eager = _train_step(m, q, k, v, do)

        def step(q, k, v):
            return m(q, k, v)

        qq, kk, vv = (t.detach().requires_grad_() for t in (q, k, v))
        explain = torch._dynamo.explain(step)(qq, kk, vv)
        assert explain.graph_break_count == 0, explain.break_reasons
        torch._dynamo.reset()
        cstep = torch.compile(step, fullgraph=True)
        m.zero_grad()
        qq, kk, vv = (t.detach().requires_grad_() for t in (q, k, v))
        o = cstep(qq, kk, vv)
        o.backward(do)
        compiled = (o.detach(), qq.grad, kk.grad, vv.grad, m.proj_l.weight.grad, m.proj_l.bias.grad)
    finally:
        utils.set_linear_branch(prev)
        torch._dynamo.reset()
    for name, x, y in zip(NAMES, eager, compiled):
        err = _rel(y, x.double())
        print(f"compiled vs eager {name}: {err:.3e}")
        assert err < 5e-3, (name, err)


# ------------------------------------------------------------------------------------------------ tangent
def _restated_tangent(q, k, v, w, qt, kt, vt, feature):
    """o_l_t in float32 at the tangent kernels' rounding points."""
    dt = q.dtype
    qh, kh, vh, qth, kth, vth = (t.transpose(1, 2).float() for t in (q, k, v, qt, kt, vt))

    def jphi(x, xt):
        c = _phi(x, feature)
        if feature == "softmax":
            return c * (xt - (c * xt).sum(-1, keepdim=True))
        return xt * (torch.where(x > 0, torch.ones_like(x), torch.exp(x)) if feature == "elu" else (x > 0).float())

    cq, ck = _rnd(_phi(qh, feature), dt), _rnd(_phi(kh, feature), dt)
    cqd, ckd = jphi(qh, qth), jphi(kh, kth)
    m, s = ck.transpose(-1, -2) @ vh, ck.sum(-2, keepdim=True)
    md = _rnd(ckd, dt).transpose(-1, -2) @ vh + ck.transpose(-1, -2) @ vth
    sd = ckd.sum(-2, keepdim=True)
    mt, mdt = _rnd_mat(m, dt), _rnd_mat(md, dt)
    den = 1e-5 + (cq * s).sum(-1, keepdim=True)
    dden = (cqd * s).sum(-1, keepdim=True) + (cq * sd).sum(-1, keepdim=True)
    u = (cq @ mt) / den
    ud = (_rnd(cqd, dt) @ mt + cq @ mdt) / den - u * dden / den
    return _rnd((_rnd(ud, dt) @ _rnd(w, dt).T).transpose(1, 2), dt)


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("feature", FEATURES)
@pytest.mark.parametrize("b,l,h", [(1, 1000, 2), (2, 333, 3), (1, 512, 2), (1, 40, 2)])
def test_tangent_against_float64(dtype, feature, b, l, h):
    from turbodiffusion_b200.SLA.core import linear_branch_jvp
    q, k, v, _, w, bias = _inputs(b, l, h, DTYPES[dtype], seed=3 * l + h)
    qt, kt, vt, _, _, _ = _inputs(b, l, h, DTYPES[dtype], seed=5 * l + h)
    o, ot = linear_branch_jvp(q, k, v, qt, kt, vt, w, bias, feature)
    _, ex = torch.func.jvp(lambda a, c, e: _exact(a, c, e, w.double(), bias.double(), feature),
                           (q.double(), k.double(), v.double()), (qt.double(), kt.double(), vt.double()))
    r32 = _restated_tangent(q, k, v, w, qt, kt, vt, feature)
    m = _module(feature, (128, 64), DTYPES[dtype], 0)
    with torch.no_grad():
        m.proj_l.weight.copy_(w)
        m.proj_l.bias.copy_(bias)
    import torch.autograd.forward_ad as fwAD
    with fwAD.dual_level():
        ref = fwAD.unpack_dual(m._linear_branch(fwAD.make_dual(q, qt), fwAD.make_dual(k, kt), fwAD.make_dual(v, vt))).tangent
    err, err32, errr = _rel(ot, ex), _rel(r32, ex), _rel(ref, ex)
    print(f"{dtype} {feature} b={b} l={l} h={h} o_l_t: fused {err:.3e}  float32 restatement {err32:.3e}  "
          f"reference torch {errr:.3e}")
    assert torch.isfinite(ot).all()
    assert err <= 1.5 * err32 + 1e-6 and err <= errr, (err, err32, errr)
    assert torch.equal(o, _fused(q, k, v, torch.zeros_like(q), w, bias, feature)[0])


def test_tangent_dead_relu_channel_fp16():
    from turbodiffusion_b200.SLA.core import linear_branch_jvp
    q, k, v, _, w, bias = _inputs(1, 1000, 2, torch.float16, seed=3)
    qt, kt, vt, _, _, _ = _inputs(1, 1000, 2, torch.float16, seed=4)
    k[..., 5] = -k[..., 5].abs() - 0.1
    q = q.float()
    q[..., 5] = 6.0
    q[:, ::2, :, :5] = -1.0
    q[:, ::2, :, 6:] = -1.0
    q = q.half()
    _, ot = linear_branch_jvp(q, k, v, qt, kt, vt, w, bias, "relu")
    _, ex = torch.func.jvp(lambda a, c, e: _exact(a, c, e, w.double(), bias.double(), "relu"),
                           (q.double(), k.double(), v.double()), (qt.double(), kt.double(), vt.double()))
    err, err32 = _rel(ot, ex), _rel(_restated_tangent(q, k, v, w, qt, kt, vt, "relu"), ex)
    print(f"fp16 dead relu channel o_l_t: fused {err:.3e}  float32 restatement {err32:.3e}")
    assert torch.isfinite(ot).all() and err <= 1.5 * err32 + 1e-6


def test_tangent_deterministic_heads_independent_and_graph():
    from turbodiffusion_b200 import _ops
    q, k, v, _, w, bias = _inputs(2, 1000, 3, torch.bfloat16, seed=41)
    qt, kt, vt, _, _, _ = _inputs(2, 1000, 3, torch.bfloat16, seed=42)
    _, mom = _ops.sla_linear_fwd(q, k, v, w, bias, 0)
    a = _ops.sla_linear_tangent(q, k, v, qt, kt, vt, mom, w, 0)
    assert torch.equal(a, _ops.sla_linear_tangent(q, k, v, qt, kt, vt, mom, w, 0))
    sl = [t[:, :, 1:2].contiguous() for t in (q, k, v, qt, kt, vt)]
    _, mom1 = _ops.sla_linear_fwd(*sl[:3], w, bias, 0)
    assert torch.equal(a[:, :, 1:2], _ops.sla_linear_tangent(*sl, mom1, w, 0))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _ops.sla_linear_tangent(q, k, v, qt, kt, vt, mom, w, 0)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        g = _ops.sla_linear_tangent(q, k, v, qt, kt, vt, mom, w, 0)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(g, a)


# ------------------------------------------------------------------------------------------------ module against float64
def _sparse_mask(sel, l, blkq):
    sm = sel["sparse_map"].bool()
    return sm.repeat_interleave(blkq, 2)[:, :, :l].repeat_interleave(64, 3)[:, :, :, :l]


def _module_exact(q, k, v, mask, w, bias, feature):
    """float64 SparseLinearAttention: softmax attention restricted to `mask` plus the linear branch and proj_l."""
    qh, kh, vh = (t.transpose(1, 2) for t in (q, k, v))
    s = (qh @ kh.transpose(-1, -2)) * 128 ** -0.5
    p = torch.softmax(s.masked_fill(~mask, float("-inf")), -1)
    return (p @ vh).transpose(1, 2) + _exact(q, k, v, w, bias, feature)


def _bars(got, want, ref=None, what=""):
    g, w = got.double().flatten(), want.flatten()
    cos = (g @ w / (g.norm() * w.norm())).item()
    rel = _rel(got, want)
    extra = f"  reference path {_rel(ref, want):.3e}" if ref is not None else ""
    print(f"{what}: rel {rel:.3e} cos {cos:.6f}{extra}")
    assert cos >= 0.999 and rel <= 2e-2, (what, rel, cos)


def _selection(m, q, k, v):
    """The block selection of the training forward (forward_jvp and forward_ad select the same blocks from the same q, k)."""
    m._keep_selection = {}
    try:
        m(q.detach().requires_grad_(), k, v)
        return dict(m._keep_selection)
    finally:
        m._keep_selection = None


@pytest.mark.parametrize("blk", [(128, 64), (64, 64)])
@pytest.mark.parametrize("feature", FEATURES)
def test_module_training_against_float64(blk, feature):
    from turbodiffusion_b200.SLA import utils
    q, k, v, do, _, _ = _inputs(1, 1000, 2, torch.bfloat16, seed=51)
    m = _module(feature, blk, torch.bfloat16, 4)
    sel = _selection(m, q, k, v)
    mask = _sparse_mask(sel, 1000, blk[0])
    args = [t.double().requires_grad_() for t in (q, k, v)]
    w64, b64 = (p.detach().double().requires_grad_() for p in m._proj)
    o64 = _module_exact(*args, mask, w64, b64, feature)
    o64.backward(do.double())
    want = (o64.detach(), *(a.grad for a in args), w64.grad, b64.grad)
    ref = _train_step(m, q, k, v, do)
    prev = utils.set_linear_branch("fused")
    try:
        got = _train_step(m, q, k, v, do)
    finally:
        utils.set_linear_branch(prev)
    for name, x, e, r in zip(("o",) + NAMES[1:], got, want, ref):
        _bars(x, e, r, f"module {feature} {blk} {name}")


def test_module_jvp_paths_against_float64_and_bits():
    """forward_jvp with and without grad give the same bits; forward_ad with grad gives the training path's gradient bits;
    torch.func.jvp through forward gives the training output's bits; tangents meet the bars against float64."""
    import torch.autograd.forward_ad as fwAD
    from turbodiffusion_b200.SLA import utils
    q, k, v, do, _, _ = _inputs(1, 1000, 2, torch.bfloat16, seed=61)
    qt, kt, vt, _, _, _ = _inputs(1, 1000, 2, torch.bfloat16, seed=62)
    m = _module("elu", (128, 64), torch.bfloat16, 5)
    mask = _sparse_mask(_selection(m, q, k, v), 1000, 128)
    w64, b64 = (p.detach().double() for p in m._proj)
    o64, ot64 = torch.func.jvp(lambda a, c, e: _module_exact(a, c, e, mask, w64, b64, "elu"),
                               (q.double(), k.double(), v.double()), (qt.double(), kt.double(), vt.double()))
    prev = utils.set_linear_branch("fused")
    try:
        with torch.no_grad():
            o_ng, ot_ng = m.forward_jvp(q, k, v, qt, kt, vt)
        train = _train_step(m, q, k, v, do)
        qg, kg, vg = (t.detach().requires_grad_() for t in (q, k, v))
        o_g, ot_g = m.forward_jvp(qg, kg, vg, qt, kt, vt)
        assert torch.equal(o_g.detach(), o_ng) and torch.equal(ot_g, ot_ng)
        assert torch.equal(o_ng, train[0])
        m.zero_grad()
        with fwAD.dual_level():
            qd, kd, vd = (t.detach().requires_grad_() for t in (q, k, v))
            o = m(fwAD.make_dual(qd, qt), fwAD.make_dual(kd, kt), fwAD.make_dual(vd, vt))
            o_p, o_t = fwAD.unpack_dual(o)
            o_p.backward(do)
        for name, x, y in zip(NAMES[1:], (qd.grad, kd.grad, vd.grad, m.proj_l.weight.grad, m.proj_l.bias.grad), train[1:]):
            assert torch.equal(x, y), name
        fo, fot = torch.func.jvp(lambda a, c, e: m(a, c, e), (q, k, v), (qt, kt, vt))
        assert torch.equal(fo, train[0]) and torch.equal(o_p.detach(), train[0])
    finally:
        utils.set_linear_branch(prev)
    _bars(ot_ng, ot64, what="forward_jvp o_t")
    _bars(o_t, ot64, what="forward_ad o_t")
    _bars(fot, ot64, what="torch.func.jvp o_t")
    _bars(o_ng, o64, what="forward_jvp o")


def test_proj_l_tangent_takes_the_torch_branch():
    """A forward-mode tangent on proj_l's weight: the fused setting gives the reference setting's bits."""
    from turbodiffusion_b200.SLA import utils
    q, k, v, _, _, _ = _inputs(1, 1000, 2, torch.bfloat16, seed=71)
    m = _module("relu", (128, 64), torch.bfloat16, 6)
    params = {n: p.detach() for n, p in m.named_parameters()}
    wt = torch.randn_like(params["proj_l.weight"])
    qg = q.detach().requires_grad_()

    def f(w):
        return torch.func.functional_call(m, {**params, "proj_l.weight": w}, (qg, k, v))

    ref = torch.func.jvp(f, (params["proj_l.weight"],), (wt,))
    prev = utils.set_linear_branch("fused")
    try:
        got = torch.func.jvp(f, (params["proj_l.weight"],), (wt,))
    finally:
        utils.set_linear_branch(prev)
    assert torch.equal(ref[0], got[0]) and torch.equal(ref[1], got[1])
    assert ref[1].abs().sum() > 0
