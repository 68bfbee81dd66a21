"""GPU checks of the dense attention backward (tdb200_attn_dense_bwd) and the training path of ops.dense_attention /
ops.dense_attention_jvp: dq, dk and dv against float64 autograd of softmax(q.k^T * s).v over ragged lengths in bf16 and fp16,
the lse of both lse forwards against float64 (lazy rescale included), bit identity of the training path's outputs with the
inference path's, gradients through the JVP's out, exact and reproducibility cases, CUDA-graph replay, the rows the backward
writes and the memory it must not read, and shape A at full size.

Bar.  Each gradient's rel-L2 error against float64 is at most 1.5x that of F.scaled_dot_product_attention's backward in the
same dtype, on the same inputs and incoming gradient (the dense forward's tests bound the output the same way).  Where the exact
gradient is zero (a single key: the softmax is constant, so dq = dk = 0), its RMS must stay below 1e-3 instead: a relative
error to zero is undefined."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
D = 128
SM = D ** -0.5
LOG2E = 1.0 / math.log(2.0)
F64 = torch.float64
BF16, FP16 = torch.bfloat16, torch.float16
DTYPES = [pytest.param(BF16, id="bf16"), pytest.param(FP16, id="fp16")]


def _rel(got, want):
    a, b = got.to(F64).flatten(), want.to(F64).flatten()
    return ((a - b).norm() / b.norm().clamp_min(1e-300)).item()


def _inputs(b, lq, lk, h, dtype, seed, device="cuda"):
    """q, k, v and an incoming gradient d_out"""
    g = torch.Generator().manual_seed(seed)
    shapes = [(b, lq, h, D), (b, lk, h, D), (b, lk, h, D), (b, lq, h, D)]
    return [torch.randn(*s, generator=g).to(dtype).to(device) for s in shapes]


def _attn(q, k, v, sm_scale):
    s = torch.einsum("bqhd,bkhd->bhqk", q, k) * sm_scale
    return torch.einsum("bhqk,bkhd->bqhd", torch.softmax(s, -1), v)


def exact_f64(q, k, v, d_out, sm_scale=SM):
    """(out, dq, dk, dv) of float64 autograd"""
    leaves = [t.detach().to(F64).requires_grad_() for t in (q, k, v)]
    out = _attn(*leaves, sm_scale)
    out.backward(d_out.to(F64))
    return (out.detach(), *(t.grad for t in leaves))


def sdpa_grads(q, k, v, d_out, sm_scale=SM):
    leaves = [t.detach().clone().requires_grad_() for t in (q, k, v)]
    out = F.scaled_dot_product_attention(*(t.transpose(1, 2) for t in leaves), scale=sm_scale).transpose(1, 2)
    out.backward(d_out)
    return [t.grad for t in leaves]


def ours(q, k, v, d_out, sm_scale=None):
    """(out, dq, dk, dv) through ops.dense_attention's training path"""
    from turbodiffusion_b200 import ops
    leaves = [t.detach().clone().requires_grad_() for t in (q, k, v)]
    out = ops.dense_attention(*leaves, sm_scale)
    out.backward(d_out)
    return (out.detach(), *(t.grad for t in leaves))


def _check_grads(got, lib, want, what, lk):
    errs = {}
    for name, a, s, r in zip(("dq", "dk", "dv"), got, lib, want):
        assert torch.isfinite(a).all(), (what, name)
        if lk == 1 and name != "dv":
            rms = a.double().pow(2).mean().sqrt().item()
            assert r.abs().max().item() == 0.0 and rms <= 1e-3, (what, name, rms)
            continue
        e, es = _rel(a, r), _rel(s, r)
        errs[name] = (e, es)
        assert e <= 1.5 * es, (what, name, e, es)
    print(what, " ".join(f"{n} {e:.2e} (sdpa {es:.2e})" for n, (e, es) in errs.items()))


# ------------------------------------------------------------------------------------------------------------ accuracy
LQS, LKS = (1, 77, 128, 200, 1000), (1, 64, 77, 129, 226, 512)
BH = [(1, 1), (1, 3), (2, 1), (2, 3)]
CASES = [(*BH[i % 4], lq, lk) for i, (lq, lk) in enumerate((lq, lk) for lq in LQS for lk in LKS)]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("b,h,lq,lk", [pytest.param(*c, id="b{}h{}-{}x{}".format(*c)) for c in CASES])
def test_gradients_against_float64(cuda, b, h, lq, lk, dtype):
    q, k, v, d_out = _inputs(b, lq, lk, h, dtype, seed=1000 * lq + lk)
    out, *grads = ours(q, k, v, d_out)
    assert all(g.dtype == dtype and g.is_contiguous() and g.shape == t.shape for g, t in zip(grads, (q, k, v)))
    _, *want = exact_f64(q, k, v, d_out)
    _check_grads(grads, sdpa_grads(q, k, v, d_out), want, f"({b}, {h}, {lq}, {lk}) {dtype}", lk)


def test_float32_inputs_get_float32_gradients_and_sm_scale_is_passed_on(cuda):
    q, k, v, d_out = (t.float() for t in _inputs(1, 200, 300, 2, BF16, seed=3))
    out, *grads = ours(q, k, v, d_out, sm_scale=0.5 * SM)
    assert out.dtype == torch.float32 and all(g.dtype == torch.float32 for g in grads)
    _, *grads16 = ours(*(t.bfloat16() for t in (q, k, v, d_out)), sm_scale=0.5 * SM)
    assert all(torch.equal(g, g16.float()) for g, g16 in zip(grads, grads16))
    ins16 = [t.bfloat16() for t in (q, k, v, d_out)]
    _, *want = exact_f64(*ins16, sm_scale=0.5 * SM)
    _check_grads(grads16, sdpa_grads(*ins16, sm_scale=0.5 * SM), want, "sm_scale", 300)


# ------------------------------------------------------------------------------------------------------------ lse
def _lse_of(entry, ins, dtype, b, lq, lk, h):
    """lse [b, h, lq] from one of the two lse forwards, called through the C entry point"""
    from turbodiffusion_b200 import _lib
    q, k, v = ins[:3]
    out, out_t = torch.empty_like(q), torch.empty_like(q)
    lse = torch.empty(b, h, lq, dtype=torch.float32, device="cuda")
    L, tag, st = _lib.lib(), _lib.DTYPE_TAG[dtype], _lib.stream_ptr(q.device)
    if entry == "fwd":
        rc = L.tdb200_attn_dense_fwd_lse(q.data_ptr(), k.data_ptr(), v.data_ptr(), tag, out.data_ptr(), lse.data_ptr(), b, lq, lk,
                                         h, D, SM, st)
    else:
        rc = L.tdb200_attn_dense_jvp_lse(q.data_ptr(), k.data_ptr(), v.data_ptr(), q.data_ptr(), k.data_ptr(), v.data_ptr(), tag,
                                         out.data_ptr(), out_t.data_ptr(), lse.data_ptr(), b, lq, lk, h, D, SM, st)
    _lib.check(rc, f"attn_dense_{entry}_lse")
    return lse


def _ramp_inputs(lq, lk, h, dtype, step):
    """Scores whose row maxima climb by `step` (log2 units) every 64 keys, so the lazy rescale (threshold 8) fires"""
    g = torch.Generator().manual_seed(11)
    u = torch.ones(D) / D ** 0.5
    q, k, v = torch.randn(1, lq, h, D, generator=g), torch.randn(1, lk, h, D, generator=g), torch.randn(1, lk, h, D, generator=g)
    a = 4.0
    q = 2.0 * (q - (q @ u)[..., None] * u) + a * u
    k = k + (step * (torch.arange(lk) // 64) / (a * SM * LOG2E))[None, :, None, None] * u
    return [t.to(dtype).cuda() for t in (q, k, v)]


@pytest.mark.parametrize("entry", ["fwd", "jvp"])
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("scores", ["random", "ramp"])
def test_lse_against_float64(cuda, entry, dtype, scores):
    b, lq, lk, h = (2, 333, 517, 3) if scores == "random" else (1, 300, 520, 2)
    ins = _inputs(b, lq, lk, h, dtype, seed=21) if scores == "random" else _ramp_inputs(lq, lk, h, dtype, step=10.0)
    s = torch.einsum("bqhd,bkhd->bhqk", ins[0].to(F64), ins[1].to(F64)) * SM
    want = torch.logsumexp(s, -1) * LOG2E
    if scores == "ramp":   # most rows' running maximum grows by more than 8 between 64-key and between 128-key tiles
        tiles = F.pad(s * LOG2E, (0, -lk % 64), value=-math.inf).view(b, h, lq, -1, 64).amax(-1)
        run = torch.cummax(tiles, -1).values
        assert ((run[..., 2::2] - run[..., :-2:2]) > 8).any(-1).float().mean().item() > 0.9
    lse = _lse_of(entry, ins, dtype, b, lq, lk, h)
    err = (lse.to(F64) - want).abs().max().item()
    print(f"lse {entry} {scores} {dtype}: max abs error {err:.2e}, |lse| up to {want.abs().max().item():.1f}")
    assert torch.isfinite(lse).all() and err <= 1e-4, err


# ------------------------------------------------------------------------------------------------------------ bit identity
@pytest.mark.parametrize("dtype", DTYPES)
def test_training_outputs_are_the_inference_bits(cuda, dtype):
    from turbodiffusion_b200 import ops
    q, k, v, _ = _inputs(2, 700, 300, 3, dtype, seed=31)
    q_t, k_t, v_t = (torch.randn_like(t) for t in (q, k, v))
    with torch.no_grad():
        ref = ops.dense_attention(q, k, v)
        ref_o, ref_t = ops.dense_attention_jvp(q, k, v, q_t, k_t, v_t)
    leaves = [t.clone().requires_grad_() for t in (q, k, v)]
    out = ops.dense_attention(*leaves)
    out_j, out_jt = ops.dense_attention_jvp(*leaves, q_t, k_t, v_t)
    assert out.requires_grad and out_j.requires_grad and not out_jt.requires_grad
    assert torch.equal(out.detach(), ref) and torch.equal(out_j.detach(), ref_o) and torch.equal(out_jt, ref_t)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("lq,lk", [(77, 512), (1000, 129)])
def test_gradients_through_the_jvp_output(cuda, dtype, lq, lk):
    from turbodiffusion_b200 import ops
    q, k, v, d_out = _inputs(2, lq, lk, 3, dtype, seed=41 + lq)
    leaves = [t.clone().requires_grad_() for t in (q, k, v)]
    tangents = [torch.randn_like(t).requires_grad_() for t in (q, k, v)]
    out, out_t = ops.dense_attention_jvp(*leaves, *tangents)
    assert out_t.requires_grad is False
    out.backward(d_out)
    assert all(t.grad is None for t in tangents)
    grads = [t.grad for t in leaves]
    _, *want = exact_f64(q, k, v, d_out)
    _check_grads(grads, sdpa_grads(q, k, v, d_out), want, f"jvp ({lq}, {lk}) {dtype}", lk)


# ------------------------------------------------------------------------------------------------------------ exact cases
@pytest.mark.parametrize("dtype", DTYPES)
def test_zero_incoming_gradient_gives_zero_gradients(cuda, dtype):
    q, k, v, d_out = _inputs(2, 333, 200, 3, dtype, seed=51)
    _, *grads = ours(q, k, v, torch.zeros_like(d_out))
    assert all(torch.equal(g, torch.zeros_like(g)) for g in grads)


@pytest.mark.parametrize("dtype", DTYPES)
def test_bits_are_reproducible_and_independent_of_the_other_heads(cuda, dtype):
    q, k, v, d_out = _inputs(2, 700, 300, 3, dtype, seed=61)
    first = ours(q, k, v, d_out)
    again = ours(q, k, v, d_out)
    assert all(torch.equal(a, b) for a, b in zip(first, again))
    one = ours(*(t[1:2, :, 2:3].contiguous() for t in (q, k, v, d_out)))
    assert all(torch.equal(a, b[1:2, :, 2:3]) for a, b in zip(one, first))


def _bwd_call(ins, out, lse, dq, dk, dv, ws, b, lq, lk, h, dtype):
    from turbodiffusion_b200 import _lib
    q, k, v, d_out = ins
    _lib.check(_lib.lib().tdb200_attn_dense_bwd(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), d_out.data_ptr(),
                                                lse.data_ptr(), _lib.DTYPE_TAG[dtype], dq.data_ptr(), dk.data_ptr(), dv.data_ptr(),
                                                ws.data_ptr(), ws.numel(), b, lq, lk, h, D, SM, _lib.stream_ptr(q.device)),
               "attn_dense_bwd")


def _fwd_lse_call(ins, out, lse, b, lq, lk, h, dtype):
    from turbodiffusion_b200 import _lib
    q, k, v = ins[:3]
    _lib.check(_lib.lib().tdb200_attn_dense_fwd_lse(q.data_ptr(), k.data_ptr(), v.data_ptr(), _lib.DTYPE_TAG[dtype], out.data_ptr(),
                                                    lse.data_ptr(), b, lq, lk, h, D, SM, _lib.stream_ptr(q.device)),
               "attn_dense_fwd_lse")


def _workspace(b, h, lq):
    from turbodiffusion_b200 import _lib
    return torch.empty(_lib.lib().tdb200_attn_dense_bwd_workspace_bytes(b, h, lq), dtype=torch.uint8, device="cuda")


def test_cuda_graph_replay_matches_eager(cuda):
    b, lq, lk, h = 1, 900, 512, 2
    ins = _inputs(b, lq, lk, h, BF16, seed=71)
    eager = ours(*ins, sm_scale=SM)
    out, lse = torch.empty_like(ins[0]), torch.empty(b, h, lq, dtype=torch.float32, device="cuda")
    dq, dk, dv = (torch.empty_like(t) for t in ins[:3])
    ws = _workspace(b, h, lq)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        _fwd_lse_call(ins, out, lse, b, lq, lk, h, BF16)
        _bwd_call(ins, out, lse, dq, dk, dv, ws, b, lq, lk, h, BF16)
    for t in (out, dq, dk, dv):
        t.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(a, b_) for a, b_ in zip((out, dq, dk, dv), eager))


# ------------------------------------------------------------------------------------------------------------ memory
@pytest.mark.parametrize("lq,lk", [(333, 77), (128, 130), (1, 1)])
def test_rows_past_lq_and_lk_are_not_written(cuda, lq, lk):
    """dq, dk and dv are the leading rows of sentinel-filled buffers: every row from lq (dq) or lk (dk, dv) on keeps its bits."""
    b, h, extra = 2, 3, 150
    ins = _inputs(b, lq, lk, h, BF16, seed=81 + lq)
    out, lse = torch.empty_like(ins[0]), torch.empty(b, h, lq, dtype=torch.float32, device="cuda")
    _fwd_lse_call(ins, out, lse, b, lq, lk, h, BF16)
    bufs = [torch.full((b * l + extra, h, D), 7.0, dtype=BF16, device="cuda") for l in (lq, lk, lk)]
    _bwd_call(ins, out, lse, *bufs, _workspace(b, h, lq), b, lq, lk, h, BF16)
    torch.cuda.synchronize()
    _, *want = ours(*ins, sm_scale=SM)
    for buf, g, l in zip(bufs, want, (lq, lk, lk)):
        assert torch.equal(buf[: b * l].view(b, l, h, D), g)
        assert (buf[b * l:] == 7.0).all()


@pytest.mark.parametrize("poison", [float("nan"), 1e4], ids=["nan", "1e4"])
@pytest.mark.parametrize("lq,lk", [(300, 77), (200, 130)])
def test_memory_past_the_tensors_is_never_read(cuda, lq, lk, poison):
    """q, k, v, out and d_out are the leading rows of allocations whose other rows hold NaN or 1e4: every gradient equals, bit
    for bit, that of tight copies."""
    b, h = 1, 2
    ins = _inputs(b, lq, lk, h, BF16, seed=91 + lk)
    out, lse = torch.empty_like(ins[0]), torch.empty(b, h, lq, dtype=torch.float32, device="cuda")
    _fwd_lse_call(ins, out, lse, b, lq, lk, h, BF16)

    def poisoned(t):
        big = torch.full((b, 256 if t.shape[1] <= 256 else 512, h, D), poison, dtype=BF16, device="cuda")
        big[:, : t.shape[1]] = t
        view = big[:, : t.shape[1]]
        assert view.is_contiguous() and view.data_ptr() == big.data_ptr()
        return view

    ref = [torch.empty_like(t) for t in ins[:3]]
    _bwd_call(ins, out, lse, *ref, _workspace(b, h, lq), b, lq, lk, h, BF16)
    got = [torch.empty_like(t) for t in ins[:3]]
    _bwd_call([poisoned(t) for t in ins], poisoned(out), lse, *got, _workspace(b, h, lq), b, lq, lk, h, BF16)
    torch.cuda.synchronize()
    assert all(torch.isfinite(g).all() and torch.equal(g, r) for g, r in zip(got, ref))


# ------------------------------------------------------------------------------------------------------------ full size
def test_shape_a_cross_attention(cuda):
    """Wan2.1-1.3B at 480p, cross-attention: 32760 queries over 512 text keys, 12 heads of 128; every gradient against
    float64."""
    lq, lk, h = 32760, 512, 12
    g = torch.Generator(device="cuda").manual_seed(101)
    q, d_out = (torch.randn(1, lq, h, D, generator=g, device="cuda").bfloat16() for _ in range(2))
    k, v = (torch.randn(1, lk, h, D, generator=g, device="cuda").bfloat16() for _ in range(2))
    _, *grads = ours(q, k, v, d_out)
    lib = sdpa_grads(q, k, v, d_out)
    _, *want = exact_f64(q, k, v, d_out)
    _check_grads(grads, lib, want, "shape A cross", lk)


def _reference_rows(q, k, v, d_out, heads, q_rows, k_rows, chunk=2048):
    """fp32 (no TF32) dq rows q_rows[i] and dk, dv rows k_rows[i] of head heads[i], from chunked passes over all queries."""
    assert not torch.backends.cuda.matmul.allow_tf32
    lq = q.shape[1]
    dq, dk, dv = [], [], []
    for hh, qr, kr in zip(heads, q_rows, k_rows):
        qh, kh, vh, gh = (t[0, :, hh].float() for t in (q, k, v, d_out))       # [L, D]
        s = (qh[qr] @ kh.T) * SM
        p = torch.softmax(s, -1)
        o = p @ vh
        ds = p * (gh[qr] @ vh.T - (gh[qr] * o).sum(-1, keepdim=True))
        dq.append((ds @ kh) * SM)
        dk_h = torch.zeros(len(kr), D, device=q.device)
        dv_h = torch.zeros(len(kr), D, device=q.device)
        for c in range(0, lq, chunk):
            s = (qh[c:c + chunk] @ kh.T) * SM
            p = torch.softmax(s, -1)
            delta = (gh[c:c + chunk] * (p @ vh)).sum(-1, keepdim=True)
            pk = p[:, kr]
            ds = pk * (gh[c:c + chunk] @ vh[kr].T - delta)
            dv_h += pk.T @ gh[c:c + chunk]
            dk_h += (ds.T @ qh[c:c + chunk]) * SM
        dk.append(dk_h)
        dv.append(dv_h)
    return torch.stack(dq), torch.stack(dk), torch.stack(dv)


def test_shape_a_self_attention_on_sampled_rows(cuda):
    """Dense self-attention at shape A (32760 x 32760, 12 heads of 128): 64 sampled rows of dq, dk and dv in three heads, the
    first and last rows among them, against an fp32 reference that passes over every query in chunks."""
    l, h, n = 32760, 12, 64
    g = torch.Generator(device="cuda").manual_seed(111)
    q, k, v, d_out = (torch.randn(1, l, h, D, generator=g, device="cuda").bfloat16() for _ in range(4))
    _, *grads = ours(q, k, v, d_out)
    lib = sdpa_grads(q, k, v, d_out)
    heads = [0, 5, 11]
    rows = [torch.randperm(l, generator=torch.Generator().manual_seed(120 + i))[:n].cuda() for i in range(2 * len(heads))]
    for r in rows:
        r[0], r[1] = 0, l - 1
    q_rows, k_rows = rows[: len(heads)], rows[len(heads):]
    want = _reference_rows(q, k, v, d_out, heads, q_rows, k_rows)
    pick = lambda t, sel: torch.stack([t[0, r, hh] for hh, r in zip(heads, sel)])
    errs = []
    for name, a, s, w, sel in zip(("dq", "dk", "dv"), grads, lib, want, (q_rows, k_rows, k_rows)):
        assert torch.isfinite(a).all()
        e, es = _rel(pick(a, sel), w), _rel(pick(s, sel), w)
        errs.append(f"{name} {e:.2e} (sdpa {es:.2e})")
        assert e <= 1.5 * es, (name, e, es)
    print("shape A self, sampled rows:", " ".join(errs))
