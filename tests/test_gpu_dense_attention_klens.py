"""GPU checks of the dense attention operators with per-sample key lengths (k_lens: tdb200_attn_dense_{fwd,fwd_lse,jvp,jvp_lse,
tangent,bwd}_kl behind ops.dense_attention / ops.dense_attention_jvp).

Bit identity with trimming.  For every batch entry i with L = k_lens[i] > 0, out, lse, out_t (from the fused JVP and from the
forward-AD rule's tangent kernel), dq, and the rows < L of dk and dv are byte-identical to the operator without k_lens called on
entry i alone with its keys cut to L; rows >= L of dk and dv are zero.  Key and value rows past L (and their tangents) are
filled with large finite values, or with NaN, +inf and -inf, so a read of them into a result would show.  An entry with
L = 0 gives zero out, out_t and gradients, lse = +inf, and no NaN.  k_lens all equal to Lk gives the bits of the operator
without k_lens.

Float64.  The bars of the dense tests without k_lens hold per entry against float64 over its first L keys: the output cos >=
0.999 and rel-L2 <= 5e-3; the tangent within 1.5x the rel-L2 of a float32 restatement of the kernel's roundings (plus 1e-7),
through ops.dense_attention_jvp, torch.func.jvp and forward_ad; each gradient within 1.5x the rel-L2 of
F.scaled_dot_product_attention's backward with the boolean key-padding mask."""
import math

import pytest
import torch
import torch.autograd.forward_ad as fwAD
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
D = 128
SM = D ** -0.5
F64 = torch.float64
BF16, FP16 = torch.bfloat16, torch.float16
DTYPES = [pytest.param(BF16, id="bf16"), pytest.param(FP16, id="fp16")]
COS, REL = 0.999, 5e-3
POISON = 2.0e4        # finite in both 16-bit types; far larger than any score or value the inputs produce

# (b, h, lq, lk, key lengths): lengths 0, 1, the 64- and 128-key tile boundaries, lk - 1 and lk, ragged lq and lk
CASES = [
    (3, 2, 200, 300, (0, 128, 299)),
    (3, 3, 77, 300, (1, 64, 300)),
    (1, 2, 129, 77, (50,)),
    (3, 1, 1000, 226, (226, 77, 129)),
    (3, 2, 1, 513, (65, 512, 127)),
]
CASE_IDS = ["b{}h{}-{}x{}-{}".format(b, h, lq, lk, "-".join(map(str, ls))) for b, h, lq, lk, ls in CASES]


@pytest.fixture(scope="module")
def cuda():
    from turbodiffusion_b200 import _build, _lib
    _build.build()
    _lib.lib()
    assert torch.cuda.is_available()


def _inputs(b, lq, lk, h, dtype, lens, seed=0, nonfinite=False):
    """q, k, v, q_t, k_t, v_t, d_out on the GPU; key rows >= lens[i] of k, v, k_t, v_t hold +-POISON, or (nonfinite) a mix
    of NaN, +inf and -inf"""
    g = torch.Generator().manual_seed(seed)
    shapes = [(b, lq, h, D), (b, lk, h, D), (b, lk, h, D)] * 2 + [(b, lq, h, D)]
    ts = [torch.randn(*s, generator=g) for s in shapes]
    for i, n in enumerate(lens):
        for t in (ts[1], ts[2], ts[4], ts[5]):
            x = torch.randn(t[i, n:].shape, generator=g)
            bad = torch.where(x.abs() < 0.5, float("nan"), float("inf") * torch.sign(x))
            t[i, n:] = bad if nonfinite else POISON * torch.sign(x)
    return [t.to(dtype).cuda() for t in ts]


def _fwd_lse(q, k, v, k_lens=None):
    """(out, lse) of tdb200_attn_dense_fwd_lse[_kl]"""
    from turbodiffusion_b200._lib import DTYPE_TAG, check, lib, ptr, stream_ptr
    b, lq, h, d = q.shape
    out, lse = torch.empty_like(q), torch.empty(b, h, lq, dtype=torch.float32, device=q.device)
    if k_lens is None:
        check(lib().tdb200_attn_dense_fwd_lse(ptr(q), ptr(k), ptr(v), DTYPE_TAG[q.dtype], ptr(out), ptr(lse), b, lq, k.shape[1], h, d,
                                              SM, stream_ptr(q.device)), "attn_dense_fwd_lse")
    else:
        check(lib().tdb200_attn_dense_fwd_lse_kl(ptr(q), ptr(k), ptr(v), DTYPE_TAG[q.dtype], ptr(out), ptr(lse), b, lq, k.shape[1],
                                                 ptr(k_lens), h, d, SM, stream_ptr(q.device)), "attn_dense_fwd_lse_kl")
    return out, lse


def _jvp_lse(q, k, v, q_t, k_t, v_t, k_lens=None):
    """(out, out_t, lse) of tdb200_attn_dense_jvp_lse[_kl]"""
    from turbodiffusion_b200._lib import DTYPE_TAG, check, lib, ptr, stream_ptr
    b, lq, h, d = q.shape
    out, out_t = torch.empty_like(q), torch.empty_like(q)
    lse = torch.empty(b, h, lq, dtype=torch.float32, device=q.device)
    args = [ptr(t) for t in (q, k, v, q_t, k_t, v_t)] + [DTYPE_TAG[q.dtype], ptr(out), ptr(out_t), ptr(lse), b, lq, k.shape[1]]
    if k_lens is None:
        check(lib().tdb200_attn_dense_jvp_lse(*args, h, d, SM, stream_ptr(q.device)), "attn_dense_jvp_lse")
    else:
        check(lib().tdb200_attn_dense_jvp_lse_kl(*args, ptr(k_lens), h, d, SM, stream_ptr(q.device)), "attn_dense_jvp_lse_kl")
    return out, out_t, lse


def _everything(q, k, v, q_t, k_t, v_t, d_out, k_lens=None):
    """Every output of the family for one set of inputs: a dict of name -> tensor"""
    from turbodiffusion_b200 import ops
    kw = {} if k_lens is None else {"k_lens": k_lens}
    r = {}
    r["out"] = ops.dense_attention(q, k, v, **kw)
    r["out_lse"], r["lse"] = _fwd_lse(q, k, v, k_lens)
    r["jvp_out"], r["jvp_out_t"] = ops.dense_attention_jvp(q, k, v, q_t, k_t, v_t, **kw)
    r["jvp_lse_out"], r["jvp_lse_out_t"], r["jvp_lse"] = _jvp_lse(q, k, v, q_t, k_t, v_t, k_lens)
    _, r["func_out_t"] = torch.func.jvp(lambda a, b_, c: ops.dense_attention(a, b_, c, **kw), (q, k, v), (q_t, k_t, v_t))
    with fwAD.dual_level():
        o = ops.dense_attention(fwAD.make_dual(q, q_t), fwAD.make_dual(k, k_t), fwAD.make_dual(v, v_t), **kw)
        r["ad_out_t"] = fwAD.unpack_dual(o).tangent.clone()
    leaves = [t.detach().clone().requires_grad_() for t in (q, k, v)]
    out = ops.dense_attention(*leaves, **kw)
    r["train_out"] = out.detach()
    r["dq"], r["dk"], r["dv"] = torch.autograd.grad(out, leaves, d_out)
    leaves = [t.detach().clone().requires_grad_() for t in (q, k, v)]
    out, _ = ops.dense_attention_jvp(*leaves, q_t, k_t, v_t, **kw)
    r["jvp_dq"], r["jvp_dk"], r["jvp_dv"] = torch.autograd.grad(out, leaves, d_out)
    return r


KEY_ROWS = ("dk", "dv", "jvp_dk", "jvp_dv")     # outputs indexed by key rows; every other output by query rows (lse: [b, h, lq])


def _bits_equal(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int16 if a.element_size() == 2 else torch.int32),
                                              b.contiguous().view(torch.int16 if b.element_size() == 2 else torch.int32))


def _check_against_trimmed(ins, lens, what):
    q, k, v, q_t, k_t, v_t, d_out = ins
    lk = k.shape[1]
    got = _everything(*ins, k_lens=torch.tensor(lens, dtype=torch.int32, device="cuda"))
    for name, t in got.items():
        assert not torch.isnan(t).any(), (what, name)
    for i, n in enumerate(lens):
        if n == 0:
            for name, t in got.items():
                if name in ("lse", "jvp_lse"):
                    assert torch.isinf(t[i]).all() and (t[i] > 0).all(), (what, i, name)
                else:
                    assert (t[i] == 0).all(), (what, i, name)
            continue
        sl = [t[i:i + 1].contiguous() for t in (q,)] + [t[i:i + 1, :n].contiguous() for t in (k, v)] + \
             [q_t[i:i + 1].contiguous()] + [t[i:i + 1, :n].contiguous() for t in (k_t, v_t)] + [d_out[i:i + 1].contiguous()]
        want = _everything(*sl)
        for name, t in got.items():
            mine = t[i:i + 1, :n] if name in KEY_ROWS else t[i:i + 1]
            assert _bits_equal(mine, want[name]), (what, i, n, name, (mine.float() - want[name].float()).abs().max().item())
            if name in KEY_ROWS and n < lk:
                assert (t[i, n:] == 0).all(), (what, i, n, name)
    return got


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("b,h,lq,lk,lens", [pytest.param(*c, id=i) for c, i in zip(CASES, CASE_IDS)])
def test_each_entry_gets_the_bits_of_its_trimmed_call(cuda, b, h, lq, lk, lens, dtype):
    _check_against_trimmed(_inputs(b, lq, lk, h, dtype, lens), lens, f"({b}, {h}, {lq}, {lk}, {lens}) {dtype}")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("b,h,lq,lk,lens", [pytest.param(*c, id=i) for c, i in zip(CASES, CASE_IDS)])
def test_nan_and_inf_past_the_lengths_never_reach_a_result(cuda, b, h, lq, lk, lens, dtype):
    """padding left as whatever an uninitialised buffer holds: the straddling tile's rows past L are zeroed on chip"""
    _check_against_trimmed(_inputs(b, lq, lk, h, dtype, lens, nonfinite=True), lens, f"({b}, {h}, {lq}, {lk}, {lens}) {dtype} nan/inf")


@pytest.mark.parametrize("dtype", DTYPES)
def test_full_lengths_give_the_bits_of_the_operator_without_them(cuda, dtype):
    b, h, lq, lk = 3, 2, 200, 300
    ins = _inputs(b, lq, lk, h, dtype, (lk,) * b)
    got = _everything(*ins, k_lens=torch.full((b,), lk, dtype=torch.int32, device="cuda"))
    want = _everything(*ins)
    for name in want:
        assert _bits_equal(got[name], want[name]), name


@pytest.mark.parametrize("dtype", DTYPES)
def test_lengths_outside_the_keys_are_clamped_on_the_device(cuda, dtype):
    """CUDA lengths are not checked on the host: -5 acts as 0 and lk + 100 as lk"""
    b, h, lq, lk = 2, 2, 130, 200
    ins = _inputs(b, lq, lk, h, dtype, (0, lk))
    got = _everything(*ins, k_lens=torch.tensor([-5, lk + 100], dtype=torch.int32, device="cuda"))
    want = _everything(*ins, k_lens=torch.tensor([0, lk], dtype=torch.int32, device="cuda"))
    for name in want:
        assert _bits_equal(got[name], want[name]), name
    # ops: int64 lengths outside int32 are clamped before they are narrowed, so 2^32 + 5 acts as lk, not as 5 (the outputs of
    # the C entry points called directly, which take int32 lengths, are left out)
    wide = _everything(*ins, k_lens=torch.tensor([-(1 << 40), (1 << 32) + 5], dtype=torch.int64, device="cuda"))
    for name in want:
        if name not in ("out_lse", "lse", "jvp_lse_out", "jvp_lse_out_t", "jvp_lse"):
            assert _bits_equal(wide[name], want[name]), name


def test_a_mask_on_either_device_gives_the_bits_of_its_lengths(cuda):
    from turbodiffusion_b200 import ops
    b, h, lq, lk, lens = 3, 2, 100, 150, (150, 3, 0)
    q, k, v, *_ = _inputs(b, lq, lk, h, BF16, lens)
    mask = torch.arange(lk)[None, :] < torch.tensor(lens)[:, None]
    want = ops.dense_attention(q, k, v, k_lens=torch.tensor(lens))
    for m in (mask, mask.cuda()):
        assert _bits_equal(ops.dense_attention(q, k, v, k_lens=m), want)
    with pytest.raises(ValueError, match="prefix"):
        ops.dense_attention(q, k, v, k_lens=(~mask).cuda())


# ------------------------------------------------------------------------------------------------------------ float64
def _attn(q, k, v, sm_scale=SM):
    s = torch.einsum("bqhd,bkhd->bhqk", q, k) * sm_scale
    return torch.einsum("bhqk,bkhd->bqhd", torch.softmax(s, -1), v)


def _rel(got, want):
    a, b = got.to(F64).flatten(), want.to(F64).flatten()
    return ((a - b).norm() / b.norm().clamp_min(1e-300)).item()


def _cos(got, want):
    a, b = got.to(F64).flatten(), want.to(F64).flatten()
    return (torch.dot(a, b) / (a.norm() * b.norm()).clamp_min(1e-300)).item()


def _restated(q, k, v, q_t, k_t, v_t, sm_scale=SM):
    """The kernel's tangent arithmetic in float32 (tests/test_gpu_dense_attention_jvp.py's restatement)"""
    f = [t.float() for t in (q, k, v, q_t, k_t, v_t)]
    s = torch.einsum("bqhd,bkhd->bhqk", f[0], f[1]) * sm_scale
    st = (torch.einsum("bqhd,bkhd->bhqk", f[3], f[1]) + torch.einsum("bqhd,bkhd->bhqk", f[0], f[4])) * sm_scale
    p = torch.exp(s - s.amax(-1, keepdim=True))
    pst = p * st
    l, mu = p.sum(-1), pst.sum(-1)
    p_r, pst_r = (t.to(q.dtype).float() for t in (p, pst))
    o = torch.einsum("bhqk,bkhd->bqhd", p_r, f[2])
    a = torch.einsum("bhqk,bkhd->bqhd", pst_r, f[2]) + torch.einsum("bhqk,bkhd->bqhd", p_r, f[5])
    l, mu = l.transpose(1, 2)[..., None], mu.transpose(1, 2)[..., None]
    return ((a - mu / l * o) / l).to(q.dtype)


def _sdpa_masked_grads(q, k, v, d_out, lens):
    """F.scaled_dot_product_attention's gradients in q's dtype with the boolean key-padding mask (entries with keys only)"""
    leaves = [t.detach().clone().requires_grad_() for t in (q, k, v)]
    mask = (torch.arange(k.shape[1], device=q.device)[None, :] < torch.tensor(lens, device=q.device)[:, None])[:, None, None, :]
    out = F.scaled_dot_product_attention(*(t.transpose(1, 2) for t in leaves), attn_mask=mask, scale=SM).transpose(1, 2)
    out.backward(d_out)
    return [t.grad for t in leaves]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("b,h,lq,lk,lens", [pytest.param(*c, id=i) for c, i in zip(CASES, CASE_IDS)])
def test_each_entry_against_float64_over_its_keys(cuda, b, h, lq, lk, lens, dtype):
    ins = _inputs(b, lq, lk, h, dtype, lens, seed=1)
    q, k, v, q_t, k_t, v_t, d_out = ins
    got = _everything(*ins, k_lens=torch.tensor(lens, dtype=torch.int32, device="cuda"))
    nz = [i for i, n in enumerate(lens) if n > 0]
    sdpa = _sdpa_masked_grads(*(t[nz] for t in (q, k, v, d_out)), [lens[i] for i in nz])
    for j, i in enumerate(nz):
        n = lens[i]
        one = [t[i:i + 1] for t in (q,)] + [t[i:i + 1, :n] for t in (k, v)] + [q_t[i:i + 1]] + \
              [t[i:i + 1, :n] for t in (k_t, v_t)]
        what = f"({b}, {h}, {lq}, {lk}) {dtype} entry {i} L={n}"
        prim, tan = (tuple(t.to(F64) for t in ts) for ts in (one[:3], one[3:]))
        out64, out_t64 = torch.func.jvp(_attn, prim, tan)
        for name in ("out", "jvp_out", "train_out"):
            o = got[name][i:i + 1]
            assert _cos(o, out64) >= COS and _rel(o, out64) <= REL, (what, name, _cos(o, out64), _rel(o, out64))
        ref = _rel(_restated(*one), out_t64)
        for name in ("jvp_out_t", "func_out_t", "ad_out_t"):
            e = _rel(got[name][i:i + 1], out_t64)
            assert e <= 1.5 * ref + 1e-7, (what, name, e, ref)
        leaves = [t.to(F64).requires_grad_() for t in one[:3]]
        _attn(*leaves).backward(d_out[i:i + 1].to(F64))
        for name, want, lib, rows in (("dq", leaves[0].grad, sdpa[0][j:j + 1], None), ("dk", leaves[1].grad, sdpa[1][j:j + 1], n),
                                      ("dv", leaves[2].grad, sdpa[2][j:j + 1], n)):
            for pre in ("", "jvp_"):
                mine = got[pre + name][i:i + 1] if rows is None else got[pre + name][i:i + 1, :rows]
                lib_ = lib if rows is None else lib[:, :rows]
                if n == 1 and name != "dv":        # one key: softmax is constant, dq and dk are exactly zero
                    assert want.abs().max().item() == 0.0 and mine.double().pow(2).mean().sqrt().item() <= 1e-3, (what, name)
                    continue
                e, es = _rel(mine, want), _rel(lib_, want)
                assert e <= 1.5 * es, (what, pre + name, e, es)


# ------------------------------------------------------------------------------------------------------------ capture, size
def test_the_masked_backward_captures_in_a_cuda_graph(cuda):
    from turbodiffusion_b200 import ops
    b, h, lq, lk, lens = 3, 2, 200, 300, (0, 128, 299)
    q, k, v, _, _, _, d_out = _inputs(b, lq, lk, h, BF16, lens)
    k_lens = torch.tensor(lens, dtype=torch.int32, device="cuda")
    leaves = [t.detach().clone().requires_grad_() for t in (q, k, v)]

    def step():
        return torch.autograd.grad(ops.dense_attention(*leaves, k_lens=k_lens), leaves, d_out)

    eager = [t.clone() for t in step()]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static = step()
    for t in static:
        t.fill_(float("nan"))
    graph.replay()
    torch.cuda.synchronize()
    for a, e in zip(static, eager):
        assert _bits_equal(a, e)


def test_shape_a_cross_attention_at_batch_2(cuda):
    """Wan shape A's cross-attention, 32760 queries x 12 heads over 512 text keys, two prompts of 512 and 226 tokens"""
    lens = (512, 226)
    _check_against_trimmed(_inputs(2, 32760, 512, 12, BF16, lens), lens, "shape A")
