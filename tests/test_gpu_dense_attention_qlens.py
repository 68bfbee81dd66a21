"""GPU checks of the dense attention operators with per-sample query lengths (q_lens: tdb200_attn_dense_{fwd,fwd_lse,jvp,jvp_lse,
tangent,bwd}_vl behind ops.dense_attention / ops.dense_attention_jvp, with or without key lengths).

Bit identity with trimming.  For every batch entry i with Lq_i = q_lens[i] > 0, the rows < Lq_i of out, lse, out_t (from the
fused JVP and from the forward-AD rule's tangent kernel) and dq, and dk and dv (rows < Lk_i when k_lens is given), are
byte-identical to the operator without lengths called on entry i alone with q, q_t and d_out cut to Lq_i rows and k, v, k_t, v_t
cut to Lk_i.  Rows >= Lq_i of out, out_t and dq are exactly zero and of lse +inf; rows >= Lk_i of dk and dv are zero; an entry
with Lq_i = 0 has zero dk and dv.  The padded query rows of q, q_t and d_out (and the padded key rows of k, v, k_t, v_t) are
filled with large finite values, or with NaN, +inf and -inf; the tangent and backward entry points are also called directly
with those rows of out and lse filled with NaN and inf.  None of it reaches a result.

The k_lens-only call on the same NaN-padded batch (the padded query rows computed, which is all the parent commit's entry points
can do) is run beside it and shown to put NaN into dk and dv of valid keys: the failure q_lens removes.  Those entry points are
unchanged by q_lens, so this is the parent's behaviour.

Every path through the operators (no-grad, training, torch.func.jvp, forward_ad) gives the bits of the direct calls, lengths
may be CPU or CUDA tensors or prefix masks, and the masked forward and backward capture in a CUDA graph and replay with new
lengths written in place."""
import pytest
import torch
import torch.autograd.forward_ad as fwAD

pytestmark = pytest.mark.gpu
D = 128
SM = D ** -0.5
BF16, FP16 = torch.bfloat16, torch.float16
DTYPES = [pytest.param(BF16, id="bf16"), pytest.param(FP16, id="fp16")]
POISON = 2.0e4        # finite in both 16-bit types; far larger than any score or value the inputs produce

# (b, h, lq, lk, query lengths, key lengths or None): query lengths 0, 1, 63, 64, 127, 128, 129, lq - 1 and lq mixed in one
# batch, with and without key lengths; "self" marks self-attention with q_lens = k_lens (the same tensor)
CASES = [
    (5, 2, 300, 200, (0, 1, 63, 64, 299), None),
    (4, 2, 300, 257, (127, 128, 129, 300), (257, 1, 130, 64)),
    (3, 2, 129, 77, (128, 129, 0), (50, 77, 3)),
    (3, 2, 400, 400, (400, 129, 64), "self"),
    (2, 1, 1000, 1000, (999, 1), "self"),
]
CASE_IDS = ["b{}h{}-{}x{}-q{}-k{}".format(b, h, lq, lk, "-".join(map(str, ql)),
                                         kl if isinstance(kl, str) or kl is None else "-".join(map(str, kl)))
            for b, h, lq, lk, ql, kl in CASES]


@pytest.fixture(scope="module")
def cuda():
    from turbodiffusion_b200 import _build, _lib
    _build.build()
    _lib.lib()
    assert torch.cuda.is_available()


def _key_lengths(lk, ql, kl):
    return tuple(ql) if kl == "self" else (lk,) * len(ql) if kl is None else tuple(kl)


def _inputs(b, lq, lk, h, dtype, q_lens, k_lens, seed=0, nonfinite=False):
    """q, k, v, q_t, k_t, v_t, d_out on the GPU; query rows >= q_lens[i] of q, q_t, d_out and key rows >= k_lens[i] of k, v, k_t,
    v_t hold +-POISON, or (nonfinite) a mix of NaN, +inf and -inf"""
    g = torch.Generator().manual_seed(seed)
    shapes = [(b, lq, h, D), (b, lk, h, D), (b, lk, h, D)] * 2 + [(b, lq, h, D)]
    ts = [torch.randn(*s, generator=g) for s in shapes]
    for i in range(b):
        for t, n in [(ts[j], q_lens[i]) for j in (0, 3, 6)] + [(ts[j], k_lens[i]) for j in (1, 2, 4, 5)]:
            x = torch.randn(t[i, n:].shape, generator=g)
            bad = torch.where(x.abs() < 0.5, float("nan"), float("inf") * torch.sign(x))
            t[i, n:] = bad if nonfinite else POISON * torch.sign(x)
    return [t.to(dtype).cuda() for t in ts]


def _c():
    from turbodiffusion_b200 import _lib
    return _lib


def _fwd_lse(q, k, v, ql=None, kl=None):
    """(out, lse) of tdb200_attn_dense_fwd_lse or, with ql and kl, tdb200_attn_dense_fwd_lse_vl"""
    L = _c()
    b, lq, h, d = q.shape
    out, lse = torch.empty_like(q), torch.empty(b, h, lq, dtype=torch.float32, device=q.device)
    args = [L.ptr(q), L.ptr(k), L.ptr(v), L.DTYPE_TAG[q.dtype], L.ptr(out), L.ptr(lse), b, lq, k.shape[1]]
    if ql is None:
        L.check(L.lib().tdb200_attn_dense_fwd_lse(*args, h, d, SM, L.stream_ptr(q.device)), "attn_dense_fwd_lse")
    else:
        L.check(L.lib().tdb200_attn_dense_fwd_lse_vl(*args, L.ptr(ql), L.ptr(kl), h, d, SM, L.stream_ptr(q.device)),
                "attn_dense_fwd_lse_vl")
    return out, lse


def _jvp_lse(q, k, v, q_t, k_t, v_t, ql=None, kl=None):
    """(out, out_t, lse) of tdb200_attn_dense_jvp_lse[_vl]"""
    L = _c()
    b, lq, h, d = q.shape
    out, out_t = torch.empty_like(q), torch.empty_like(q)
    lse = torch.empty(b, h, lq, dtype=torch.float32, device=q.device)
    args = [L.ptr(t) for t in (q, k, v, q_t, k_t, v_t)] + [L.DTYPE_TAG[q.dtype], L.ptr(out), L.ptr(out_t), L.ptr(lse), b, lq,
                                                            k.shape[1]]
    if ql is None:
        L.check(L.lib().tdb200_attn_dense_jvp_lse(*args, h, d, SM, L.stream_ptr(q.device)), "attn_dense_jvp_lse")
    else:
        L.check(L.lib().tdb200_attn_dense_jvp_lse_vl(*args, L.ptr(ql), L.ptr(kl), h, d, SM, L.stream_ptr(q.device)),
                "attn_dense_jvp_lse_vl")
    return out, out_t, lse


def _tangent_vl(q, k, v, q_t, k_t, v_t, out, lse, ql, kl):
    L = _c()
    b, lq, h, d = q.shape
    out_t = torch.empty_like(q)
    L.check(L.lib().tdb200_attn_dense_tangent_vl(*(L.ptr(t) for t in (q, k, v, q_t, k_t, v_t, out, lse)), L.DTYPE_TAG[q.dtype],
                                                 L.ptr(out_t), b, lq, k.shape[1], L.ptr(ql), L.ptr(kl), h, d, SM,
                                                 L.stream_ptr(q.device)), "attn_dense_tangent_vl")
    return out_t


def _bwd(q, k, v, out, d_out, lse, ql=None, kl=None, entry="vl"):
    """(dq, dk, dv) of tdb200_attn_dense_bwd_vl, or (entry "kl", ql ignored) tdb200_attn_dense_bwd_kl"""
    L = _c()
    b, lq, h, d = q.shape
    dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
    nbytes = L.lib().tdb200_attn_dense_bwd_workspace_bytes(b, h, lq)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=q.device)
    args = [L.ptr(t) for t in (q, k, v, out, d_out, lse)] + [L.DTYPE_TAG[q.dtype], L.ptr(dq), L.ptr(dk), L.ptr(dv), L.ptr(ws),
                                                             nbytes, b, lq, k.shape[1]]
    if entry == "kl":
        L.check(L.lib().tdb200_attn_dense_bwd_kl(*args, L.ptr(kl), h, d, SM, L.stream_ptr(q.device)), "attn_dense_bwd_kl")
    else:
        L.check(L.lib().tdb200_attn_dense_bwd_vl(*args, L.ptr(ql), L.ptr(kl), h, d, SM, L.stream_ptr(q.device)),
                "attn_dense_bwd_vl")
    return dq, dk, dv


def _everything(q, k, v, q_t, k_t, v_t, d_out, q_lens=None, k_lens=None):
    """Every output of the family for one set of inputs: a dict of name -> tensor.  With q_lens, the operators get q_lens and
    k_lens (which may be None: the Python layer then fills it with lk) and the direct calls the _vl entry points."""
    from turbodiffusion_b200 import ops
    kw = {} if q_lens is None else {"q_lens": q_lens, "k_lens": k_lens}
    ql = None if q_lens is None else q_lens
    kl = None if q_lens is None else (k_lens if k_lens is not None else
                                      torch.full((q.shape[0],), k.shape[1], dtype=torch.int32, device=q.device))
    r = {}
    r["out"] = ops.dense_attention(q, k, v, **kw)
    r["out_lse"], r["lse"] = _fwd_lse(q, k, v, ql, kl)
    r["jvp_out"], r["jvp_out_t"] = ops.dense_attention_jvp(q, k, v, q_t, k_t, v_t, **kw)
    r["jvp_lse_out"], r["jvp_lse_out_t"], r["jvp_lse"] = _jvp_lse(q, k, v, q_t, k_t, v_t, ql, kl)
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
    if ql is not None:   # the direct backward and tangent calls, on the lse forward's out and lse
        out, lse = r["out_lse"], r["lse"]
        r["bwd_dq"], r["bwd_dk"], r["bwd_dv"] = _bwd(q, k, v, out, d_out, lse, ql, kl)
        r["tangent_out_t"] = _tangent_vl(q, k, v, q_t, k_t, v_t, out, lse, ql, kl)
    return r


KEY_ROWS = ("dk", "dv", "jvp_dk", "jvp_dv", "bwd_dk", "bwd_dv")   # indexed by key rows; every other output by query rows
LSE = ("lse", "jvp_lse")                                          # [b, h, lq]
TRIMMED_NAME = {"bwd_dq": "dq", "bwd_dk": "dk", "bwd_dv": "dv", "tangent_out_t": "ad_out_t"}


def _bits_equal(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int16 if a.element_size() == 2 else torch.int32),
                                              b.contiguous().view(torch.int16 if b.element_size() == 2 else torch.int32))


def _lens_args(q_lens, kl_spec, lk):
    ql = torch.tensor(q_lens, dtype=torch.int32, device="cuda")
    if kl_spec == "self":
        return ql, ql
    return ql, (None if kl_spec is None else torch.tensor(kl_spec, dtype=torch.int32, device="cuda"))


def _check_against_trimmed(ins, q_lens, kl_spec, what):
    q, k, v, q_t, k_t, v_t, d_out = ins
    lq, lk = q.shape[1], k.shape[1]
    k_lens = _key_lengths(lk, q_lens, kl_spec)
    ql, kl = _lens_args(q_lens, kl_spec, lk)
    got = _everything(*ins, q_lens=ql, k_lens=kl)
    for name, t in got.items():
        assert not torch.isnan(t).any(), (what, name)
    for i, (n, m) in enumerate(zip(q_lens, k_lens)):
        for name, t in got.items():   # the padded rows
            if name in KEY_ROWS:
                assert (t[i, m:] == 0).all(), (what, i, name)
                if n == 0:
                    assert (t[i] == 0).all(), (what, i, name)
            elif name in LSE:
                assert torch.isinf(t[i, :, n:]).all() and (t[i, :, n:] > 0).all(), (what, i, name)
            else:
                assert (t[i, n:] == 0).all(), (what, i, name)
        if n == 0:
            continue
        sl = [q[i:i + 1, :n].contiguous()] + [t[i:i + 1, :m].contiguous() for t in (k, v)] + \
             [q_t[i:i + 1, :n].contiguous()] + [t[i:i + 1, :m].contiguous() for t in (k_t, v_t)] + [d_out[i:i + 1, :n].contiguous()]
        want = _everything(*sl)
        for name, t in got.items():
            mine = t[i:i + 1, :m] if name in KEY_ROWS else t[i:i + 1, :, :n] if name in LSE else t[i:i + 1, :n]
            ref = want[TRIMMED_NAME.get(name, name)]
            assert _bits_equal(mine, ref), (what, i, n, m, name, (mine.float() - ref.float()).abs().max().item())
    return got


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("b,h,lq,lk,q_lens,k_lens", [pytest.param(*c, id=i) for c, i in zip(CASES, CASE_IDS)])
def test_each_entry_gets_the_bits_of_its_trimmed_call(cuda, b, h, lq, lk, q_lens, k_lens, dtype):
    ins = _inputs(b, lq, lk, h, dtype, q_lens, _key_lengths(lk, q_lens, k_lens))
    _check_against_trimmed(ins, q_lens, k_lens, f"({b}, {h}, {lq}, {lk}, {q_lens}, {k_lens}) {dtype}")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("b,h,lq,lk,q_lens,k_lens", [pytest.param(*c, id=i) for c, i in zip(CASES, CASE_IDS)])
def test_nan_and_inf_past_the_lengths_never_reach_a_result(cuda, b, h, lq, lk, q_lens, k_lens, dtype):
    """padding left as whatever an uninitialised buffer holds: the dK/dV kernel zeroes the straddling block's Q and dO rows"""
    ins = _inputs(b, lq, lk, h, dtype, q_lens, _key_lengths(lk, q_lens, k_lens), nonfinite=True)
    _check_against_trimmed(ins, q_lens, k_lens, f"({b}, {h}, {lq}, {lk}, {q_lens}, {k_lens}) {dtype} nan/inf")


@pytest.mark.parametrize("dtype", DTYPES)
def test_nan_in_the_padded_rows_of_out_and_lse_never_reaches_a_result(cuda, dtype):
    """the tangent and the backward read out (and lse) only in rows below q_lens: poisoned there, their bits do not move"""
    b, h, lq, lk, q_lens = 3, 2, 300, 257, (129, 0, 300)
    ins = _inputs(b, lq, lk, h, dtype, q_lens, (lk,) * b, nonfinite=True)
    q, k, v, q_t, k_t, v_t, d_out = ins
    ql = torch.tensor(q_lens, dtype=torch.int32, device="cuda")
    kl = torch.full((b,), lk, dtype=torch.int32, device="cuda")
    out, lse = _fwd_lse(q, k, v, ql, kl)
    want = _bwd(q, k, v, out, d_out, lse, ql, kl) + (_tangent_vl(q, k, v, q_t, k_t, v_t, out, lse, ql, kl),)
    bad_out, bad_lse = out.clone(), lse.clone()
    for i, n in enumerate(q_lens):
        bad_out[i, n:] = float("nan")
        bad_out[i, n::3] = float("inf")
        bad_lse[i, :, n:] = float("nan")
        bad_lse[i, :, n::2] = -float("inf")
    got = _bwd(q, k, v, bad_out, d_out, bad_lse, ql, kl) + (_tangent_vl(q, k, v, q_t, k_t, v_t, bad_out, bad_lse, ql, kl),)
    for name, a, e in zip(("dq", "dk", "dv", "out_t"), got, want):
        assert _bits_equal(a, e), name


def test_key_lengths_alone_let_a_nan_query_pad_reach_dk_and_dv(cuda):
    """The failure query lengths remove.  With k_lens alone the padded query rows are computed; NaN or inf in them reaches dk
    and dv of valid keys through 0 * NaN in the dK/dV kernel's sums over query rows.  tdb200_attn_dense_bwd_kl is unchanged by
    q_lens, so this is what the parent commit computes; with q_lens the same batch gives finite dk and dv."""
    b, h, lq, lk, q_lens = 2, 2, 300, 200, (150, 300)
    q, k, v, q_t, k_t, v_t, d_out = _inputs(b, lq, lk, h, BF16, q_lens, (lk,) * b, nonfinite=True)
    kl = torch.full((b,), lk, dtype=torch.int32, device="cuda")
    ql = torch.tensor(q_lens, dtype=torch.int32, device="cuda")
    L = _c()
    out, lse = torch.empty_like(q), torch.empty(b, h, lq, dtype=torch.float32, device="cuda")
    L.check(L.lib().tdb200_attn_dense_fwd_lse_kl(L.ptr(q), L.ptr(k), L.ptr(v), L.DTYPE_TAG[q.dtype], L.ptr(out), L.ptr(lse), b, lq,
                                                 lk, L.ptr(kl), h, D, SM, L.stream_ptr(q.device)), "attn_dense_fwd_lse_kl")
    _, dk, dv = _bwd(q, k, v, out, d_out, lse, kl=kl, entry="kl")
    assert torch.isnan(dk[0]).any() and torch.isnan(dv[0]).any()
    out, lse = _fwd_lse(q, k, v, ql, kl)
    _, dk, dv = _bwd(q, k, v, out, d_out, lse, ql, kl)
    assert torch.isfinite(dk).all() and torch.isfinite(dv).all()


@pytest.mark.parametrize("dtype", DTYPES)
def test_full_lengths_give_the_bits_of_the_operator_without_them(cuda, dtype):
    b, h, lq, lk = 3, 2, 200, 300
    ins = _inputs(b, lq, lk, h, dtype, (lq,) * b, (lk,) * b)
    got = _everything(*ins, q_lens=torch.full((b,), lq, dtype=torch.int32, device="cuda"))
    want = _everything(*ins)
    for name in want:
        assert _bits_equal(got[name], want[name]), name


@pytest.mark.parametrize("dtype", DTYPES)
def test_lengths_outside_the_queries_are_clamped_on_the_device(cuda, dtype):
    """CUDA lengths are not checked on the host: -5 acts as 0 and lq + 100 as lq, as do int64 lengths beyond int32"""
    b, h, lq, lk = 2, 2, 130, 200
    ins = _inputs(b, lq, lk, h, dtype, (0, lq), (lk, lk))
    want = _everything(*ins, q_lens=torch.tensor([0, lq], dtype=torch.int32, device="cuda"))
    got = _everything(*ins, q_lens=torch.tensor([-5, lq + 100], dtype=torch.int32, device="cuda"))
    for name in want:
        assert _bits_equal(got[name], want[name]), name
    from turbodiffusion_b200 import ops
    q, k, v, *_ = ins
    wide = ops.dense_attention(q, k, v, q_lens=torch.tensor([-(1 << 40), (1 << 32) + 5], dtype=torch.int64, device="cuda"))
    assert _bits_equal(wide, want["out"])


def test_masks_and_lengths_on_either_device_give_the_same_bits(cuda):
    from turbodiffusion_b200 import ops
    b, h, lq, lk, q_lens = 3, 2, 150, 150, (150, 3, 0)
    q, k, v, q_t, k_t, v_t, _ = _inputs(b, lq, lk, h, BF16, q_lens, q_lens)
    mask = torch.arange(lq)[None, :] < torch.tensor(q_lens)[:, None]
    want = ops.dense_attention(q, k, v, q_lens=torch.tensor(q_lens, dtype=torch.int32, device="cuda"), k_lens=mask.cuda())
    want_t = ops.dense_attention_jvp(q, k, v, q_t, k_t, v_t, q_lens=torch.tensor(q_lens), k_lens=torch.tensor(q_lens))
    for m in (mask, mask.cuda(), torch.tensor(q_lens), torch.tensor(q_lens).cuda()):
        assert _bits_equal(ops.dense_attention(q, k, v, q_lens=m, k_lens=m), want)
        for a, e in zip(ops.dense_attention_jvp(q, k, v, q_t, k_t, v_t, q_lens=m, k_lens=m), want_t):
            assert _bits_equal(a, e)
    with pytest.raises(ValueError, match="prefix"):
        ops.dense_attention(q, k, v, q_lens=(~mask).cuda())


# ------------------------------------------------------------------------------------------------------------ capture, size
def test_the_masked_forward_and_backward_capture_and_replay_with_new_lengths(cuda):
    from turbodiffusion_b200 import ops
    b, h, lq, lk = 3, 2, 300, 300
    first, second = (0, 129, 300), (300, 1, 64)
    q, k, v, _, _, _, d_out = _inputs(b, lq, lk, h, BF16, (lq,) * b, (lk,) * b)
    lens = torch.tensor(first, dtype=torch.int32, device="cuda")
    leaves = [t.detach().clone().requires_grad_() for t in (q, k, v)]

    def step():
        out = ops.dense_attention(*leaves, q_lens=lens, k_lens=lens)
        return (out.detach(),) + torch.autograd.grad(out, leaves, d_out)

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static = step()
    for new in (first, second):
        lens.copy_(torch.tensor(new, dtype=torch.int32))
        eager = [t.clone() for t in step()]
        for t in static:
            t.fill_(float("nan"))
        graph.replay()
        torch.cuda.synchronize()
        for name, a, e in zip(("out", "dq", "dk", "dv"), static, eager):
            assert _bits_equal(a, e), (new, name)


def test_wan_pair_self_attention(cuda):
    """Two Wan2.1 480p clips of 81 and 49 frames (32760 and 20280 tokens) packed to one L, self-attention (2 of the 12 heads)"""
    lens = (32760, 20280)
    ins = _inputs(2, 32760, 32760, 2, BF16, lens, lens, nonfinite=True)
    _check_against_trimmed(ins, lens, "self", "Wan pair")
