"""CPU checks of the dense attention operators' per-sample query lengths: the six _vl entry points return their codes and a
message naming the entry point before any CUDA call (the _kl twins' checks, plus a null or misaligned q_lens or k_lens; on a
host without a GPU, a check that ran after the first CUDA call could only report a CUDA error), a query-padding mask becomes
lengths and a mask that does not keep a prefix of its row is refused before any library call, and ops.dense_attention /
dense_attention_jvp reach the entry points they reached before when q_lens is None and the _vl twins when it is set, with
k_lens filled with Lk when only query lengths are given (checked with a recording stand-in for the library).  Lengths and
masks on a CUDA device are checked in tests/test_gpu_dense_attention_qlens.py."""
import ctypes

import pytest

INVALID, UNSUPPORTED, WORKSPACE = -1, -2, -5
BF16, FP16 = 0, 1
NULL = ctypes.c_void_p(0)


def _p(v=4096):
    return ctypes.c_void_p(v)          # non-null, 16-byte aligned, never dereferenced: validation runs before any CUDA call


@pytest.fixture(scope="module")
def lib():
    from turbodiffusion_b200 import _build, _lib
    _build.build()
    return _lib.lib()


FWD_PTRS = ("q", "k", "v", "out", "q_lens", "k_lens")
FWD_LSE_PTRS = ("q", "k", "v", "out", "lse", "q_lens", "k_lens")
JVP_PTRS = ("q", "k", "v", "q_t", "k_t", "v_t", "out", "out_t", "q_lens", "k_lens")
JVP_LSE_PTRS = ("q", "k", "v", "q_t", "k_t", "v_t", "out", "out_t", "lse", "q_lens", "k_lens")
TANGENT_PTRS = ("q", "k", "v", "q_t", "k_t", "v_t", "out", "lse", "out_t", "q_lens", "k_lens")
BWD_PTRS = ("q", "k", "v", "out", "d_out", "lse", "dq", "dk", "dv", "workspace", "q_lens", "k_lens")
MISALIGNED = {"lse": 4098, "workspace": 4098, "q_lens": 4098, "k_lens": 4098}   # the 4-byte-aligned arrays; 16-bit tensors at 4100


def _fwd(lib, dtype=BF16, b=2, lq=256, lk=77, h=2, d=128, sm_scale=0.088, **ptrs):
    a = {n: ptrs.get(n, _p()) for n in FWD_PTRS}
    return lib.tdb200_attn_dense_fwd_vl(a["q"], a["k"], a["v"], dtype, a["out"], b, lq, lk, a["q_lens"], a["k_lens"], h, d, sm_scale,
                                        None)


def _fwd_lse(lib, dtype=BF16, b=2, lq=256, lk=77, h=2, d=128, sm_scale=0.088, **ptrs):
    a = {n: ptrs.get(n, _p()) for n in FWD_LSE_PTRS}
    return lib.tdb200_attn_dense_fwd_lse_vl(a["q"], a["k"], a["v"], dtype, a["out"], a["lse"], b, lq, lk, a["q_lens"], a["k_lens"],
                                            h, d, sm_scale, None)


def _jvp(lib, dtype=BF16, b=2, lq=256, lk=77, h=2, d=128, sm_scale=0.088, **ptrs):
    a = {n: ptrs.get(n, _p()) for n in JVP_PTRS}
    return lib.tdb200_attn_dense_jvp_vl(a["q"], a["k"], a["v"], a["q_t"], a["k_t"], a["v_t"], dtype, a["out"], a["out_t"], b, lq,
                                        lk, a["q_lens"], a["k_lens"], h, d, sm_scale, None)


def _jvp_lse(lib, dtype=BF16, b=2, lq=256, lk=77, h=2, d=128, sm_scale=0.088, **ptrs):
    a = {n: ptrs.get(n, _p()) for n in JVP_LSE_PTRS}
    return lib.tdb200_attn_dense_jvp_lse_vl(a["q"], a["k"], a["v"], a["q_t"], a["k_t"], a["v_t"], dtype, a["out"], a["out_t"],
                                            a["lse"], b, lq, lk, a["q_lens"], a["k_lens"], h, d, sm_scale, None)


def _tangent(lib, dtype=BF16, b=2, lq=256, lk=77, h=2, d=128, sm_scale=0.088, **ptrs):
    a = {n: ptrs.get(n, _p()) for n in TANGENT_PTRS}
    return lib.tdb200_attn_dense_tangent_vl(a["q"], a["k"], a["v"], a["q_t"], a["k_t"], a["v_t"], a["out"], a["lse"], dtype,
                                            a["out_t"], b, lq, lk, a["q_lens"], a["k_lens"], h, d, sm_scale, None)


def _bwd(lib, dtype=BF16, b=2, lq=256, lk=77, h=2, d=128, sm_scale=0.088, workspace_bytes=1 << 40, **ptrs):
    a = {n: ptrs.get(n, _p()) for n in BWD_PTRS}
    return lib.tdb200_attn_dense_bwd_vl(a["q"], a["k"], a["v"], a["out"], a["d_out"], a["lse"], dtype, a["dq"], a["dk"], a["dv"],
                                        a["workspace"], workspace_bytes, b, lq, lk, a["q_lens"], a["k_lens"], h, d, sm_scale, None)


SHAPE_CASES = [
    ("b = 0", dict(b=0), INVALID, b"shape"),
    ("lq = 0", dict(lq=0), INVALID, b"shape"),
    ("lk < 0", dict(lk=-5), INVALID, b"shape"),
    ("h = 0", dict(h=0), INVALID, b"shape"),
    ("dtype tag", dict(dtype=7), UNSUPPORTED, b"dtype"),
    ("head dim 64", dict(d=64), UNSUPPORTED, b"head dim"),
    ("batch beyond the grid", dict(b=70000), UNSUPPORTED, b"too large"),
    ("lk * h * d of 2^39 elements", dict(lk=1 << 30, h=4), UNSUPPORTED, b"too large"),
    ("lq * h * d of 2^39 elements", dict(lq=1 << 30, h=4), UNSUPPORTED, b"too large"),
]


def _pointer_cases(names):
    return ([(f"null {n}", {n: NULL}, INVALID, b"null") for n in names] +
            [(f"misaligned {n}", {n: _p(MISALIGNED.get(n, 4100))}, INVALID, b"aligned") for n in names])


ENTRIES = [("fwd_vl", _fwd, FWD_PTRS), ("fwd_lse_vl", _fwd_lse, FWD_LSE_PTRS), ("jvp_vl", _jvp, JVP_PTRS),
           ("jvp_lse_vl", _jvp_lse, JVP_LSE_PTRS), ("tangent_vl", _tangent, TANGENT_PTRS), ("bwd_vl", _bwd, BWD_PTRS)]
CASES = [(entry, fn, f"attn_dense_{entry}:".encode(), *c) for entry, fn, names in ENTRIES
         for c in _pointer_cases(names) + SHAPE_CASES]
CASES += [("bwd_vl", _bwd, b"attn_dense_bwd_vl:", "workspace one byte short", dict(b=2, h=2, lq=256, workspace_bytes=4 * 2 * 2 * 256 - 1),
           WORKSPACE, b"workspace")]


@pytest.mark.parametrize("entry,fn,prefix,name,kw,code,needle",
                         [pytest.param(*c, id=f"{c[0]}-{c[3]}".replace(" ", "-")) for c in CASES])
def test_argument_checks_return_codes(lib, entry, fn, prefix, name, kw, code, needle):
    rc = fn(lib, **kw)
    msg = lib.tdb200_last_error() or b""
    assert rc == code, (entry, name, rc, msg)
    assert msg.startswith(prefix) and needle in msg, (entry, name, msg)


def test_a_misaligned_q_lens_is_named(lib):
    for entry, fn, _ in ENTRIES:
        assert fn(lib, q_lens=_p(4098)) == INVALID
        assert b"q_lens" in (lib.tdb200_last_error() or b""), entry


def test_valid_calls_without_a_gpu_report_an_error_code(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("this check is for hosts without a GPU")
    for dtype in (BF16, FP16):
        for _, fn, _ in ENTRIES:
            rc = fn(lib, dtype=dtype)
            assert rc in (-3, -4) and lib.tdb200_last_error(), (fn.__name__, rc)


def test_twins_are_exported_beside_the_entry_points_they_mirror(lib):
    from turbodiffusion_b200 import _lib
    names = set(_lib.exported_names())
    for base in ("fwd", "fwd_lse", "jvp", "jvp_lse", "tangent", "bwd"):
        assert {f"tdb200_attn_dense_{base}", f"tdb200_attn_dense_{base}_kl", f"tdb200_attn_dense_{base}_vl"} <= names
    assert lib.tdb200_abi_version() == 2          # added symbols break no caller


# ------------------------------------------------------------------------------------------------ lengths and masks
def _query_lens(q_lens, b=3, lq=6):
    import torch
    from turbodiffusion_b200.ops.core import _query_lens
    return _query_lens("dense_attention", q_lens, b, lq, torch.device("cpu"))


def test_no_lengths_stay_none():
    assert _query_lens(None) is None


@pytest.mark.parametrize("dtype", ["int64", "int32", "int16", "uint8"])
def test_integer_lengths_become_int32(dtype):
    import torch
    out = _query_lens(torch.tensor([6, 0, 3], dtype=getattr(torch, dtype)))
    assert out.dtype == torch.int32 and out.is_contiguous() and out.tolist() == [6, 0, 3]


def test_a_prefix_mask_becomes_its_lengths():
    import torch
    mask = torch.tensor([[1, 1, 1, 1, 1, 1], [0, 0, 0, 0, 0, 0], [1, 1, 1, 0, 0, 0]], dtype=torch.bool)
    out = _query_lens(mask)
    assert out.dtype == torch.int32 and out.tolist() == [6, 0, 3]


@pytest.mark.parametrize("row", [[0, 1, 1, 1, 1, 1], [1, 0, 1, 0, 0, 0], [1, 1, 1, 0, 0, 1], [0, 0, 0, 0, 0, 1]],
                         ids=["leading-false", "hole", "trailing-true", "last-only"])
def test_a_mask_that_is_not_a_prefix_is_refused(row):
    import torch
    mask = torch.ones(3, 6, dtype=torch.bool)
    mask[1] = torch.tensor(row, dtype=torch.bool)
    with pytest.raises(ValueError, match="query-padding mask must keep a prefix"):
        _query_lens(mask)


@pytest.mark.parametrize("q_lens,match", [
    ("lengths [2]", "q_lens must be an integer tensor"), ("lengths [3, 1]", "integer tensor"), ("float lengths", "integer tensor"),
    ("mask [3, 5]", r"query-padding mask \[B, Lq\]"), ("mask [2, 6]", "mask"), ("-1", r"q_lens .* outside \[0, Lq"),
    ("lq + 1", r"outside \[0, Lq = 6\]"),
])
def test_bad_lengths_and_masks_are_refused(q_lens, match):
    import torch
    arg = {"lengths [2]": torch.tensor([1, 2]), "lengths [3, 1]": torch.tensor([[1], [2], [3]]),
           "float lengths": torch.tensor([1.0, 2.0, 3.0]), "mask [3, 5]": torch.ones(3, 5, dtype=torch.bool),
           "mask [2, 6]": torch.ones(2, 6, dtype=torch.bool), "-1": torch.tensor([1, -1, 3]),
           "lq + 1": torch.tensor([1, 7, 3])}[q_lens]
    with pytest.raises(ValueError, match=match):
        _query_lens(arg)


def test_a_list_is_refused():
    with pytest.raises(TypeError, match="q_lens"):
        _query_lens([1, 2, 3])


def test_key_lengths_keep_their_messages():
    import torch
    from turbodiffusion_b200.ops.core import _key_lens
    with pytest.raises(ValueError, match=r"k_lens \[1, 7, 3\] outside \[0, Lk = 6\]"):
        _key_lens("dense_attention", torch.tensor([1, 7, 3]), 3, 6, torch.device("cpu"))
    with pytest.raises(ValueError, match="key-padding mask must keep a prefix"):
        _key_lens("dense_attention", torch.tensor([[0, 1]] * 3, dtype=torch.bool), 3, 2, torch.device("cpu"))


# ------------------------------------------------------------------------------------------------ dispatch
# position of q_lens in each _vl entry point's arguments (k_lens follows it)
_QPOS = {"tdb200_attn_dense_fwd_vl": 8, "tdb200_attn_dense_fwd_lse_vl": 9, "tdb200_attn_dense_jvp_vl": 12,
         "tdb200_attn_dense_jvp_lse_vl": 13, "tdb200_attn_dense_tangent_vl": 13, "tdb200_attn_dense_bwd_vl": 15}


class _Recorder:
    """Stands in for the library: records which entry points are called, and what the q_lens and k_lens of the _vl twins hold
    at the time of the call (CPU tensors stand in for device tensors, so their pointers can be read)"""

    def __init__(self, b):
        self.b = b
        self.calls = []
        self.lens = []

    def __getattr__(self, name):
        pos = _QPOS.get(name)

        def fn(*args):
            self.calls.append(name)
            if pos is not None:
                read = lambda p: list((ctypes.c_int32 * self.b).from_address(p)) if p else None  # noqa: E731
                self.lens.append((read(args[pos]), read(args[pos + 1])))
            return 256 if name.endswith("_workspace_bytes") else 0
        return fn


@pytest.fixture
def recorder(monkeypatch):
    from turbodiffusion_b200.ops import core
    rec = _Recorder(2)
    monkeypatch.setattr(core, "lib", lambda: rec)
    monkeypatch.setattr(core, "require_cuda", lambda *t: None)      # CPU tensors stand in for device tensors
    monkeypatch.setattr(core, "stream_ptr", lambda device=None: 0)
    return rec


def _qkv(grad=()):
    import torch
    q, k, v = torch.zeros(2, 5, 2, 128, dtype=torch.bfloat16), torch.zeros(2, 4, 2, 128, dtype=torch.bfloat16), \
        torch.zeros(2, 4, 2, 128, dtype=torch.bfloat16)
    for i in grad:
        (q, k, v)[i].requires_grad_()
    return q, k, v


def _qlens():
    import torch
    return torch.tensor([5, 2], dtype=torch.int64)


def test_no_grad_without_query_lengths_takes_todays_entry_points(recorder):
    import torch
    from turbodiffusion_b200 import ops
    q, k, v = _qkv()
    ops.dense_attention(q, k, v)
    ops.dense_attention(q, k, v, q_lens=None)
    ops.dense_attention(q, k, v, k_lens=torch.tensor([4, 1]), q_lens=None)
    ops.dense_attention_jvp(q, k, v, q, k, v, q_lens=None)
    ops.dense_attention_jvp(q, k, v, q, k, v, k_lens=torch.tensor([4, 1]))
    assert recorder.calls == ["tdb200_attn_dense_fwd"] * 2 + ["tdb200_attn_dense_fwd_kl", "tdb200_attn_dense_jvp",
                                                               "tdb200_attn_dense_jvp_kl"]


def test_no_grad_with_query_lengths_takes_the_vl_twins(recorder):
    import torch
    from turbodiffusion_b200 import ops
    q, k, v = _qkv()
    ops.dense_attention(q, k, v, q_lens=_qlens())
    ops.dense_attention(q, k, v, q_lens=_qlens(), k_lens=torch.tensor([3, 0]))
    ops.dense_attention_jvp(q, k, v, q, k, v, q_lens=torch.tensor([[1, 1, 0, 0, 0], [1, 1, 1, 1, 1]], dtype=torch.bool),
                            k_lens=torch.tensor([[1, 1, 0, 0], [1, 1, 1, 1]], dtype=torch.bool))
    assert recorder.calls == ["tdb200_attn_dense_fwd_vl"] * 2 + ["tdb200_attn_dense_jvp_vl"]
    assert recorder.lens == [([5, 2], [4, 4]), ([5, 2], [3, 0]), ([2, 5], [2, 4])]   # k_lens = Lk when only q_lens is given


@pytest.mark.parametrize("with_lens", [False, True], ids=["none", "lengths"])
def test_training_paths_pick_by_query_lengths(recorder, with_lens):
    import torch
    from turbodiffusion_b200 import ops
    ql = _qlens() if with_lens else None
    sfx = "_vl" if with_lens else ""
    q, k, v = _qkv(grad=(0, 1, 2))
    ops.dense_attention(q, k, v, q_lens=ql).float().sum().backward()
    assert recorder.calls == [f"tdb200_attn_dense_fwd_lse{sfx}", "tdb200_attn_dense_bwd_workspace_bytes", f"tdb200_attn_dense_bwd{sfx}"]
    assert all(t.grad is not None and t.grad.shape == t.shape for t in (q, k, v))
    recorder.calls.clear()
    q, k, v = _qkv(grad=(0, 1, 2))
    q_t, k_t, v_t = (torch.zeros_like(t) for t in (q, k, v))
    out, out_t = ops.dense_attention_jvp(q, k, v, q_t, k_t, v_t, q_lens=ql)
    assert out.requires_grad and not out_t.requires_grad
    out.float().sum().backward()
    assert recorder.calls == [f"tdb200_attn_dense_jvp_lse{sfx}", "tdb200_attn_dense_bwd_workspace_bytes", f"tdb200_attn_dense_bwd{sfx}"]
    if with_lens:   # the backward reads the lengths the forward saved
        assert recorder.lens == [([5, 2], [4, 4])] * 4


@pytest.mark.parametrize("with_lens", [False, True], ids=["none", "lengths"])
@pytest.mark.parametrize("how", ["func.jvp", "forward_ad"])
def test_forward_ad_picks_by_query_lengths(recorder, with_lens, how):
    import torch
    import torch.autograd.forward_ad as fwAD
    from turbodiffusion_b200 import ops
    ql = _qlens() if with_lens else None
    sfx = "_vl" if with_lens else ""
    q, k, v = _qkv()
    if how == "func.jvp":
        torch.func.jvp(lambda q_: ops.dense_attention(q_, k, v, q_lens=ql), (q,), (torch.zeros_like(q),))
    else:
        with fwAD.dual_level():
            out = ops.dense_attention(fwAD.make_dual(q, torch.zeros_like(q)), k, v, q_lens=ql)
            assert fwAD.unpack_dual(out).tangent is not None
    assert recorder.calls == [f"tdb200_attn_dense_fwd_lse{sfx}", f"tdb200_attn_dense_tangent{sfx}"]


def test_query_lengths_are_checked_before_any_library_call(recorder):
    import torch
    from turbodiffusion_b200 import ops
    q, k, v = _qkv(grad=(0,))
    with pytest.raises(ValueError):
        ops.dense_attention(q, k, v, q_lens=torch.tensor([6, 1]))
    with pytest.raises(ValueError):
        ops.dense_attention(q, k, v, q_lens=torch.tensor([-1, 1]))
    with pytest.raises(ValueError):
        ops.dense_attention_jvp(q, k, v, q.detach(), k, v, q_lens=torch.tensor([[0, 1, 1, 1, 1], [1, 0, 0, 0, 0]], dtype=torch.bool))
    with pytest.raises(ValueError):
        ops.dense_attention(q, k, v, q_lens=torch.ones(2, 4, dtype=torch.bool))   # a key-sized mask
    assert recorder.calls == []
