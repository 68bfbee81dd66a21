"""GPU checks of the software-pipelined 128 x 64 SLA forward kernel (sla_attn_fwd_kernel) at the edges of its pipeline, on
hand-made block lists, against the oracle at the existing bars.

The kernel issues S_{j+1} = Q.K_{j+1}^T beside P_j.V_j, with a prologue for S_0 and a separate path for the last entry, over
three-slot K and V rings.  So the cases are: 1 to 4 LUT entries (one entry alone, and the ring depth -1, 0, +1); the ragged
last key block first or last in the LUT; the lazy rescale of O firing at the second or the last entry, or never (largest
block first); bf16 and fp16; head dim 64 on the INT8 path; the 16-bit forward and its lse forward; and a CUDA-graph replay.

Bars (those of tests/test_gpu_sla.py): INT8 Q.K: cos >= 0.999, rel-L2 <= 2e-2 against the fp32 oracle, and at large scores
rel-L2 <= 3e-2 against the oracle's INT8 emulation with cos >= 0.99 against fp32; 16-bit Q.K: cos >= 0.9999, rel-L2 <= 5e-3;
lse within 1e-3 + 1e-5 max|s| (log2 units) of float64."""
import math

import pytest
import torch

from oracle import td_oracle as O

pytestmark = pytest.mark.gpu
BLKQ, BLKK = 128, 64
L = 1000                   # 16 key blocks, the last one ragged (40 keys); 8 query blocks, the last one ragged
NBLK = -(-L // BLKK)
RAGGED = NBLK - 1


def _inputs(d, dtype, seed, boost=None, h=2):
    """q, k, v [1, L, H, d] on the GPU; `boost` = (key block, factor) scales that block's keys, so its scores are larger."""
    g = torch.Generator().manual_seed(seed)
    q, k, v = (torch.randn(1, L, h, d, generator=g) for _ in range(3))
    if boost is not None:
        blk, f = boost
        k[:, blk * BLKK:(blk + 1) * BLKK] *= f
    return [t.to(dtype).cuda() for t in (q, k, v)]


def _lut(entries, h=2):
    mblk = -(-L // BLKQ)
    return torch.tensor(entries, dtype=torch.int32).view(1, 1, 1, -1).expand(1, h, mblk, len(entries)).contiguous().cuda()


def _weights(d):
    g = torch.Generator().manual_seed(5)
    return (torch.randn(d, d, generator=g) * 0.05).cuda(), (torch.randn(d, generator=g) * 0.05).cuda()


def _int8_forward(q, k, v, lut, w, bias):
    from turbodiffusion_b200.SLA.core import attn_fwd, linear_moments, project_moments
    from turbodiffusion_b200.SLA.utils import quant_qk
    d = q.shape[-1]
    prep = quant_qk(q, k)
    kv, ksum = linear_moments(k, v)
    kvw = project_moments(w, kv, q.dtype)
    return attn_fwd(prep, v, q, lut, lut.shape[-1], kvw, ksum, bias.float().contiguous(), d ** -0.5)


def _qk16_forward(q, k, v, lut, w, bias):
    from turbodiffusion_b200.SLA.core import attn_fwd_qk16, linear_moments, project_moments
    d = q.shape[-1]
    kv, ksum = linear_moments(k, v)
    kvw = project_moments(w, kv, q.dtype)
    return attn_fwd_qk16(q, k, v, lut, lut.shape[-1], kvw, ksum, bias.float().contiguous(), d ** -0.5)


def _check(out, q, k, v, lut, w, bias, cos, rel):
    exact = O.sla_forward(q.cpu(), k.cpu(), v.cpu(), w.cpu(), bias.cpu(), 0.0, mode="exact", lut=lut.cpu(), dtype=q.dtype)
    s = O.stats(out.cpu(), exact)
    assert s["cos"] >= cos and s["rel_l2"] <= rel, s
    return s


LUTS = {
    "one": [3],
    "two": [3, 8],
    "three": [3, 8, 1],
    "four": [3, 8, 1, 12],
    "ragged_first": [RAGGED, 2, 7, 4, 9],
    "ragged_last": [2, 7, 4, 9, RAGGED],
    "ragged_alone": [RAGGED],
}
DTYPES = [pytest.param(torch.bfloat16, id="bf16"), pytest.param(torch.float16, id="fp16")]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("name", list(LUTS))
def test_int8_forward_lut_shapes(cuda, name, dtype):
    q, k, v = _inputs(128, dtype, 10 + len(name))
    lut = _lut(LUTS[name])
    w, bias = _weights(128)
    _check(_int8_forward(q, k, v, lut, w, bias), q, k, v, lut, w, bias, 0.999, 2e-2)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("name", list(LUTS))
def test_qk16_forward_lut_shapes(cuda, name, dtype):
    q, k, v = _inputs(128, dtype, 20 + len(name))
    lut = _lut(LUTS[name])
    w, bias = _weights(128)
    _check(_qk16_forward(q, k, v, lut, w, bias), q, k, v, lut, w, bias, 0.9999, 5e-3)


# the boosted block at LUT position `pos`: its scores exceed every earlier entry's maximum by far more than 2^8, so the lazy
# rescale of O fires there (position 0: the largest block comes first and the rescale never fires)
RESCALE = {"first": 0, "second": 1, "last": 4}


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("where", list(RESCALE))
def test_lazy_rescale_position(cuda, where, dtype):
    entries = [5, 2, 11, 7, RAGGED]
    pos = RESCALE[where]
    q, k, v = _inputs(128, dtype, 31, boost=(entries[pos], 8.0))
    lut = _lut(entries)
    w, bias = _weights(128)
    # INT8 Q.K at large scores: the bars of test_sage_sla_forward_large_scores_exercise_the_lazy_rescale (the score
    # quantisation itself moves the output a few 1e-2 from fp32)
    out = _int8_forward(q, k, v, lut, w, bias).cpu()
    args = (q.cpu(), k.cpu(), v.cpu(), w.cpu(), bias.cpu(), 0.0)
    s_sage = O.stats(out, O.sla_forward(*args, mode="sage", lut=lut.cpu(), dtype=dtype))
    s_exact = O.stats(out, O.sla_forward(*args, mode="exact", lut=lut.cpu(), dtype=dtype))
    assert s_sage["rel_l2"] <= 3e-2 and s_exact["cos"] >= 0.99, (s_sage, s_exact)
    _check(_qk16_forward(q, k, v, lut, w, bias), q, k, v, lut, w, bias, 0.9999, 5e-3)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("name", ["one", "four", "ragged_last"])
def test_int8_forward_head_dim_64(cuda, name, dtype):
    q, k, v = _inputs(64, dtype, 40 + len(name))
    lut = _lut(LUTS[name])
    w, bias = _weights(64)
    _check(_int8_forward(q, k, v, lut, w, bias), q, k, v, lut, w, bias, 0.999, 2e-2)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("name", ["one", "two", "four", "ragged_first", "ragged_last"])
def test_qk16_lse_forward(cuda, name, dtype):
    from turbodiffusion_b200.SLA.core import attn_fwd_qk16_lse
    q, k, v = _inputs(128, dtype, 50 + len(name), boost=(LUTS[name][-1], 4.0))
    lut = _lut(LUTS[name])
    sm = 128 ** -0.5
    o_s, lse = attn_fwd_qk16_lse(q, k, v, lut, lut.shape[-1], sm)
    qh, kh, vh = (t.transpose(1, 2).contiguous().cpu() for t in (q, k, v))
    want = O.sparse_attention(qh.float(), kh.float(), vh.float(), lut.cpu(), BLKQ, BLKK).transpose(1, 2)
    s = O.stats(o_s.cpu(), want)
    assert s["cos"] >= 0.9999 and s["rel_l2"] <= 5e-3, s
    # float64 row log-sum-exp over the selected keys, log2 units
    sel = torch.zeros(NBLK, dtype=torch.bool)
    sel[lut[0, 0, 0].long().cpu()] = True
    keep = sel[torch.arange(L) // BLKK]
    scores = (qh.double() @ kh.double().transpose(-1, -2)) * (sm / math.log(2.0))
    scores = scores.masked_fill(~keep, -math.inf)
    want_lse = torch.logsumexp(scores * math.log(2.0), -1) / math.log(2.0)
    smax = scores.masked_fill(~keep, 0.0).abs().amax(-1)
    err = (lse.cpu().double() - want_lse).abs()
    assert bool((err <= 1e-3 + 1e-5 * smax).all()), err.max().item()


def test_cuda_graph_replay(cuda):
    q, k, v = _inputs(128, torch.bfloat16, 60)
    lut = _lut(LUTS["ragged_last"])
    w, bias = _weights(128)
    from turbodiffusion_b200.SLA.core import linear_moments, project_moments
    from turbodiffusion_b200.SLA.utils import quant_qk
    from turbodiffusion_b200.SLA.core import attn_fwd
    prep = quant_qk(q, k)
    kv, ksum = linear_moments(k, v)
    kvw = project_moments(w, kv, q.dtype)
    pb = bias.float().contiguous()
    eager = attn_fwd(prep, v, q, lut, lut.shape[-1], kvw, ksum, pb, 128 ** -0.5)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        attn_fwd(prep, v, q, lut, lut.shape[-1], kvw, ksum, pb, 128 ** -0.5)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = attn_fwd(prep, v, q, lut, lut.shape[-1], kvw, ksum, pb, 128 ** -0.5)
    out.zero_()
    for _ in range(3):
        graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager)
