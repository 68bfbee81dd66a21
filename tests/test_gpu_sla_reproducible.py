"""Bit-reproducible SLA inference: the linear-attention moments are summed in a fixed order (csrc/sla_moments.cu).

  * linear_moments repeats bit for bit, at shapes A and B, for 64-wide head pairs with an odd head count, every feature map,
    fp16, b = 2, short and ragged lengths, and fewer tiles than the split cap;
  * a head slice and a single sample give the same bits as the corresponding heads / sample of a larger call;
  * the moments stay within test_linear_moments' bar against float64; a second launch into the same buffer doubles it;
  * the modules, the 30-block shape-A step (eager and CUDA-graph replay) and the Ulysses per-rank primitives are bit-identical
    across runs and to the single-GPU module's heads.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

SHAPE_A = (32760, 12, 128)   # (L, heads, head dim): Wan2.1-1.3B 480p
SHAPE_B = (75600, 40, 128)   # Wan2.1-14B 720p
FEATURES = ("softmax", "elu", "relu")
FEATURE_TAG = {"softmax": 0, "elu": 1, "relu": 2}


def _rand(shape, seed, dtype=torch.bfloat16, device="cuda", kbias=0.0):
    g = torch.Generator(device=device).manual_seed(seed)
    t = torch.randn(*shape, generator=g, device=device)
    if kbias:
        t += torch.randn(1, 1, shape[2], shape[3], generator=g, device=device) * kbias
    return t.to(dtype)


def _kv(b, l, h, d, seed, dtype=torch.bfloat16):
    return _rand((b, l, h, d), seed, dtype, kbias=2.0), _rand((b, l, h, d), seed + 1, dtype)


def _bits_equal(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def _module_bits_equal(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int16), b.contiguous().view(torch.int16))


# ---- the moments kernel -------------------------------------------------------------------------------------------------
REPEAT_CASES = [
    # b, l, h, d, feature, dtype
    (1, *SHAPE_A, "softmax", torch.bfloat16),
    (1, *SHAPE_B, "softmax", torch.bfloat16),
    (1, 32760, 24, 64, "softmax", torch.bfloat16),      # the 24 x 64 configuration: twelve head pairs
    (1, 5000, 7, 64, "softmax", torch.bfloat16),        # odd head count: the last pair has one head
    (2, 600, 3, 128, "elu", torch.float16),
    (2, 600, 5, 64, "relu", torch.float16),
    (1, 1, 2, 128, "softmax", torch.bfloat16),
    (2, 127, 3, 64, "elu", torch.bfloat16),
    (1, 128, 1, 128, "relu", torch.float16),
    (1, 600, 1, 128, "softmax", torch.float16),         # 5 tiles: fewer tiles than the split cap
    (3, 1100, 2, 128, "softmax", torch.bfloat16),       # 9 tiles: one split owns two
]


@pytest.mark.parametrize("b,l,h,d,feature,dtype", REPEAT_CASES)
def test_moments_repeat_bit_for_bit(cuda, b, l, h, d, feature, dtype):
    from turbodiffusion_b200.SLA.core import linear_moments
    k, v = _kv(b, l, h, d, 11 + l + h, dtype)
    kv0, ks0 = linear_moments(k, v, FEATURE_TAG[feature])
    for _ in range(19):
        kv, ks = linear_moments(k, v, FEATURE_TAG[feature])
        assert _bits_equal(kv, kv0) and _bits_equal(ks, ks0)


@pytest.mark.parametrize("l,h,d,a,e", [(32760, 12, 128, 2, 4), (32760, 12, 128, 11, 12), (2000, 7, 64, 1, 4),
                                       (2000, 7, 64, 3, 7), (2000, 7, 64, 6, 7), (700, 5, 128, 0, 5)])
@pytest.mark.parametrize("feature", FEATURES)
def test_moments_of_a_head_slice_are_those_heads_of_the_full_call(cuda, l, h, d, a, e, feature):
    """A slice starting at an odd head moves every 64-wide head to the other half of its pair."""
    from turbodiffusion_b200.SLA.core import linear_moments
    k, v = _kv(1, l, h, d, 70 + h)
    kv, ks = linear_moments(k, v, FEATURE_TAG[feature])
    kv_s, ks_s = linear_moments(k[:, :, a:e].contiguous(), v[:, :, a:e].contiguous(), FEATURE_TAG[feature])
    assert _bits_equal(kv_s, kv[:, a:e]) and _bits_equal(ks_s, ks[:, a:e])


@pytest.mark.parametrize("l,h,d", [(32760, 12, 128), (1000, 3, 64), (100, 2, 128)])
def test_moments_of_a_sample_alone_are_that_sample_of_a_batch(cuda, l, h, d):
    from turbodiffusion_b200.SLA.core import linear_moments
    k, v = _kv(3, l, h, d, 90)
    kv, ks = linear_moments(k, v)
    for i in range(3):
        kv_i, ks_i = linear_moments(k[i:i + 1].contiguous(), v[i:i + 1].contiguous())
        assert _bits_equal(kv_i, kv[i:i + 1]) and _bits_equal(ks_i, ks[i:i + 1]), i


def _phi64(k, feature):
    """The feature map in float64, rounded to the kernel's 16-bit type as it is before the MMA."""
    x = k.double()
    if feature == "softmax":
        p = torch.softmax(x, -1)
    elif feature == "elu":
        p = torch.nn.functional.elu(x) + 1
    else:
        p = torch.relu(x)
    return p.to(k.dtype).double()


def _rel_l2(got, ref):
    return ((got.double() - ref).norm() / ref.norm()).item()


@pytest.mark.parametrize("b,l,h,d,feature,dtype", [(1, 32760, 2, 128, "softmax", torch.bfloat16),
                                                   (2, 600, 3, 128, "elu", torch.float16),
                                                   (1, 1000, 5, 64, "relu", torch.bfloat16),
                                                   (1, 127, 3, 64, "softmax", torch.float16),
                                                   (1, 1, 1, 128, "elu", torch.bfloat16),
                                                   (3, 1100, 2, 128, "softmax", torch.bfloat16)])
def test_moments_against_float64(cuda, b, l, h, d, feature, dtype):
    """test_linear_moments' bar: rel-L2 < 3e-3 for kv and ksum."""
    from turbodiffusion_b200.SLA.core import linear_moments
    k, v = _kv(b, l, h, d, 130 + l, dtype)
    kv, ks = linear_moments(k, v, FEATURE_TAG[feature])
    phi = _phi64(k, feature).transpose(1, 2)            # [b, h, l, d]
    vh = v.double().transpose(1, 2)
    kv_ref = vh.transpose(-1, -2) @ phi                  # [b, h, dv, dk]
    ks_ref = phi.sum(-2)
    assert _rel_l2(kv, kv_ref) < 3e-3 and _rel_l2(ks, ks_ref) < 3e-3, (_rel_l2(kv, kv_ref), _rel_l2(ks, ks_ref))


@pytest.mark.parametrize("b,l,h,d", [(1, 32760, 12, 128), (2, 1000, 5, 64), (1, 90, 1, 128)])
def test_second_launch_into_the_same_buffer_doubles_it(cuda, b, l, h, d):
    from turbodiffusion_b200._lib import DTYPE_TAG, check, lib, ptr, stream_ptr
    k, v = _kv(b, l, h, d, 170 + h)
    buf = torch.zeros(b * h * d * (d + 1), dtype=torch.float32, device=cuda)

    def launch():
        check(lib().tdb200_sla_linear_moments(ptr(k), ptr(v), DTYPE_TAG[k.dtype], b, l, h, d, 0, ptr(buf),
                                              ptr(buf) + 4 * b * h * d * d, stream_ptr(k.device)), "sla_linear_moments")

    launch()
    once = buf.clone()
    assert once.abs().sum() > 0
    launch()
    assert _bits_equal(buf, once + once)


# ---- modules and the step -----------------------------------------------------------------------------------------------
def _shape_a_qkv(seed=5):
    l, h, d = SHAPE_A
    return _rand((1, l, h, d), seed), _rand((1, l, h, d), seed + 1, kbias=2.0), _rand((1, l, h, d), seed + 2)


def _with_random_proj(mod, d, seed=9):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        mod.proj_l.weight.copy_(torch.randn(d, d, generator=g) * 0.05)
        mod.proj_l.bias.copy_(torch.randn(d, generator=g) * 0.05)
    return mod


MODULES = [("sagesla", "sm100", None), ("sagesla", "sm90", None), ("sla", None, (128, 64)), ("sla", None, (64, 64))]


@pytest.mark.parametrize("kind,arch,blocks", MODULES)
def test_module_forward_is_bit_identical_across_calls_at_shape_a(cuda, kind, arch, blocks):
    from turbodiffusion_b200.SLA import SageSparseLinearAttention, SparseLinearAttention
    from turbodiffusion_b200.SLA.utils import set_served_arch
    d = SHAPE_A[2]
    prev = set_served_arch(arch or "sm100")
    try:
        if kind == "sagesla":
            mod = SageSparseLinearAttention(d, 0.1)
        else:
            mod = SparseLinearAttention(d, 0.1, BLKQ=blocks[0], BLKK=blocks[1])
        mod = _with_random_proj(mod.to(cuda), d)
        q, k, v = _shape_a_qkv()
        with torch.no_grad():
            ref = mod(q, k, v)
            for _ in range(3):
                assert _module_bits_equal(mod(q, k, v), ref)
    finally:
        set_served_arch(prev)


def test_wan_step_at_shape_a_is_bit_identical_eager_and_in_a_cuda_graph(cuda):
    """The 30-block step (random_block_state gives every block a random non-zero proj_l), twice eager and as a graph replay."""
    from turbodiffusion_b200.block import WanHotPath
    from turbodiffusion_b200.ops import wan_rope_angles
    L, dim, heads, ffn, layers, text, thw = 32760, 1536, 12, 8960, 30, 512, (21, 30, 52)
    model = WanHotPath(dim, ffn, heads, layers, cuda, topk=0.1, seed=1234)
    assert all(blk.sla.proj_l.weight.abs().sum() > 0 for blk in model.blocks)
    g = torch.Generator().manual_seed(7)
    x = torch.randn(L, dim, generator=g).bfloat16().to(cuda)
    e0 = (torch.randn(6, dim, generator=g) * 0.1).to(cuda)
    ctx = torch.randn(text, dim, generator=g).bfloat16().to(cuda)
    angles = wan_rope_angles(*thw, dim // heads).to(cuda)
    first = model.step(x, e0, angles, ctx).clone()
    second = model.step(x, e0, angles, ctx).clone()
    assert _module_bits_equal(second, first)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        model.step(x, e0, angles, ctx)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ys = model.step(x, e0, angles, ctx)
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        assert _module_bits_equal(ys, first)


@pytest.mark.parametrize("arch", ["sm100", "sm90"])
@pytest.mark.parametrize("world", [2, 4, 8])
def test_ulysses_ranks_equal_the_single_gpu_heads_bit_for_bit(cuda, arch, world):
    """Each rank's UlyssesGpuPrims.attend on its head range (12 heads over 8 ranks: 2,2,2,2,1,1,1,1) equals those heads of the
    single-GPU module output."""
    from turbodiffusion_b200.dist import UlyssesGpuPrims, split_heads
    from turbodiffusion_b200.SLA import SageSparseLinearAttention
    from turbodiffusion_b200.SLA.utils import set_served_arch
    l, h, d = SHAPE_A
    prev = set_served_arch(arch)
    try:
        mod = _with_random_proj(SageSparseLinearAttention(d, 0.1).to(cuda), d)
        q, k, v = _shape_a_qkv(seed=21)
        with torch.no_grad():
            ref = mod(q, k, v)
            prims = UlyssesGpuPrims(mod, arch)
            counts, offsets = split_heads(h, world)
            for n, a in zip(counts, offsets):
                qs, ks, vs = (t[:, :, a:a + n].contiguous() for t in (q, k, v))
                got = prims.attend(lambda: qs, lambda: ks, lambda: vs)
                assert _module_bits_equal(got, ref[:, :, a:a + n]), (a, n)
    finally:
        set_served_arch(prev)
