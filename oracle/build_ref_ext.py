"""Build the REFERENCE's own CUDA extension `turbo_diffusion_ops` (quant_cuda / gemm_cuda / *_norm_cuda) from the
sources where they lie under /root/reference, into oracle/_ref/ (git-ignored, travels to the GPU box with gpurun).

TEST INFRASTRUCTURE ONLY: used by tests/test_gpu_vs_reference_ext.py to cross-check the H100 kernels against the
reference kernels on the same GPU and to time the reference GEMM on H100.  Never imported by turbodiffusion_b200.
No reference source is copied into this repository; the compile reads them in place with the reference's own flags
(setup.py:22-41), arch restricted to sm_90.
"""
import os
import sys

REF = "/root/reference"
HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_ref")


def build(verbose=False):
    if not os.path.isdir(REF):
        return None
    import glob
    existing = glob.glob(os.path.join(OUT, "turbo_diffusion_ops*.so"))
    if existing:
        return existing[0]
    os.makedirs(OUT, exist_ok=True)
    os.environ.setdefault("TORCH_CUDA_ARCH_LIST", "10.0")
    os.environ.setdefault("MAX_JOBS", "6")
    from torch.utils.cpp_extension import load
    ops = os.path.join(REF, "turbodiffusion", "ops")
    cutlass = os.path.join(ops, "cutlass")
    nvcc_flags = ["-O3", "-std=c++17", "-U__CUDA_NO_HALF_OPERATORS__", "-U__CUDA_NO_HALF_CONVERSIONS__",
                  "-U__CUDA_NO_BFLOAT16_OPERATORS__", "-U__CUDA_NO_BFLOAT16_CONVERSIONS__",
                  "-U__CUDA_NO_BFLOAT162_OPERATORS__", "-U__CUDA_NO_BFLOAT162_CONVERSIONS__", "--expt-relaxed-constexpr",
                  "--expt-extended-lambda", "--use_fast_math", "-lineinfo", "-DCUTLASS_DEBUG_TRACE_LEVEL=0", "-DNDEBUG",
                  "-DEXECMODE=0", "-gencode", "arch=compute_90,code=sm_90"]
    load(name="turbo_diffusion_ops",
         sources=[os.path.join(ops, f) for f in ("bindings.cpp", "quant/quant.cu", "norm/rmsnorm.cu", "norm/layernorm.cu", "gemm/gemm.cu")],
         extra_include_paths=[os.path.join(cutlass, "include"), os.path.join(cutlass, "tools", "util", "include"), ops],
         extra_cflags=["-O3", "-std=c++17"], extra_cuda_cflags=nvcc_flags, build_directory=OUT, verbose=verbose,
         is_python_module=False)
    got = glob.glob(os.path.join(OUT, "turbo_diffusion_ops*.so"))
    return got[0] if got else None


if __name__ == "__main__":
    print(build(verbose="-v" in sys.argv))
