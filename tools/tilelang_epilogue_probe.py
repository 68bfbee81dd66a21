"""Pins the rounding points of the LTX per-row W8A8 GEMM epilogue (SURVEY row f3) without a GPU.

Imports the reference's TileLang kernel factory from /root/reference (read-only, build container only), lowers it to CUDA C
with TileLang's own code generator, compiles that with nvcc the way TileLang's JIT does (default flags: -fmad=true, no
fast-math; tilelang/jit/adapter/libgen.py) and counts the floating-point SASS instructions of the epilogue.  Result:
per thread 64 I2FP.F32.S32 + 64 FMUL + 64 FFMA and no FADD, i.e.
    c = bf16( fma( float(acc) * sA[i], sB[j], bias[j] ) )
which is what oracle.td_oracle.ltx_gemm_post_scale and tdb200_gemm_w8a8_rowwise compute.

usage: python tools/tilelang_epilogue_probe.py [out_dir]     (needs /root/reference, tilelang, nvcc; not used at run time)
"""
import collections
import importlib.util
import os
import re
import subprocess
import sys

REF = "/root/reference/TurboT2AV/LTX-2/packages/ltx-distillation/src/ltx_distillation/tilelang_w8a8.py"


def main():
    out_dir = sys.argv[1] if len(sys.argv) > 1 else os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "gpurun_out")
    os.makedirs(out_dir, exist_ok=True)
    import tilelang
    from tilelang import tvm
    spec = importlib.util.spec_from_file_location("ref_tilelang_w8a8", REF)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    jit = mod._tl_gemm_int8_post_scale_bias          # tilelang_w8a8.py:78-117
    try:
        prim = jit.get_tir(256, 256, 256)
    except Exception:
        jit.func.mode = "lazy"
        prim = jit.func(256, 256, 256)
    target = tvm.target.Target("cuda -arch=sm_90")
    with target:
        art = tilelang.lower(prim, target=target)
    cu = os.path.join(out_dir, "tl_post_scale_gemm.cu")
    with open(cu, "w") as f:
        f.write(art.kernel_source)
    tl_root = os.path.dirname(tilelang.__file__)
    cubin = cu.replace(".cu", ".cubin")
    subprocess.run(["nvcc", "-std=c++17", "-w", "-gencode", "arch=compute_90a,code=sm_90a", "-I" + os.path.join(tl_root, "src"),
                    "-I" + os.path.join(tl_root, "3rdparty", "cutlass", "include"), "-cubin", "-o", cubin, cu], check=True)
    sass = subprocess.run(["cuobjdump", "-sass", cubin], check=True, capture_output=True, text=True).stdout
    counts = collections.Counter(re.findall(r"\b(I2FP?[A-Z0-9.]*|FFMA[A-Z0-9.]*|FMUL[A-Z0-9.]*|FADD[A-Z0-9.]*|F2FP[A-Z0-9.]*)", sass))
    epilogue = [ln.strip() for ln in art.kernel_source.splitlines() if re.search(r"__[2345]\.x = ", ln)]
    print("# generated CUDA C of the epilogue (one lane of the float2):")
    for ln in epilogue:
        print("   ", ln)
    print("# SASS floating-point instruction counts of the whole kernel (sm_90a, nvcc default flags):")
    for k, v in sorted(counts.items()):
        print(f"    {v:4d}  {k}")


if __name__ == "__main__":
    main()
