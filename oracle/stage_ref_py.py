"""Stage the reference's own PYTHON sources (network, sampler-side utilities, model surgery, SLA Triton kernels, ops/core.py)
into oracle/_ref/py/ (git-ignored: nothing here enters history), where tests/test_gpu_reference_model.py finds them.

TEST INFRASTRUCTURE ONLY, like oracle/build_ref_ext.py: the test runs the UNMODIFIED reference WanModel on this repo's
operators through install().  Never imported by turbodiffusion_b200.  Needs the reference sources at /root/reference; without
them nothing is staged and the test skips.

    python oracle/stage_ref_py.py        (also called by __graft_entry__.build() when /root/reference is present)
"""
import os
import shutil
import sys

REF = "/root/reference/turbodiffusion"
HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_ref", "py")

# package -> files/directories copied verbatim (no cutlass tree, no checkpoints, no assets)
WANTED = ["rcm/__init__.py", "rcm/networks", "rcm/utils", "imaginaire", "SLA", "ops/__init__.py", "ops/core.py",
          "inference/modify_model.py"]


def stage(verbose=False):
    if not os.path.isdir(REF):
        return None
    os.makedirs(OUT, exist_ok=True)
    for rel in WANTED:
        src, dst = os.path.join(REF, rel), os.path.join(OUT, rel)
        if not os.path.exists(src):
            continue
        if os.path.isdir(src):
            shutil.copytree(src, dst, dirs_exist_ok=True,
                            ignore=shutil.ignore_patterns("__pycache__", "*.pyc", "*.so", "*.png", "*.jpg", "*.mp4", "*.pth"))
        else:
            os.makedirs(os.path.dirname(dst), exist_ok=True)
            shutil.copy2(src, dst)
        if verbose:
            print("staged", rel)
    return OUT


if __name__ == "__main__":
    print(stage(verbose="-v" in sys.argv))
