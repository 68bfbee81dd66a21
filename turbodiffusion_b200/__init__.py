"""turbodiffusion_b200 — H100 (sm_90a) implementation of TurboDiffusion's denoise hot path.

Host code is Python/PyTorch (device memory, streams, torch.distributed); all arithmetic runs in hand-written CUDA
kernels inside libtdb200.so, reached through the C ABI in include/tdb200.h.  The sub-packages mirror the reference's
operator API:  turbodiffusion_b200.ops  <->  turbodiffusion.ops,   turbodiffusion_b200.SLA  <->  turbodiffusion.SLA,
turbodiffusion_b200.turbo_diffusion_ops  <->  the pybind module turbo_diffusion_ops.
"""
from __future__ import annotations

import sys

__version__ = "0.1.0"


def install(sage_arch: str = "sm100", sla_linear_branch: str = "reference", sage_pv: str = None) -> None:
    """Register this package under the reference's module names so unmodified reference code
    (`from ops import FastLayerNorm, FastRMSNorm, Int8Linear`, `from SLA import ...`, `import turbo_diffusion_ops`;
    turbodiffusion/inference/modify_model.py:33-37) resolves to this implementation.  `sage_arch` is handed to
    SLA.utils.set_served_arch: "sm90" gives SageSLA the block sizes the reference uses on an H100 (BLKQ=64, BLKK=128).
    `sla_linear_branch` is handed to SLA.utils.set_linear_branch: "fused" runs SparseLinearAttention's training linear branch
    through the CUDA kernels of SLA.core.linear_branch, also in modules that reference code constructs.  `sage_pv`, when given,
    is handed to SLA.utils.set_sage_pv: "fp8" runs SageSLA's P.V on e4m3 P and V; None keeps the current setting (whose
    default comes from TDB200_SAGE_PV)."""
    from . import ops, SLA, turbo_diffusion_ops
    from .SLA.utils import set_linear_branch, set_sage_pv, set_served_arch
    set_linear_branch(sla_linear_branch)
    set_served_arch(sage_arch)
    if sage_pv is not None:
        set_sage_pv(sage_pv)
    for name, mod in (("turbo_diffusion_ops", turbo_diffusion_ops), ("ops", ops), ("SLA", SLA),
                      ("turbodiffusion.ops", ops), ("turbodiffusion.SLA", SLA)):
        sys.modules[name] = mod
