"""The wgmma kernels compile to pipelined MMAs without spills (host only: nvcc cross-compiles for sm_90a without a GPU).

ptxas note C7514 ("wgmma.mma_async instructions are serialized due to non wgmma instructions reading accumulator registers of a
wgmma between start and end of the pipeline stage") means it put a wait after every wgmma of that kernel, so each MMA's whole
latency is exposed.  It appears silently after an edit that reads or copies an accumulator while its MMA may be in flight (a
fence through a reinterpreted pointer, a P.V left in flight across a loop's back edge).  Spills put local-memory traffic in the
inner loops.  Each source that issues wgmma is compiled with the library's own nvcc flags plus -Xptxas -v.
"""
from __future__ import annotations

import concurrent.futures as cf
import os
import re
import shutil
import subprocess

import pytest

from turbodiffusion_b200 import _build

_NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"


def _wgmma_sources():
    out = []
    for src in _build.sources():
        with open(os.path.join(_build.CSRC, src)) as f:
            if "wgmma_commit()" in f.read():
                out.append(src)
    return out


def _ptxas_report(src, tmp):
    cmd = [_NVCC] + _build.NVCC_FLAGS + ["-Xptxas", "-v", "-I", _build.INCLUDE, "-c", os.path.join(_build.CSRC, src),
                                         "-o", os.path.join(tmp, src[:-3] + ".o")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, f"nvcc failed on {src}:\n{r.stderr}"
    return r.stderr


def _findings(report):
    """(kernel, problem) for every C7514 note and every kernel with spill stores or loads in one ptxas -v report."""
    found, kernel = [], None
    for line in report.splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", line)
        if m:
            kernel = m.group(1)
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and (int(m.group(1)) or int(m.group(2))):
            found.append((kernel, line.strip()))
        if "C7514" in line:
            m = re.search(r"in the function '([^']+)'", line)
            found.append((m.group(1) if m else kernel, "C7514: wgmma serialized"))
    return found


@pytest.fixture(scope="module")
def reports(tmp_path_factory):
    if not os.path.exists(_NVCC):
        pytest.skip("nvcc not available")
    tmp = str(tmp_path_factory.mktemp("ptxas"))
    srcs = _wgmma_sources()
    with cf.ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        return dict(zip(srcs, ex.map(lambda s: _ptxas_report(s, tmp), srcs)))


def test_every_wgmma_source_is_checked(reports):
    assert {"sla_attn.cu", "dense_attn.cu", "sla_attn_bwd.cu", "sla_moments.cu", "gemm_w8a8.cu"} <= set(reports)


def test_no_kernel_serializes_its_wgmma(reports):
    bad = [(src, k) for src, rep in reports.items() for k, what in _findings(rep) if what.startswith("C7514")]
    assert not bad, f"ptxas serialised the wgmma of: {bad}"


def test_no_kernel_spills(reports):
    bad = [(src, k, what) for src, rep in reports.items() for k, what in _findings(rep) if not what.startswith("C7514")]
    assert not bad, f"spills: {bad}"


def test_findings_parser():
    rep = ("ptxas info    : Compiling entry function 'k1' for 'sm_90a'\n"
           "    0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads\n"
           "ptxas info    : Compiling entry function 'k2' for 'sm_90a'\n"
           "ptxas info    : (C7514) Potential Performance Loss: wgmma.mma_async instructions are serialized due to non wgmma "
           "instructions reading accumulator registers of a wgmma between start and end of the pipeline stage in the function 'k2'\n"
           "    8 bytes stack frame, 4 bytes spill stores, 4 bytes spill loads\n")
    assert _findings(rep) == [("k2", "C7514: wgmma serialized"),
                              ("k2", "8 bytes stack frame, 4 bytes spill stores, 4 bytes spill loads")]
