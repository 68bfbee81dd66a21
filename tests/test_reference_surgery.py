"""Drop-in check of the operator API (SURVEY 8b): the reference's UNMODIFIED model surgery
(turbodiffusion/inference/modify_model.py:40-81: replace_attention + replace_linear_norm) is run on a small reference
WanModel twice in sub-processes - once resolving `ops` / `SLA` / `turbo_diffusion_ops` to the reference's own packages,
once to turbodiffusion_b200 via install() - and must produce the same module tree interface: identical state-dict keys,
shapes and dtypes (`int8_weight`, `scale`, `bias`, `...local_attn.proj_l.*`), i.e. a TurboDiffusion `-quant.pth`
checkpoint loads into either.  Needs /root/reference (build container only); no CUDA call is made (quantize=False)."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = "/root/reference/turbodiffusion"

SCRIPT = r'''
import json, sys, types
mode = sys.argv[1]
sys.path.insert(0, sys.argv[2])
import torch
stub = types.ModuleType("rcm.utils.model_utils")      # pulls in imageio (not installed); only used by create_model()
stub.load_state_dict = lambda *a, **k: {}
if mode == "ours":
    import turbodiffusion_b200
    turbodiffusion_b200.install()
else:
    ext = types.ModuleType("turbo_diffusion_ops")      # the reference's CUDA-only pybind module (not needed for surgery)
    ext.quant_cuda = ext.gemm_cuda = None
    sys.modules["turbo_diffusion_ops"] = ext
sys.path.insert(0, sys.argv[3])
sys.path.insert(0, sys.argv[3] + "/inference")
sys.modules["rcm.utils.model_utils"] = stub
import modify_model as mm
torch.manual_seed(0)
m = mm.WanModel2pt1(dim=256, eps=1e-6, ffn_dim=512, freq_dim=64, in_dim=16, model_type="t2v", num_heads=2, num_layers=2,
                    out_dim=16, text_len=32)
mm.replace_attention(m, "sla", 0.1)
mm.replace_linear_norm(m, replace_linear=True, replace_norm=True, quantize=False)
sd = m.state_dict()
blk = m.blocks[0]
out = {"state": {k: [list(v.shape), str(v.dtype)] for k, v in sd.items()},
       "types": {"attn": type(blk.self_attn.attn_op.local_attn).__name__, "linear": type(blk.self_attn.q).__name__,
                 "ln": type(blk.norm3).__name__, "rms": type(blk.self_attn.norm_q).__name__,
                 "attn_module": type(blk.self_attn.attn_op.local_attn).__module__.split(".")[0]},
       "topk": blk.self_attn.attn_op.local_attn.topk,
       "proj_l_zero": bool((blk.self_attn.attn_op.local_attn.proj_l.weight == 0).all())}
print("RESULT" + json.dumps(out))
'''


def _run(mode):
    p = subprocess.run([sys.executable, "-c", SCRIPT, mode, ROOT, REF], capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr[-3000:]
    line = [ln for ln in p.stdout.splitlines() if ln.startswith("RESULT")][-1]
    return json.loads(line[len("RESULT"):])


@pytest.mark.skipif(not os.path.isdir(REF), reason="needs the upstream TurboDiffusion sources at /root/reference (not part of this repository): the test builds "
                           "the upstream module tree itself")
def test_unmodified_reference_surgery_builds_the_same_interface():
    ours, ref = _run("ours"), _run("ref")
    assert ours["types"]["attn_module"] == "turbodiffusion_b200" and ref["types"]["attn_module"] == "SLA"
    for k in ("attn", "linear", "ln", "rms"):
        assert ours["types"][k] == ref["types"][k]
    assert ours["state"].keys() == ref["state"].keys()
    diff = {k: (ours["state"][k], ref["state"][k]) for k in ref["state"] if ours["state"][k] != ref["state"][k]}
    assert not diff, diff
    assert ours["topk"] == ref["topk"] and ours["proj_l_zero"] and ref["proj_l_zero"]    # SLA/core.py:163-166 zero init
    quant_keys = [k for k in ours["state"] if k.endswith("int8_weight")]
    assert len(quant_keys) == 2 * 10                                                     # 10 linears per block, proj_l skipped


LTX_SCRIPT = r'''
import json, sys
sys.path.insert(0, sys.argv[1])
import torch
import turbodiffusion_b200
turbodiffusion_b200.install()
base = sys.argv[2]
for p in ("ltx-distillation/src", "ltx-core/src", "ltx-pipelines/src", "ltx-trainer/src"):
    sys.path.insert(0, base + "/" + p)
import ltx_distillation.acceleration as acc
ops = acc._td_w8a8_ops()                                   # acceleration.py:690-703
model = torch.nn.Sequential(torch.nn.RMSNorm(64, eps=1e-6), torch.nn.LayerNorm(64, eps=1e-6))
n_norm = acc.replace_ltx_norms(model)                      # acceleration.py:619-635
sage = acc.LTXSageSLAAttention(head_dim=128, topk=0.3, use_bf16=True)      # acceleration.py:226-240
sla = acc.LTXSLAAttention(head_dim=64, topk=0.3, block_q=128, block_k=64, use_bf16=True)
print("RESULT" + json.dumps({
    "ops": [f.__module__ + "." + f.__name__ for f in ops], "n_norm": n_norm,
    "norm_types": [type(m).__module__ + "." + type(m).__name__ for m in model],
    "sage": type(sage.local_attn).__module__, "sla": type(sla.local_attn).__module__,
    "sage_state": sorted(sage.state_dict().keys())}))
'''


@pytest.mark.skipif(not os.path.isdir("/root/reference/TurboT2AV/LTX-2/packages"), reason="needs the upstream TurboT2AV LTX-2 packages at /root/reference (not part of this repository)")
def test_ltx_acceleration_backend_resolves_to_this_package():
    """The LTX-2 client (TurboT2AV ltx_distillation/acceleration.py) looks the W8A8 / FastNorm / SLA operators up by name
    at run time; with install() every lookup must land in turbodiffusion_b200 (incl. the gemm_cuda_swizzle* exports the
    reference snapshot's own extension lacks)."""
    p = subprocess.run([sys.executable, "-c", LTX_SCRIPT, ROOT, "/root/reference/TurboT2AV/LTX-2/packages"],
                       capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr[-3000:]
    r = json.loads([ln for ln in p.stdout.splitlines() if ln.startswith("RESULT")][-1][len("RESULT"):])
    assert r["ops"] == ["turbodiffusion_b200.ops.core.int8_quant", "turbodiffusion_b200.turbo_diffusion_ops.quant_cuda",
                        "turbodiffusion_b200.turbo_diffusion_ops.gemm_cuda_swizzle",
                        "turbodiffusion_b200.turbo_diffusion_ops.gemm_cuda_swizzle_bias"]
    assert r["n_norm"] == 2 and r["norm_types"] == ["turbodiffusion_b200.ops.core.FastRMSNorm",
                                                     "turbodiffusion_b200.ops.core.FastLayerNorm"]
    assert r["sage"].startswith("turbodiffusion_b200") and r["sla"].startswith("turbodiffusion_b200")
    assert r["sage_state"] == ["local_attn.proj_l.bias", "local_attn.proj_l.weight"]
