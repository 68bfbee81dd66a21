"""f1 (SURVEY 8f): the UNMODIFIED reference network runs on this repo's operators.

The reference's own python sources (rcm/networks/wan2pt1.py WanModel, rcm/utils/{a2a_cp,attention}.py, inference/modify_model.py)
are staged by oracle/stage_ref_py.py into the git-ignored oracle/_ref/py/ (it travels to the GPU box like oracle/_ref's compiled
extension).  With turbodiffusion_b200.install() the reference surgery (modify_model.py:40-81) resolves `ops`, `SLA` and
`turbo_diffusion_ops` to this package, quantises the random-init linears on the GPU (Int8Linear.from_linear(quantize=True),
:156-183's path) and WanModel.forward (wan2pt1.py:598-721: patch/time/text embeddings, blocks, Head, unpatchify) executes with
every block operator served by libtdb200.so.  Checked:
  * each reference block's output equals turbodiffusion_b200.block.WanBlockB200 (the fused composition bench.py times) fed the
    same block inputs and the block's own state dict, within the block tolerance (rel-L2 <= 1e-2, cos >= 0.9999);
  * the reference model's state dict carries the quantised checkpoint keys and loads back (strict) into a fresh surgery'd model.
"""
import os
import sys
import types

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_PY = os.path.join(ROOT, "oracle", "_ref", "py")


def _import_reference():
    if not os.path.isdir(os.path.join(REF_PY, "rcm")):
        pytest.skip("oracle/_ref/py not staged: the test runs the upstream TurboDiffusion WanModel sources, which are not part of "
                    "this repository (oracle/stage_ref_py.py stages them where /root/reference exists)")
    import turbodiffusion_b200
    turbodiffusion_b200.install()
    for p in (REF_PY, os.path.join(REF_PY, "inference")):
        if p not in sys.path:
            sys.path.insert(0, p)
    stub = types.ModuleType("rcm.utils.model_utils")   # pulls in imageio (not installed); only used by create_model()
    stub.load_state_dict = lambda *a, **k: {}
    sys.modules.setdefault("rcm.utils.model_utils", stub)
    import modify_model as mm
    return mm


def _build(mm, dim, heads, ffn, layers, text_len, attention, topk):
    torch.manual_seed(0)
    m = mm.WanModel2pt1(dim=dim, eps=1e-6, ffn_dim=ffn, freq_dim=64, in_dim=16, model_type="t2v", num_heads=heads,
                        num_layers=layers, out_dim=16, text_len=text_len)
    m.init_weights()
    with torch.no_grad():   # non-trivial modulation / norm weights / biases so every fused path is exercised
        for blk in m.blocks:
            blk.modulation.normal_(0, 0.3)
            for lin in (blk.self_attn.q, blk.self_attn.k, blk.self_attn.v, blk.self_attn.o, blk.cross_attn.q, blk.cross_attn.k,
                        blk.cross_attn.v, blk.cross_attn.o, blk.ffn[0], blk.ffn[2]):
                lin.bias.normal_(0, 0.02)
            for nrm in (blk.self_attn.norm_q, blk.self_attn.norm_k, blk.cross_attn.norm_q, blk.cross_attn.norm_k):
                nrm.weight.normal_(1.0, 0.1)
            blk.norm3.weight.normal_(1.0, 0.1)
            blk.norm3.bias.normal_(0, 0.05)
    # the reference flow (modify_model.py:159-183): bf16 checkpoint weights, replace_attention (fp32 proj_l), move to the GPU,
    # then replace_linear_norm, which quantises the linears on the device
    m = m.to(torch.bfloat16)
    mm.replace_attention(m, attention, topk)
    m = m.to("cuda")
    mm.replace_linear_norm(m, replace_linear=True, replace_norm=True, quantize=True)
    m = m.to("cuda")   # the FastNorm buffers are created on the host by from_*norm; create_model moves the net last, too (:139)
    with torch.no_grad():
        for blk in m.blocks:  # proj_l is zero-initialised (SLA/core.py:163-166): give the linear branch something to do
            blk.self_attn.attn_op.local_attn.proj_l.weight.normal_(0, 0.05)
            blk.self_attn.attn_op.local_attn.proj_l.bias.normal_(0, 0.05)
    return m.eval()


@pytest.mark.parametrize("attention", ["sagesla", "sla"])
def test_reference_wan_model_forward_on_b200_operators(cuda, attention):
    mm = _import_reference()
    from turbodiffusion_b200.block import WanBlockB200
    from oracle import td_oracle as O
    dim, heads, ffn, layers, text_len, topk = 256, 2, 512, 3, 32, 0.3
    m = _build(mm, dim, heads, ffn, layers, text_len, attention, topk)
    blk0 = m.blocks[0]
    assert type(blk0.self_attn.q).__module__.startswith("turbodiffusion_b200")
    assert type(blk0.self_attn.attn_op.local_attn).__module__.startswith("turbodiffusion_b200")
    assert type(blk0.norm3).__module__.startswith("turbodiffusion_b200")

    captured = []

    def hook(mod, args, kwargs, out):
        captured.append((args[0].detach().clone(), {k: (v.detach().clone() if torch.is_tensor(v) else v) for k, v in kwargs.items()},
                         out.detach().clone()))

    handles = [b.register_forward_hook(hook, with_kwargs=True) for b in m.blocks]
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn(1, 16, 3, 20, 40, device=cuda, generator=g).bfloat16()          # -> L = 3*10*20 = 600 tokens
    t = torch.tensor([[500.0]], device=cuda)
    ctx = torch.randn(1, text_len, 4096, device=cuda, generator=g).bfloat16()
    with torch.no_grad():
        y = m(x, t, ctx)
    torch.cuda.synchronize()
    for h in handles:
        h.remove()
    assert y.shape == x.shape and torch.isfinite(y.float()).all()
    assert len(captured) == layers

    for i, (xin, kw, out) in enumerate(captured):
        sd = {k: v for k, v in m.blocks[i].state_dict().items()}
        blk = WanBlockB200(sd, dim, heads, eps=1e-6, topk=topk, attention=attention)
        got = blk(xin[0], kw["e"][0].float(), kw["freqs"].view(xin.shape[1], -1).float(), kw["context"][0])
        s = O.stats(got.cpu(), out[0].cpu())
        assert s["cos"] >= 0.9999 and s["rel_l2"] <= 1e-2, (attention, i, s)

    # checkpoint round trip: the quantised state dict loads (strict) into a freshly surgery'd model and reproduces y
    sd = m.state_dict()
    assert any(k.endswith("int8_weight") for k in sd) and any(k.endswith("local_attn.proj_l.weight") for k in sd)
    m2 = _build(mm, dim, heads, ffn, layers, text_len, attention, topk)
    m2.load_state_dict(sd, strict=True)
    with torch.no_grad():
        y2 = m2(x, t, ctx)
    assert torch.equal(y, y2)
