"""-m gpu: LoRA merging on the CUDA path.
  * a pipeline loaded with a LoRA gives bitwise the images and latents of one loaded from a checkpoint directory
    whose UNet and text encoder were merged beforehand with the reference's arithmetic (editany_lora.py:241-264);
  * SD1.5 at 512x512, 1 image + CFG, two ControlNets and a rank-64 LoRA at multiplier 0.5: the engine's eps is
    within the 1e-2 gate of the CPU oracle on the merged weights, while the LoRA moves eps by far more than the gate,
    and the captured step has the base engine's launch count."""
import os
import shutil

import numpy as np
import pytest
import torch

from editanything_b200 import lora as L
from editanything_b200 import weights as W
from editanything_b200.denoise import DenoiseEngine, ddim_schedule
from editanything_b200.unet_spec import SD15, build_topology, make_state_dict
from oracle import unet_oracle as O
from oracle.inputs import make_inputs
from tests import synth_lora as SL
from tests.test_lora_cpu import BASE, _model_root, _reenact

pytestmark = pytest.mark.gpu
EPS_TOL = 1e-2


def _premerged_root(root, lora_path, multiplier):
    """A copy of the base model directory with the LoRA merged into its UNet and text encoder files."""
    from safetensors.torch import load_file, save_file
    src = os.path.join(root, *BASE.split("/"))
    dst = os.path.join(root, "premerged", "sd15")
    shutil.copytree(src, dst)
    ufile = os.path.join(dst, "unet", "diffusion_pytorch_model.safetensors")
    usd = load_file(ufile)
    te = SL.text_encoder_fp16(src)
    te_sd = te.state_dict()
    for layer, e in L.read_lora(lora_path).items():
        target, _ = L.layer_tokens(layer)
        path = layer[len("lora_unet_" if target == "unet" else "lora_te_"):]
        sd = usd if target == "unet" else te_sd
        key = next(k for k in sd if k.replace(".", "_") == path + "_weight")
        base16 = sd[key].to(torch.float16)
        merged = _reenact(base16, e["lora_up.weight"], e["lora_down.weight"], float(e["alpha"]), multiplier)
        if target == "unet":
            usd[key] = merged
        else:
            te_sd[key].copy_(merged)
    save_file({k: v.contiguous() for k, v in usd.items()}, ufile)
    shutil.rmtree(os.path.join(dst, "text_encoder"))
    te.save_pretrained(os.path.join(dst, "text_encoder"))
    return dst


def _request(output_type):
    """A 64x64 inpainting request with a text prompt (so the text encoder's merge counts) and two control images."""
    from PIL import Image
    g = np.random.RandomState(0)
    image = Image.fromarray(g.randint(0, 256, (64, 64, 3)).astype(np.uint8))
    mask = np.zeros((64, 64), dtype=np.uint8)
    mask[16:48, 8:40] = 255
    tg = torch.Generator().manual_seed(1)
    conds = [torch.rand(1, 3, 64, 64, generator=tg) * 255, torch.rand(1, 3, 64, 64, generator=tg)]
    return dict(prompt="a photo of a cat", negative_prompt="lowres", image=image, mask_image=Image.fromarray(mask),
                controlnet_conditioning_image=conds, height=64, width=64, num_inference_steps=5, guidance_scale=9.0,
                generator=torch.manual_seed(3), controlnet_conditioning_scale=[0.5, 1.0], output_type=output_type)


def test_lora_pipeline_equals_premerged_checkpoint(tmp_path, monkeypatch):
    from editanything_b200.loading import ControlNetModel, ControlNetModel2
    from editanything_b200.pipeline import StableDiffusionControlNetInpaintPipeline as Pipe
    root = str(tmp_path)
    _, _, a, _ = _model_root(root)
    monkeypatch.setenv("EA_MODEL_ROOT", root)
    cn = [ControlNetModel2.from_pretrained("shgao/edit-anything-v0-4-sd15"),
          ControlNetModel.from_pretrained("lllyasviel/control_v11p_sd15_inpaint")]
    lora = Pipe.from_pretrained(BASE, controlnet=cn, lora=[(a, 0.5)])
    pre = Pipe.from_pretrained(_premerged_root(root, a, 0.5), controlnet=cn)
    plain = Pipe.from_pretrained(BASE, controlnet=cn)
    assert lora.engine.dev.type == "cuda"
    outs = {}
    for name, p in (("lora", lora), ("pre", pre), ("plain", plain)):
        res = {}
        for ot in ("latent", "np"):
            res[ot] = p(**_request(ot)).images
        outs[name] = res
    lat, img = outs["lora"]["latent"], outs["lora"]["np"]
    assert torch.equal(lat, outs["pre"]["latent"]) and np.array_equal(img, outs["pre"]["np"])
    assert not torch.equal(lat, outs["plain"]["latent"])


def _sd15_lora(path, rank=64):
    """A rank-64 LoRA on every LoRA-able layer of the SD1.5 UNet, sized so that at multiplier 0.5 each delta is
    about a tenth of the layer's weights."""
    shapes = SL.unet_diffusers_shapes(SD15)
    g = torch.Generator().manual_seed(64)
    t = {}
    for p in SL.unet_targets(shapes):
        s = shapes[p + ".weight"]
        up = torch.randn(s[0], rank, generator=g) * 0.025
        down = torch.randn(rank, s[1], generator=g) / s[1] ** 0.5
        if len(s) == 4:
            up, down = up[:, :, None, None], down[:, :, None, None]
        name = SL.kohya_name(p, "unet")
        t[name + ".lora_up.weight"] = up.half()
        t[name + ".lora_down.weight"] = down.half()
        t[name + ".alpha"] = torch.tensor(float(rank), dtype=torch.float16)
    return SL.save(t, path)


def _launches(eng, x):
    ts, a, ap = ddim_schedule(50)
    eng.set_schedule([int(t) for t in ts[:2]], list(a[:2]), list(ap[:2]))
    eng.begin(x[:1, :4], guidance=7.5)
    eng.step()
    torch.cuda.synchronize()
    return eng.launches_per_step


def test_sd15_512_rank64_lora_vs_cpu_oracle(tmp_path):
    cfg = SD15
    base = make_state_dict(cfg, "unet", 81)
    km = W.key_map(cfg, "unet", base.keys())
    dsd = {km[k]: v for k, v in base.items()}
    path = _sd15_lora(str(tmp_path / "rank64.safetensors"))
    L.merge([(path, 0.5)], unet_sd=dsd)
    merged = W.diffusers_to_ldm(dsd, "unet", cfg)
    del dsd
    csds = [make_state_dict(cfg, "controlnet", 82 + i) for i in range(2)]
    x, ctx, hints = make_inputs(cfg, 2, 64, 77, 6, n_controlnets=2)
    scales = [0.5, 1.0]
    dev = torch.device("cuda:0")
    eng = DenoiseEngine(cfg, merged, csds, dev)
    eng.prepare(ctx, hints, scales)
    plain = DenoiseEngine(cfg, base, csds, dev)
    plain.prepare(ctx, hints, scales)
    t = 501
    eps = eng.eps(x, t).cpu()
    eps_plain = plain.eps(x, t).cpu()
    with torch.no_grad():
        ref = O.apply_model({k: v.float() for k, v in merged.items()}, build_topology(cfg),
                            [(sd, build_topology(cfg, with_decoder=False)) for sd in csds], x, torch.full((2,), t),
                            ctx, hints, scales)
    err = (eps - ref).abs().max().item()
    moved = (eps - eps_plain).abs().max().item()
    print(f"sd15_512 rank-64 LoRA x0.5: eps max-abs vs oracle {err:.3e}, LoRA - base {moved:.3e}")
    assert err < EPS_TOL, err
    assert moved > 20 * EPS_TOL, moved
    n_lora, n_plain = _launches(eng, x), _launches(plain, x)
    assert n_lora == n_plain and n_lora > 100, (n_lora, n_plain)
