"""Synthetic kohya-format LoRA files (test infrastructure) and the fixtures their merge is checked on.

Layer names are the kohya spelling of a diffusers module path: "lora_unet_" / "lora_te_" + the path with "." -> "_".
By default the factors are small dyadic rationals k/64 (|k| <= 8, rank <= 8) stored as fp16: every product and sum
of `up @ down` is exact in fp32 whatever the summation order, so the merged weights do not depend on the BLAS."""
import hashlib
import os

import torch
from torch import nn

from editanything_b200 import weights as W
from editanything_b200.unet_spec import TINY, TINY21, make_state_dict, param_shapes

UNET_SEED = 51               # the base UNet of synth_ckpt.write_pipeline(..., seed=51)
UNET_KINDS = ("attn1.to_q", "attn1.to_k", "attn1.to_v", "attn1.to_out.0", "attn2.to_q", "attn2.to_k", "attn2.to_v",
              "attn2.to_out.0", "ff.net.0.proj", "ff.net.2", "proj_in", "proj_out", "time_emb_proj", "conv_shortcut")
TE_KINDS = ("self_attn.q_proj", "self_attn.k_proj", "self_attn.v_proj", "self_attn.out_proj", "mlp.fc1", "mlp.fc2")

# name: (UNet config, [(seed, rank, alpha, targets "unet" / "te" / "both")], multiplier)
CASES = {
    "tiny_unet": (TINY, [(1, 8, 4.0, "unet")], 1.0),
    "tiny21_unet": (TINY21, [(2, 4, 2.0, "unet")], 1.0),
    "tiny_text_encoder": (TINY, [(3, 8, 8.0, "te")], 1.0),
    "tiny_alpha0": (TINY, [(4, 4, 0.0, "both")], 1.0),
    "tiny_mult_half": (TINY, [(5, 8, 4.0, "both")], 0.5),
    "tiny_two_files": (TINY, [(6, 8, 4.0, "both"), (7, 2, 1.0, "both")], 1.0),
}


def unet_diffusers_shapes(cfg):
    """{diffusers parameter name: shape} of a UNet2DConditionModel with this config."""
    shapes = param_shapes(cfg, "unet")
    km = W.key_map(cfg, "unet", shapes.keys())
    return {km[k]: s for k, (s, _) in shapes.items()}


def unet_diffusers_state_dict(cfg, seed=UNET_SEED):
    """The diffusers-keyed fp32 UNet that synth_ckpt.write_unet_like writes for this config and seed."""
    sd = make_state_dict(cfg, "unet", seed)
    km = W.key_map(cfg, "unet", sd.keys())
    return {km[k]: v for k, v in sd.items()}


def unet_targets(keys):
    """The diffusers module paths of every LoRA-able UNet layer among parameter names `keys`."""
    return [k[:-len(".weight")] for k in keys if k.endswith(".weight") and any(k[:-len(".weight")].endswith("." + t)
                                                                               for t in UNET_KINDS)]


def te_targets(keys):
    return [k[:-len(".weight")] for k in keys if k.endswith(".weight") and any(k[:-len(".weight")].endswith("." + t)
                                                                               for t in TE_KINDS)]


def kohya_name(path, target):
    return ("lora_unet_" if target == "unet" else "lora_te_") + path.replace(".", "_")


def factors(weight_shape, rank, g, dyadic=True):
    """(up, down) for a weight of this shape (Linear or 1x1 conv)."""
    out, inp = weight_shape[0], weight_shape[1]
    conv = len(weight_shape) == 4
    if dyadic:
        up = torch.randint(-8, 9, (out, rank), generator=g).to(torch.float16) / 64
        down = torch.randint(-8, 9, (rank, inp), generator=g).to(torch.float16) / 64
    else:
        up = torch.randn(out, rank, generator=g) * 0.1
        down = torch.randn(rank, inp, generator=g) * 0.1
    if conv:
        up, down = up[:, :, None, None], down[:, :, None, None]
    return up.contiguous(), down.contiguous()


def lora_tensors(targets, rank, alpha, seed, dyadic=True):
    """{kohya key: tensor} for targets {(target, diffusers path): weight shape}."""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for (target, path), shape in targets.items():
        name = kohya_name(path, target)
        up, down = factors(shape, rank, g, dyadic)
        out[name + ".lora_up.weight"], out[name + ".lora_down.weight"] = up, down
        out[name + ".alpha"] = torch.tensor(float(alpha), dtype=torch.float16 if dyadic else torch.float32)
    return out


def save(tensors, path):
    from safetensors.torch import save_file
    os.makedirs(os.path.dirname(path), exist_ok=True)
    save_file({k: v.contiguous() for k, v in tensors.items()}, path)
    return path


def case_targets(cfg, which, te_shapes):
    """{(target, path): shape} of a case's file: the UNet's LoRA-able layers, the text encoder's, or both."""
    t = {}
    if which in ("unet", "both"):
        us = unet_diffusers_shapes(cfg)
        t.update({("unet", p): us[p + ".weight"] for p in unet_targets(us)})
    if which in ("te", "both"):
        t.update({("te", p): te_shapes[p + ".weight"] for p in te_targets(te_shapes)})
    return t


def write_case(name, dirpath, te_shapes):
    """Write one case's LoRA files under dirpath; returns ([paths], multiplier, cfg)."""
    cfg, files, mult = CASES[name]
    paths = []
    for i, (seed, rank, alpha, which) in enumerate(files):
        paths.append(save(lora_tensors(case_targets(cfg, which, te_shapes), rank, alpha, seed),
                          os.path.join(dirpath, f"{name}_{i}.safetensors")))
    return paths, mult, cfg


def text_encoder_fp16(root):
    """The tiny CLIP text encoder of synth_ckpt.write_pipeline's directory `root`, loaded in fp16 like
    `from_pretrained(torch_dtype=torch.float16)`."""
    from transformers import CLIPTextModel
    return CLIPTextModel.from_pretrained(os.path.join(root, "text_encoder"), torch_dtype=torch.float16).eval()


def module_tree(sd):
    """An nn.Module tree whose parameters are `sd` (dotted names): what `nn.Module.__getattr__` walks on a
    UNet2DConditionModel with these weights."""
    root = nn.Module()
    for k, v in sd.items():
        *path, leaf = k.split(".")
        m = root
        for p in path:
            if p not in m._modules:
                m.add_module(p, nn.Module())
            m = m._modules[p]
        m.register_parameter(leaf, nn.Parameter(v.detach().clone(), requires_grad=False))
    return root


def fingerprint(t):
    t = t.detach().cpu().contiguous()
    return f"{t.dtype}:{tuple(t.shape)}:" + hashlib.sha256(t.view(torch.uint8).numpy().tobytes()).hexdigest()
