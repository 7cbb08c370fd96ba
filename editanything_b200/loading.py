"""Checkpoint loading behind the reference's constructors (SURVEY.md §8b row B2):

    ControlNetModel2.from_pretrained(controlnet_path, torch_dtype=torch.float16)               editany_lora.py:352-355
    ControlNetModel.from_pretrained("lllyasviel/control_v11p_sd15_inpaint", torch_dtype=...)   editany_lora.py:359-362
    StableDiffusionControlNetInpaintPipeline.from_pretrained(base, controlnet=[...], torch_dtype=..., safety_checker=None)
                                                                                               editany_lora.py:372-377

Checkpoints are diffusers-layout DIRECTORIES (model_index.json, unet/, vae/, text_encoder/, tokenizer/, scheduler/;
a ControlNet is config.json + diffusion_pytorch_model.{safetensors,bin}).  There is no network on the deployment
boxes: hub ids resolve through $EA_MODEL_ROOT/<org>/<name>, $EA_MODEL_ROOT/<org>--<name> or the local HF cache
(models--<org>--<name>/snapshots/*).  The weights are re-keyed to the ldm/cldm names (editanything_b200.weights)
and packed into the H100 engines; text encoder and tokenizer come from `transformers`.
"""
import glob
import json
import os
from types import SimpleNamespace

import torch

from .unet_spec import UNetConfig


def resolve_model_path(name_or_path):
    if os.path.isdir(name_or_path):
        return name_or_path
    roots = [r for r in (os.environ.get("EA_MODEL_ROOT"), os.path.join(os.getcwd(), "models")) if r]
    cands = []
    for r in roots:
        cands += [os.path.join(r, name_or_path), os.path.join(r, name_or_path.replace("/", "--"))]
    hub = os.environ.get("HF_HUB_CACHE") or os.path.join(os.environ.get("HF_HOME", os.path.expanduser("~/.cache/huggingface")), "hub")
    cands += sorted(glob.glob(os.path.join(hub, "models--" + name_or_path.replace("/", "--"), "snapshots", "*")))
    for c in cands:
        if os.path.isdir(c):
            return c
    raise FileNotFoundError(f"checkpoint '{name_or_path}' not found locally (no network here): looked in {cands}; "
                            "set EA_MODEL_ROOT to the directory that holds the diffusers-layout checkpoints")


def load_weights(dirpath, stems=("diffusion_pytorch_model", "model", "pytorch_model")):
    """{name: tensor} from <dir>/<stem>.safetensors (preferred) or <stem>.bin; fp16 variants accepted."""
    for stem in stems:
        for var in ("", ".fp16"):
            p = os.path.join(dirpath, stem + var + ".safetensors")
            if os.path.exists(p):
                from safetensors.torch import load_file
                return load_file(p)
            p = os.path.join(dirpath, stem + var + ".bin")
            if os.path.exists(p):
                return torch.load(p, map_location="cpu", weights_only=True)
    raise FileNotFoundError(f"no weight file ({'/'.join(stems)}.safetensors|.bin) in {dirpath}")


def _read_json(path):
    with open(path) as f:
        return json.load(f)


def unet_config_from_diffusers(c):
    """diffusers UNet2DConditionModel / ControlNetModel config.json -> UNetConfig.  `attention_head_dim` is the
    number of heads when an int (SD1.x: 8) and the per-level head counts when a list (SD2.x: [5, 10, 20, 20], i.e.
    64-wide heads) - SURVEY.md Appendix B."""
    boc = list(c["block_out_channels"])
    mc = boc[0]
    ahd = c.get("attention_head_dim", 8)
    kw = dict(in_channels=c.get("in_channels", 4), model_channels=mc, num_res_blocks=c.get("layers_per_block", 2),
              channel_mult=tuple(b // mc for b in boc), context_dim=c.get("cross_attention_dim", 768),
              use_linear_in_transformer=bool(c.get("use_linear_projection", False)))
    if "out_channels" in c:
        kw["out_channels"] = c["out_channels"]
    if isinstance(ahd, (list, tuple)):
        kw["num_head_channels"] = mc // int(ahd[0])
    else:
        kw["num_heads"] = int(ahd)
    # attention at every level but the last (CrossAttnDownBlock2D x3 + DownBlock2D)
    types = c.get("down_block_types")
    if types is not None:
        kw["attention_resolutions"] = tuple(sorted((2 ** i for i, t in enumerate(types) if "CrossAttn" in t), reverse=True))
    return UNetConfig(**kw)


class ControlNetModel:
    """What the reference holds in `controlnet=[...]`: a loaded ControlNet checkpoint (config + ldm-keyed weights).
    The network itself runs inside DenoiseEngine; this object carries the weights there."""

    def __init__(self, cfg: UNetConfig, state_dict_ldm, config=None, dtype=torch.float16):
        self.cfg, self.state_dict_ldm, self.dtype = cfg, state_dict_ldm, dtype
        self.config = SimpleNamespace(**(config or {}))

    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path, torch_dtype=None, subfolder=None, **_unused):
        from .weights import diffusers_to_ldm
        root = resolve_model_path(pretrained_model_name_or_path)
        if subfolder:
            root = os.path.join(root, subfolder)
        c = _read_json(os.path.join(root, "config.json"))
        cfg = unet_config_from_diffusers(c)
        sd = diffusers_to_ldm(load_weights(root), "controlnet", cfg)
        return cls(cfg, sd, c, torch_dtype or torch.float16)

    def to(self, *a, **k):
        return self


class ControlNetModel2(ControlNetModel):
    """utils/stable_diffusion_controlnet.py:ControlNetModel2 - the reference's ControlNet variant whose forward also
    accepts a spatial `conditioning_scale` map (:777-802); same checkpoint format."""


def vae_config_from_diffusers(c):
    from .vae_spec import VaeConfig
    boc = list(c.get("block_out_channels", [128, 256, 512, 512]))
    return VaeConfig(ch=boc[0], ch_mult=tuple(b // boc[0] for b in boc), num_res_blocks=c.get("layers_per_block", 2),
                     z_channels=c.get("latent_channels", 4), embed_dim=c.get("latent_channels", 4),
                     scaling_factor=c.get("scaling_factor", 0.18215), out_ch=c.get("out_channels", 3))


def load_pipeline_parts(base_model_path, device, *, text_encoder=None, tokenizer=None, vae=None, scheduler=None,
                        unet_packed=None, lora=(), merge_text_encoder=True):
    """Everything `StableDiffusionControlNetInpaintPipeline.from_pretrained` needs from the base checkpoint:
    (cfg, unet ldm state dict or None when `unet_packed` is shared, vae engine, text_encoder, tokenizer, scheduler).
    lora: [(path, multiplier), ...] merged (editanything_b200.lora) into the diffusers UNet state dict it loads,
    before the ldm re-keying and any packing, and with `merge_text_encoder` into the text encoder in place
    (editany_lora.py:378-381).  Every entry is checked before any weight changes."""
    from . import lora as L
    from .pipeline import DDIMScheduler
    from .vae import VaeEngine
    from .weights import diffusers_to_ldm, vae_diffusers_to_ldm
    root = resolve_model_path(base_model_path)
    ucfg = unet_config_from_diffusers(_read_json(os.path.join(root, "unet", "config.json")))
    if scheduler is None:
        # read before any weight: a prediction type the sampler cannot run ("sample", or anything unknown) raises
        # here rather than when sampling.  SD2.1-768 sets "v_prediction".
        sp = os.path.join(root, "scheduler", "scheduler_config.json")
        sc = _read_json(sp) if os.path.exists(sp) else {}
        scheduler = DDIMScheduler(sc.get("beta_start", 0.00085), sc.get("beta_end", 0.012),
                                  sc.get("num_train_timesteps", 1000), sc.get("prediction_type", "epsilon"))
    usd = None
    if unet_packed is None:
        usd = load_weights(os.path.join(root, "unet"))
    if vae is None:
        vcfg = vae_config_from_diffusers(_read_json(os.path.join(root, "vae", "config.json")))
        vsd = vae_diffusers_to_ldm(load_weights(os.path.join(root, "vae")), vcfg, parts=("decoder", "encoder"))
        vae = VaeEngine(vcfg, vsd, device)
    if text_encoder is None or tokenizer is None:
        from transformers import CLIPTextModel, CLIPTokenizer
        if tokenizer is None:
            tokenizer = CLIPTokenizer.from_pretrained(os.path.join(root, "tokenizer"))
        if text_encoder is None:
            text_encoder = CLIPTextModel.from_pretrained(os.path.join(root, "text_encoder"), torch_dtype=torch.float16)
            text_encoder = text_encoder.to(device).eval()
    L.merge(lora, unet_sd=usd, text_encoder=text_encoder if merge_text_encoder else None)
    if usd is not None:
        usd = diffusers_to_ldm(usd, "unet", ucfg)
    return ucfg, usd, vae, text_encoder, tokenizer, scheduler
