"""Generate tests/golden/vae_*.pt by RUNNING the reference's own Decoder
(ldm/modules/diffusionmodules/model.py:546-652, imported from /root/reference; build container only).

    python -m oracle.make_golden_vae [--full]

Weights are the deterministic synthetic ones of editanything_b200.vae_spec.make_vae_state_dict; latents
are seeded N(0,1) scaled like the sampler's output.  The stored tensor is decode_latents' image
((x / 2 + 0.5).clamp(0, 1), utils/stable_diffusion_controlnet_inpaint.py:718-722)."""
import os
import sys

import torch

from oracle.make_golden import golden_sample

from editanything_b200.vae_spec import SD_VAE, VAE_TINY, make_vae_state_dict
from oracle import vae_oracle as V

GOLD = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
CASES = {"vae_tiny": (VAE_TINY, 2, 16, 401, 7)}          # name -> (cfg, batch, latent side, weight seed, latent seed)
FULL_CASES = {"vae_sd": (SD_VAE, 1, 64, 402, 8)}


def make_latents(cfg, B, side, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, cfg.z_channels, side, side, generator=g) * cfg.scaling_factor * 4.0


def run_case(name, spec):
    cfg, B, side, wseed, lseed = spec
    sd = make_vae_state_dict(cfg, wseed)
    lat = make_latents(cfg, B, side, lseed)
    ref = V.reference_decoder(cfg, sd)
    raw = ref(lat / cfg.scaling_factor)
    img = (raw / 2 + 0.5).clamp(0, 1)
    rec = {"meta": dict(name=name, B=B, side=side, weight_seed=wseed, latent_seed=lseed,
                        generator="reference ldm Decoder + post_quant_conv", raw_abs_max=float(raw.abs().max()),
                        raw_std=float(raw.std())),
           "image": img.to(torch.float16) if side >= 64 else img.clone(),
           "raw_center": raw[:, :, raw.shape[2] // 2 - 8:raw.shape[2] // 2 + 8, raw.shape[3] // 2 - 8:raw.shape[3] // 2 + 8].clone()}
    if side >= 64:   # files stay below 1 MB: a fixed, seeded sample of half of the image rows
        idx = golden_sample(rec["image"].shape[2], rec["image"].shape[2] // 2, 512)
        rec["image"] = rec["image"].index_select(2, idx).clone()
        rec["image_index"] = (2, idx)
    torch.save(rec, os.path.join(GOLD, name + ".pt"))
    print(name, tuple(img.shape), "raw abs max", float(raw.abs().max()), "raw std", float(raw.std()),
          "fraction clamped", float(((raw / 2 + 0.5) < 0).float().mean() + ((raw / 2 + 0.5) > 1).float().mean()))


ENC_CASES = {"vae_enc_tiny": (VAE_TINY, 2, 32, 411, 17)}     # name -> (cfg, batch, image side, weight seed, image seed)
ENC_FULL_CASES = {"vae_enc_sd": (SD_VAE, 1, 512, 412, 18)}


def make_image(B, side, seed):
    """A masked source image as prepare_masked_image_latents sees it: [-1, 1] pixels, a masked block zeroed."""
    g = torch.Generator().manual_seed(seed)
    img = torch.rand(B, 3, side, side, generator=g) * 2 - 1
    img[:, :, side // 4:side // 2, side // 4:side // 2] = 0.0
    return img


def run_enc_case(name, spec):
    cfg, B, side, wseed, iseed = spec
    sd = make_vae_state_dict(cfg, wseed, part="encoder")
    m = V.reference_encoder(cfg, sd)(make_image(B, side, iseed))
    rec = {"meta": dict(name=name, B=B, side=side, weight_seed=wseed, image_seed=iseed,
                        generator="reference ldm Encoder + quant_conv"), "moments": m.clone()}
    torch.save(rec, os.path.join(GOLD, name + ".pt"))
    print(name, tuple(m.shape), "mean abs max", float(m[:, :m.shape[1] // 2].abs().max()), "logvar range",
          float(m[:, m.shape[1] // 2:].min()), float(m[:, m.shape[1] // 2:].max()))


if __name__ == "__main__":
    os.makedirs(GOLD, exist_ok=True)
    torch.set_num_threads(os.cpu_count())
    for n, s in (FULL_CASES if "--full" in sys.argv else CASES).items():
        run_case(n, s)
    for n, s in (ENC_FULL_CASES if "--full" in sys.argv else ENC_CASES).items():
        run_enc_case(n, s)
