"""Re-enactment of the reference pipeline's 9-channel (inpainting UNet) branch on the CPU oracle networks (test
infrastructure), shared by tests/test_inpaint9_cpu.py and tests/test_gpu_inpaint9.py.

utils/stable_diffusion_controlnet_inpaint.py: masked image (:1396), mask latents (:1016-1054), masked-image latents
(:1056-1105) drawn after the initial noise (:1440-1468), per-step UNet input cat([x, mask, masked latents]) with the
ControlNets on x alone (:1550-1560, :1607-1624), no blend and no paste-back (:1647, :1658)."""
from types import SimpleNamespace

import torch
import torch.nn.functional as F

from editanything_b200.pipeline import DDIMScheduler
from editanything_b200.unet_spec import build_topology, controlnet_config
from oracle import unet_oracle as O


class RecordingVAE:
    """The diffusers AutoencoderKL surface the pipeline touches; records what it encodes and draws its latent
    sample from the generator it is given (so the order of the pipeline's random draws is checked)."""
    config = SimpleNamespace(scaling_factor=0.18215, latent_channels=4, block_out_channels=(1, 2, 3, 4))

    def __init__(self):
        self.seen = []

    def encode(self, x):
        self.seen.append(x.detach().cpu().clone())
        z = F.avg_pool2d(x.cpu().float(), 8)
        z = torch.cat([z, z.mean(1, keepdim=True)], 1)

        def sample(generator=None):
            return z + 0.1 * torch.randn(z.shape, generator=generator)
        return SimpleNamespace(latent_dist=SimpleNamespace(sample=sample))

    def decode(self, z):
        return SimpleNamespace(sample=F.interpolate(z[:, :3], scale_factor=8, mode="nearest"))


def apply_model_9ch(usd, cfg, csds, x9, t, ctx, hints, scales):
    """ControlNets on x9[:, :4], the UNet on all 9 channels (the reference's own modules do the same in
    oracle/make_golden_inpaint.py)."""
    ut, ct = build_topology(cfg), build_topology(controlnet_config(cfg), with_decoder=False)
    tt = torch.full((x9.shape[0],), int(t))
    control = None
    for sd, hint, s in zip(csds, hints, scales):
        outs = [o * s for o in O.controlnet_forward(sd, ct, x9[:, :4], hint, tt, ctx)]
        control = outs if control is None else [a + b for a, b in zip(control, outs)]
    return O.unet_forward(usd, ut, x9, tt, ctx, control)


def reference_loop_9ch(cfg, usd, csds, image, mask, conds, pe, ne, *, steps, gs, scales, seed, n_img=1,
                       scheduler=None, pre=None):
    """Final latents of the reference __call__ (in_channels == 9) with `scheduler` (default DDIM); `pre`, when a
    list, receives the latents every callback would see."""
    vae = RecordingVAE()
    sch = scheduler if scheduler is not None else DDIMScheduler()
    sch.set_timesteps(steps)
    gen = torch.manual_seed(seed)
    H, W = image.shape[2], image.shape[3]
    h, w = H // 8, W // 8
    lat = torch.randn((n_img, 4, h, w), generator=gen)                                  # prepare_latents
    mbin = (mask >= 0.5).float()
    masked = image * (mbin < 0.5)
    mask_lat = F.interpolate(mbin, size=(h, w)).repeat(n_img, 1, 1, 1)
    masked_lat = (0.18215 * vae.encode(masked).latent_dist.sample(generator=gen)).repeat(n_img, 1, 1, 1)
    cond = torch.cat([torch.cat([mask_lat] * 2), torch.cat([masked_lat] * 2)], 1)
    ctx = torch.cat([ne.repeat(n_img, 1, 1), pe.repeat(n_img, 1, 1)])
    hints = [torch.cat([c.repeat_interleave(n_img, 0)] * 2) for c in conds]
    for t in sch.timesteps:
        x9 = torch.cat([torch.cat([lat] * 2), cond], 1)
        with torch.no_grad():
            e = apply_model_9ch(usd, cfg, csds, x9, t, ctx, hints, scales)
        lat = sch.step(e[:n_img] + gs * (e[n_img:] - e[:n_img]), t, lat).prev_sample
        if pre is not None:
            pre.append(lat.clone())
    return lat, masked
