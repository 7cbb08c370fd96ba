"""Restatement of the alpha-mixing inpaint pipeline (utils/stable_diffusion_controlnet_inpaint.py:1706-2092, 4-channel
branch) for the tests - TEST INFRASTRUCTURE.  The latents, the scheduler update, the start blend and every mix are
computed in float64; the networks are the float32 CPU oracle (oracle/unet_oracle.py), whose output is widened.

Random draws follow the reference: the latents from `generator`, then randn_like(init) on the global CPU generator
once for the start (:1975) and once per step i < S - 1 (:2041), in that order."""
import torch
import torch.nn.functional as F

from editanything_b200.pipeline import DDIMScheduler, randn_tensor
from editanything_b200.unet_spec import build_topology
from oracle import unet_oracle as O


def mix_ref(x, known, mask, noise, k_init, k_noise, in_window, alpha):
    """ea_latent_mix in float64 for one active row: x / known / noise [..., 4] (or any layout where `mask`
    broadcasts), mask 1 = keep."""
    x, known, noise, mask = (t.double() for t in (x, known, noise, mask))
    p = k_init * known + k_noise * noise
    keep = p if in_window else x
    return keep * mask + ((1 - alpha) * x + alpha * p) * (1 - mask)


def reference_mixing(cfg, usd, csds, image, mask, conds, pe, ne, *, steps, gs, scales, seed, alpha, ratio, vae,
                     n_img=1, scheduler=None, seen=None):
    """Final latents (float64) of the mixing pipeline's __call__ with `scheduler` (default DDIM).  image [1, 3, H, W]
    in [-1, 1]; mask [1, 1, H, W] (1 = repaint); conds: one [1, 3, H, W] hint per net; scales: one float or map
    (already multiplied by the scale map, :1874-1880) per net; `seen`, when a list, receives the latents after every
    scheduler step, before the mix - what a callback sees."""
    sch = scheduler if scheduler is not None else DDIMScheduler()
    sch.set_timesteps(steps)
    ts = sch.timesteps
    S = len(ts)
    do_cfg = gs > 1.0
    gen = torch.manual_seed(seed)                                          # the global CPU generator, as the pipeline
    H, W = image.shape[2], image.shape[3]
    lat = randn_tensor((n_img, 4, H // 8, W // 8), generator=gen).double()
    init = (vae.config.scaling_factor * vae.encode(image).latent_dist.sample(generator=gen)).repeat(n_img, 1, 1, 1)
    m = 1 - F.interpolate((mask >= 0.5).float(), (H // 8, W // 8), mode="nearest").double()      # 1 = keep
    lat = m * sch.add_noise(init.double(), torch.randn_like(init).double(), ts[0]) + (1 - m) * lat   # :1965-1977
    rows = 2 * n_img if do_cfg else n_img
    ctx = torch.cat([ne.repeat(n_img, 1, 1), pe.repeat(n_img, 1, 1)]) if do_cfg else pe.repeat(n_img, 1, 1)
    hints = [c.repeat_interleave(n_img, 0) for c in conds]
    hints = [torch.cat([h, h]) for h in hints] if do_cfg else hints
    ut, ct = build_topology(cfg), build_topology(cfg, with_decoder=False)
    for i, t in enumerate(ts):
        x_in = sch.scale_model_input(torch.cat([lat] * 2) if do_cfg else lat, t)
        with torch.no_grad():
            e = O.apply_model(usd, ut, [(sd, ct) for sd in csds], x_in.float(), torch.full((rows,), int(t)), ctx,
                              hints, scales).double()
        if do_cfg:
            e = e[:n_img] + gs * (e[n_img:] - e[:n_img])
        lat = sch.step(e, t, lat).prev_sample
        if seen is not None:
            seen.append(lat.clone())
        if i < S - 1:                                                      # :2039-2051
            p = sch.add_noise(init.double(), torch.randn_like(init).double(), ts[i + 1])
            if i < S * ratio:
                lat = p * m + ((1 - alpha) * lat + alpha * p) * (1 - m)
            else:
                lat = lat * m + ((1 - alpha) * lat + alpha * p) * (1 - m)
    return lat
