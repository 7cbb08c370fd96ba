"""Generate tests/golden/*.pt by running the REFERENCE's own modules (build container only).

    python -m oracle.make_golden [--full]

Golden vectors are produced by the unmodified reference code under /root/reference
(cldm.cldm.ControlNet / ControlledUnetModel, cldm.ddim_hacked / ldm DDIM schedule helpers) with
the deterministic synthetic weights of editanything_b200.unet_spec.make_state_dict.  They pin the
oracle restatement (oracle/unet_oracle.py) and the CUDA path on machines where /root/reference
does not exist.
"""
import os
import sys

import numpy as np
import torch

from editanything_b200.unet_spec import SD15, SD21, TINY, TINY21, make_state_dict
from oracle import ref_shim
from oracle.inputs import make_inputs

GOLD = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")

# name -> (cfg, batch, latent side, ctx len, timesteps, controlnet seeds, scales, input seed)
CASES = {
    "tiny_sd15": (TINY, 2, 16, 13, [981, 1], (102, 103), [0.5, 1.0], 7),
    "tiny_sd21": (TINY21, 2, 16, 20, [501], (102,), [1.0], 8),
    "tiny_sd15_32": (TINY, 2, 32, 77, [741], (102, 103), [0.5, 1.0], 9),
}
FULL_CASES = {
    # BASELINE.json configs[1] shapes: SD1.5 512x512, N=1 + CFG -> B=2, 64x64 latents, L=77; three timesteps
    # of the 50-step DDIM table (first, middle, last)
    "sd15_512": (SD15, 2, 64, 77, [981, 501, 1], (102, 103), [0.5, 1.0], 11),
    # configs[2]: SD2.1 (models/cldm_v21.yaml:21-55) 768x768, N=4 + CFG -> B=8, 96x96 latents, 1 ControlNet
    "sd21_768": (SD21, 8, 96, 77, [501], (102,), [1.0], 12),
    # configs[3]: SD1.5 512x512, 4 images per GPU + CFG -> B=8, SAM + inpaint ControlNets
    "sd15_512_b8": (SD15, 8, 64, 77, [741], (102, 103), [0.5, 1.0], 13),
    # configs[4]: SD1.5 1024x1024 tile refinement (128x128 latents, 16384 tokens), N=1 + CFG, tile ControlNet
    "sd15_1024": (SD15, 2, 128, 77, [961], (102,), [1.0], 14),
}
# Every row of the batch is independent in the reference networks (GroupNorm is per sample, attention per
# sample); the big cases are therefore evaluated `chunk` rows at a time - the reference's fp32 attention
# materialises [rows*heads, T, T] logits (8.6 GB per row at 16384 tokens).
CHUNK = {"sd21_768": 2, "sd15_1024": 1, "sd15_512_b8": 4}
SAMPLE = {"sd21_768": 4}      # batch rows kept of the full-size eps


def golden_sample(n, k, seed):
    """k of n indices, sorted, the same on every run."""
    return torch.randperm(n, generator=torch.Generator().manual_seed(seed))[:k].sort().values
UNET_SEED = 101


def run_case(name, spec):
    cfg, B, lat, L, ts, cn_seeds, scales, in_seed = spec
    usd = make_state_dict(cfg, "unet", UNET_SEED)
    csds = [make_state_dict(cfg, "controlnet", s) for s in cn_seeds]
    unet, cns = ref_shim.build_reference_nets(cfg, usd, csds)
    x, ctx, hints = make_inputs(cfg, B, lat, L, in_seed, n_controlnets=len(cn_seeds))
    out = {"meta": dict(name=name, B=B, lat=lat, L=L, timesteps=ts, cn_seeds=list(cn_seeds), scales=scales,
                        in_seed=in_seed, unet_seed=UNET_SEED)}
    chunk = CHUNK.get(name, B)
    for t in ts:
        eps_rows, control = [], None
        for b0 in range(0, B, chunk):
            sl = slice(b0, b0 + chunk)
            tt = torch.full((x[sl].shape[0],), t, dtype=torch.long)
            e, c = ref_shim.reference_apply_model(unet, cns, x[sl], tt, ctx[sl], [h[sl] for h in hints], scales)
            eps_rows.append(e.clone())
            control = c if control is None else [torch.cat([a, b_]) for a, b_ in zip(control, c)]
        eps = torch.cat(eps_rows)
        out[f"eps_t{t}"] = eps.clone()
        # the summed, scaled control residuals (what the UNet decoder consumes): keep two of the 13
        if cfg.model_channels <= 64:
            out[f"control0_t{t}"] = control[0].clone().to(torch.float16)
        if name in SAMPLE:   # files stay below 1 MB: a fixed, seeded sample of the batch rows (and its index)
            idx = golden_sample(eps.shape[0], SAMPLE[name], 768)
            out[f"eps_t{t}"] = eps.index_select(0, idx).clone()
            out[f"eps_t{t}_index"] = (0, idx)
    torch.save(out, os.path.join(GOLD, name + ".pt"))
    print(name, {k: (tuple(v.shape) if torch.is_tensor(v) else v) for k, v in out.items() if k != "meta"})


def ddim_golden():
    """Schedule tables and one p_sample_ddim evaluation from the reference sampler."""
    ref_shim.load()
    from ldm.modules.diffusionmodules.util import (make_beta_schedule, make_ddim_sampling_parameters,
                                                   make_ddim_timesteps)
    from cldm.ddim_hacked import DDIMSampler
    betas = make_beta_schedule("linear", 1000, linear_start=0.00085, linear_end=0.012)  # cldm_v21.yaml:4-5
    ac = np.cumprod(1.0 - betas, axis=0)
    out = {}
    for S in (20, 30, 50):
        ts = make_ddim_timesteps("uniform", S, 1000, verbose=False)
        sig, a, ap = make_ddim_sampling_parameters(ac, ts, 0.0, verbose=False)
        out[f"S{S}"] = dict(timesteps=torch.tensor(ts), alphas=torch.tensor(a), alphas_prev=torch.tensor(ap),
                            sigmas=torch.tensor(sig))

    class FakeModel:  # the attributes DDIMSampler reads (SURVEY.md §8c)
        num_timesteps = 1000
        device = torch.device("cpu")
        parameterization = "eps"

        def __init__(self):
            self.betas = torch.tensor(betas)
            self.alphas_cumprod = torch.tensor(ac)
            self.alphas_cumprod_prev = torch.tensor(np.append(1.0, ac[:-1]))

        def apply_model(self, x, t, c):
            return torch.tanh(x * 0.7 + c)      # any deterministic function of (x, cond)

    m = FakeModel()
    sampler = DDIMSampler(m)
    sampler.register_buffer = lambda n, a: setattr(sampler, n, a if not torch.is_tensor(a) else a.cpu())
    sampler.make_schedule(50, ddim_eta=0.0, verbose=False)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(2, 4, 8, 8, generator=g)
    index = 37
    t = torch.full((2,), int(sampler.ddim_timesteps[index]), dtype=torch.long)
    x_prev, pred_x0 = sampler.p_sample_ddim(x, torch.tensor(0.3), t, index, unconditional_guidance_scale=9.0,
                                            unconditional_conditioning=torch.tensor(-0.2))
    out["p_sample"] = dict(x=x, index=index, e_cond=m.apply_model(x, t, torch.tensor(0.3)),
                           e_uncond=m.apply_model(x, t, torch.tensor(-0.2)), guidance=9.0,
                           x_prev=x_prev, pred_x0=pred_x0)
    torch.save(out, os.path.join(GOLD, "ddim.pt"))
    print("ddim", list(out))


def main():
    os.makedirs(GOLD, exist_ok=True)
    torch.manual_seed(0)
    if "--full" in sys.argv:
        torch.set_num_threads(os.cpu_count())
        only = [a for a in sys.argv[1:] if not a.startswith("--")]
        for n, s in FULL_CASES.items():
            if not only or n in only:
                run_case(n, s)
        return
    for n, s in CASES.items():
        run_case(n, s)
    ddim_golden()


if __name__ == "__main__":
    main()
