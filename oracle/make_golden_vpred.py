"""Generate tests/golden/ddim_vpred.pt with the REFERENCE's own sampler (build container only).

    python -m oracle.make_golden_vpred

Two p_sample_ddim evaluations of cldm.ddim_hacked.DDIMSampler for a v-prediction model (parameterization "v", the
SD2.1-768 base models): one guided (unconditional_guidance_scale 7.5, the combine applied to v, cldm/ddim_hacked.py:
190-192) and one unguided (scale 1, one model evaluation, :187-188).  The sampler converts v to eps and x0 with the
model's predict_eps_from_z_and_v / predict_start_from_z_and_v (:194-217); the fake model takes both methods from the
reference's own DDPM class (ldm/models/diffusion/ddpm.py:290-302), so they are not restated here.  It pins the v-mode
fused update (ea_out_cfg_vpred / ea_out_vpred) on machines where /root/reference does not exist.
"""
import os

import numpy as np
import torch

from oracle import ref_shim

GOLD = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")


def main():
    ref_shim.load()
    from ldm.models.diffusion.ddpm import DDPM
    from ldm.modules.diffusionmodules.util import make_beta_schedule
    from cldm.ddim_hacked import DDIMSampler
    betas = make_beta_schedule("linear", 1000, linear_start=0.00085, linear_end=0.012)  # cldm_v21.yaml:4-5
    ac = np.cumprod(1.0 - betas, axis=0)

    class FakeModel:  # the attributes DDIMSampler reads (SURVEY.md §8c), for a v-prediction model
        num_timesteps = 1000
        device = torch.device("cpu")
        parameterization = "v"
        predict_eps_from_z_and_v = DDPM.predict_eps_from_z_and_v
        predict_start_from_z_and_v = DDPM.predict_start_from_z_and_v

        def __init__(self):
            self.betas = torch.tensor(betas)
            self.alphas_cumprod = torch.tensor(ac)
            self.alphas_cumprod_prev = torch.tensor(np.append(1.0, ac[:-1]))
            self.sqrt_alphas_cumprod = torch.tensor(np.sqrt(ac))
            self.sqrt_one_minus_alphas_cumprod = torch.tensor(np.sqrt(1.0 - ac))
            self.calls = 0

        def apply_model(self, x, t, c):
            self.calls += 1
            return torch.tanh(x * 0.7 + c)      # any deterministic function of (x, cond)

    out = {}
    for name, scale, n, index, seed in (("guided", 7.5, 2, 17, 8), ("unguided", 1.0, 3, 23, 9)):
        m = FakeModel()
        sampler = DDIMSampler(m)
        sampler.register_buffer = lambda n_, a: setattr(sampler, n_, a if not torch.is_tensor(a) else a.cpu())
        sampler.make_schedule(50, ddim_eta=0.0, verbose=False)
        x = torch.randn(n, 4, 8, 8, generator=torch.Generator().manual_seed(seed))
        timestep = int(sampler.ddim_timesteps[index])
        t = torch.full((n,), timestep, dtype=torch.long)
        c, uc = torch.tensor(0.3), torch.tensor(-0.2)
        x_prev, pred_x0 = sampler.p_sample_ddim(x, c, t, index, unconditional_guidance_scale=scale,
                                                unconditional_conditioning=uc)
        assert m.calls == (2 if scale != 1.0 else 1)
        f = FakeModel()
        v_c, v_u = f.apply_model(x, t, c), f.apply_model(x, t, uc)
        out[name] = dict(x=x, index=index, timestep=timestep, guidance=scale, v_cond=v_c, v_uncond=v_u,
                         v=v_u + scale * (v_c - v_u) if scale != 1.0 else v_c,
                         a_t=float(sampler.ddim_alphas[index]), a_prev=float(sampler.ddim_alphas_prev[index]),
                         x_prev=x_prev, pred_x0=pred_x0)
    torch.save(out, os.path.join(GOLD, "ddim_vpred.pt"))
    for k, d in out.items():
        print("ddim_vpred", k, {n: (tuple(v.shape) if torch.is_tensor(v) else v) for n, v in d.items()})


if __name__ == "__main__":
    main()
