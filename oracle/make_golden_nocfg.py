"""Generate tests/golden/ddim_nocfg.pt with the REFERENCE's own sampler (build container only).

    python -m oracle.make_golden_nocfg

One p_sample_ddim evaluation of cldm.ddim_hacked.DDIMSampler at unconditional_guidance_scale = 1: the sampler then
evaluates the model once, on the conditional input alone (cldm/ddim_hacked.py:187-188), and the DDIM update reads that
output directly.  The batch is odd (3 images) because unguided sampling runs the networks on the N images themselves.
It pins the unguided fused update (ea_out_ddim) on machines where /root/reference does not exist.
"""
import os

import numpy as np
import torch

from oracle import ref_shim

GOLD = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")


def main():
    ref_shim.load()
    from ldm.modules.diffusionmodules.util import make_beta_schedule
    from cldm.ddim_hacked import DDIMSampler
    betas = make_beta_schedule("linear", 1000, linear_start=0.00085, linear_end=0.012)  # cldm_v21.yaml:4-5
    ac = np.cumprod(1.0 - betas, axis=0)

    class FakeModel:  # the attributes DDIMSampler reads (SURVEY.md §8c)
        num_timesteps = 1000
        device = torch.device("cpu")
        parameterization = "eps"

        def __init__(self):
            self.betas = torch.tensor(betas)
            self.alphas_cumprod = torch.tensor(ac)
            self.alphas_cumprod_prev = torch.tensor(np.append(1.0, ac[:-1]))
            self.calls = 0

        def apply_model(self, x, t, c):
            self.calls += 1
            return torch.tanh(x * 0.7 + c)      # any deterministic function of (x, cond)

    m = FakeModel()
    sampler = DDIMSampler(m)
    sampler.register_buffer = lambda n, a: setattr(sampler, n, a if not torch.is_tensor(a) else a.cpu())
    sampler.make_schedule(50, ddim_eta=0.0, verbose=False)
    x = torch.randn(3, 4, 8, 8, generator=torch.Generator().manual_seed(6))
    index = 23
    t = torch.full((3,), int(sampler.ddim_timesteps[index]), dtype=torch.long)
    x_prev, pred_x0 = sampler.p_sample_ddim(x, torch.tensor(0.3), t, index, unconditional_guidance_scale=1.0,
                                            unconditional_conditioning=torch.tensor(-0.2))
    assert m.calls == 1, "the unguided sampler evaluates the model once"
    e = FakeModel().apply_model(x, t, torch.tensor(0.3))
    out = {"p_sample": dict(x=x, index=index, timestep=int(sampler.ddim_timesteps[index]), e=e,
                            a_t=float(sampler.ddim_alphas[index]), a_prev=float(sampler.ddim_alphas_prev[index]),
                            x_prev=x_prev, pred_x0=pred_x0)}
    torch.save(out, os.path.join(GOLD, "ddim_nocfg.pt"))
    print("ddim_nocfg", {k: (tuple(v.shape) if torch.is_tensor(v) else v) for k, v in out["p_sample"].items()})


if __name__ == "__main__":
    main()
