"""Generate tests/golden/t2i_guess.pt with the REFERENCE's own modules (build container only).

    python -m oracle.make_golden_guess_t2i

One guided p_sample_ddim of cldm.ddim_hacked.DDIMSampler in guess mode, as the reference's cldm text-to-image path
runs it (tools/sam2image_ori_version.py:133-142): the conditional call carries c_concat = [hint], the unconditional
one c_concat = None, so ControlLDM.apply_model (cldm/cldm.py:328-341) runs the UNet without control on that half.
The model is the reference's cldm.cldm.ControlNet and ControlledUnetModel at TINY size with the seeded weights of
editanything_b200.unet_spec.make_state_dict (whose zero-initialised tensors are drawn like every other weight),
control_scales = logspace(-1, 0, 13) * s (the guess-mode weights of ControlNetModel2.forward,
utils/stable_diffusion_controlnet.py:787-792) and only_mid_control = False.  `apply_model` is the reference's
ControlLDM.apply_model itself, called unbound on a namespace that holds those modules.

It pins "no ControlNet residual on the unconditional half" on machines where /root/reference does not exist.
"""
import os
from types import SimpleNamespace

import numpy as np
import torch

from editanything_b200.unet_spec import TINY, make_state_dict
from oracle import ref_shim
from oracle.inputs import make_inputs

GOLD = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
UNET_SEED, CN_SEED, IN_SEED = 111, 112, 113
N, LAT, L, SCALE, GUIDANCE, STEPS, INDEX = 2, 8, 7, 0.8, 6.0, 20, 13


def main():
    C = ref_shim.load()
    from ldm.modules.diffusionmodules.util import make_beta_schedule
    from cldm.ddim_hacked import DDIMSampler
    usd = make_state_dict(TINY, "unet", UNET_SEED)
    csd = make_state_dict(TINY, "controlnet", CN_SEED)
    unet, (cn,) = ref_shim.build_reference_nets(TINY, usd, [csd])
    x, ctx, (hint,) = make_inputs(TINY, 2 * N, LAT, L, IN_SEED, n_controlnets=1)
    x, hint = x[:N], hint[:N]
    ctx_uncond, ctx_cond = ctx[:N], ctx[N:]
    scales = [float(v) * SCALE for v in torch.logspace(-1, 0, 13)]

    b = make_beta_schedule("linear", 1000, linear_start=0.00085, linear_end=0.012)     # cldm_v15.yaml
    ac = np.cumprod(1.0 - b, axis=0)
    holder = SimpleNamespace(control_model=cn, model=SimpleNamespace(diffusion_model=unet), control_scales=scales,
                             only_mid_control=False)
    calls = []

    class Model:  # the attributes DDIMSampler reads; apply_model = the reference's ControlLDM.apply_model
        num_timesteps = 1000
        device = torch.device("cpu")
        parameterization = "eps"
        betas = torch.tensor(b)
        alphas_cumprod = torch.tensor(ac)
        alphas_cumprod_prev = torch.tensor(np.append(1.0, ac[:-1]))

        def apply_model(self, x_, t_, cond):
            calls.append(cond["c_concat"] is not None)
            return C.ControlLDM.apply_model(holder, x_, t_, cond)

    sampler = DDIMSampler(Model())
    sampler.register_buffer = lambda n, a: setattr(sampler, n, a if not torch.is_tensor(a) else a.cpu())
    sampler.make_schedule(STEPS, ddim_eta=0.0, verbose=False)
    t = torch.full((N,), int(sampler.ddim_timesteps[INDEX]), dtype=torch.long)
    cond = {"c_concat": [hint], "c_crossattn": [ctx_cond]}
    un_cond = {"c_concat": None, "c_crossattn": [ctx_uncond]}
    with torch.no_grad():
        x_prev, pred_x0 = sampler.p_sample_ddim(x, cond, t, INDEX, unconditional_guidance_scale=GUIDANCE,
                                                unconditional_conditioning=un_cond)
        e_cond = C.ControlLDM.apply_model(holder, x, t, cond)
        e_uncond = C.ControlLDM.apply_model(holder, x, t, un_cond)
    assert calls == [True, False], calls
    out = dict(meta=dict(cfg="TINY", unet_seed=UNET_SEED, cn_seed=CN_SEED, in_seed=IN_SEED, N=N, lat=LAT, L=L,
                         scale=SCALE, guidance=GUIDANCE, steps=STEPS, index=INDEX),
               x=x, hint=hint, ctx_uncond=ctx_uncond, ctx_cond=ctx_cond, timestep=int(t[0]),
               a_t=float(sampler.ddim_alphas[INDEX]), a_prev=float(sampler.ddim_alphas_prev[INDEX]),
               e_cond=e_cond, e_uncond=e_uncond, x_prev=x_prev, pred_x0=pred_x0)
    torch.save(out, os.path.join(GOLD, "t2i_guess.pt"))
    print("t2i_guess", {k: (tuple(v.shape) if torch.is_tensor(v) else v) for k, v in out.items() if k != "meta"})


if __name__ == "__main__":
    main()
