"""Generate the 9-channel (inpainting UNet) golden vectors with the REFERENCE's own modules (build container only).

    python -m oracle.make_golden_inpaint [--full]

Like oracle/make_golden.py, but the UNet is a reference `ControlledUnetModel` with in_channels = 9 (latents, mask,
masked-image latents: utils/stable_diffusion_controlnet_inpaint.py:1550-1558) and the ControlNet a reference
`ControlNet` with in_channels = 4 (models/cldm_v21.yaml:44) that reads the latent channels x[:, :4] (:1607-1615).
"""
import os
import sys

import torch

from editanything_b200.unet_spec import SD2_INPAINT, TINY21_INPAINT, controlnet_config, make_state_dict
from oracle import ref_shim
from oracle.inputs import make_inputs
from oracle.make_golden import GOLD, UNET_SEED

# name -> (cfg, batch, latent side, ctx len, timesteps, controlnet seeds, scales, input seed)
CASES = {
    "tiny_sd21_inpaint": (TINY21_INPAINT, 2, 16, 20, [981, 501], (102,), [1.0], 15),
}
FULL_CASES = {
    # stabilityai/stable-diffusion-2-inpainting at 512x512: 1 image + CFG -> B=2, 64x64 latents, L=77, one SD2.1
    # EditAnything ControlNet; first / middle / last timestep of the 50-step DDIM table
    "sd2_inpaint_512": (SD2_INPAINT, 2, 64, 77, [981, 501, 1], (102,), [1.0], 16),
}


def build_nets(cfg, usd, csds):
    C = ref_shim.load()
    unet = C.ControlledUnetModel(out_channels=cfg.out_channels, **ref_shim.ctor_kwargs(cfg)).eval()
    unet.load_state_dict(usd, strict=True)
    cns = []
    for sd in csds:
        cn = C.ControlNet(hint_channels=cfg.hint_channels, **ref_shim.ctor_kwargs(controlnet_config(cfg))).eval()
        cn.load_state_dict(sd, strict=True)
        cns.append(cn)
    return unet, cns


def run_case(name, spec):
    cfg, B, lat, L, ts, cn_seeds, scales, in_seed = spec
    usd = make_state_dict(cfg, "unet", UNET_SEED)
    csds = [make_state_dict(controlnet_config(cfg), "controlnet", s) for s in cn_seeds]
    unet, cns = build_nets(cfg, usd, csds)
    x, ctx, hints = make_inputs(cfg, B, lat, L, in_seed, n_controlnets=len(cn_seeds))
    out = {"meta": dict(name=name, B=B, lat=lat, L=L, timesteps=ts, cn_seeds=list(cn_seeds), scales=scales,
                        in_seed=in_seed, unet_seed=UNET_SEED)}
    for t in ts:
        tt = torch.full((B,), t, dtype=torch.long)
        with torch.no_grad():
            control = None
            for cn, hint, s in zip(cns, hints, scales):
                outs = [o * s for o in cn(x=x[:, :4], hint=hint, timesteps=tt, context=ctx)]
                control = outs if control is None else [a + b for a, b in zip(control, outs)]
            eps = unet(x=x, timesteps=tt, context=ctx, control=list(control), only_mid_control=False)
        out[f"eps_t{t}"] = eps.clone()
    torch.save(out, os.path.join(GOLD, name + ".pt"))
    print(name, {k: (tuple(v.shape) if torch.is_tensor(v) else v) for k, v in out.items() if k != "meta"})


def main():
    os.makedirs(GOLD, exist_ok=True)
    torch.manual_seed(0)
    cases = CASES
    if "--full" in sys.argv:
        torch.set_num_threads(os.cpu_count())
        cases = FULL_CASES
    for n, s in cases.items():
        run_case(n, s)


if __name__ == "__main__":
    main()
