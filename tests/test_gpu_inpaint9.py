"""-m gpu: 9-channel inpainting UNets (stabilityai/stable-diffusion-2-inpainting) on the H100 kernels - the network
against the reference-generated golden vectors at reduced width and at full size, the pipeline's 9-channel branch
against the oracle re-enactment of tests/inpaint_ref.py, and the application built from diffusers-layout checkpoints.

Tolerances as in tests/test_gpu_parity.py (per-step eps max-abs < 1e-2) and tests/test_gpu_pipeline.py (latents
rel-Frobenius < 3e-2 and max-abs < 0.15 after 8 steps at guidance 5)."""
import os

import numpy as np
import pytest
import torch
from PIL import Image

from editanything_b200.denoise import DenoiseEngine
from editanything_b200.pipeline import DDIMScheduler, StableDiffusionControlNetInpaintPipeline
from editanything_b200.schedulers import UniPCMultistepScheduler
from editanything_b200.unet_spec import SD2_INPAINT, TINY, TINY21, TINY21_INPAINT, controlnet_config, make_state_dict
from oracle.inputs import make_inputs
from tests.inpaint_ref import RecordingVAE, reference_loop_9ch

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
EPS_TOL = 1e-2
DEV = torch.device("cuda:0")


def _check_golden(name, cfg):
    g = torch.load(os.path.join(GOLD, name + ".pt"))
    m = g["meta"]
    eng = DenoiseEngine(cfg, make_state_dict(cfg, "unet", m["unet_seed"]),
                        [make_state_dict(controlnet_config(cfg), "controlnet", s) for s in m["cn_seeds"]], DEV)
    assert [R.n for R in eng.runner.groups] == [2]           # the UNet encoder and the ControlNet in lockstep
    torch.cuda.empty_cache()
    x, ctx, hints = make_inputs(cfg, m["B"], m["lat"], m["L"], m["in_seed"], n_controlnets=len(m["cn_seeds"]))
    eng.prepare(ctx, hints, m["scales"])
    for t in m["timesteps"]:
        eps = eng.eps(x, t).cpu()
        ref = g[f"eps_t{t}"]
        err = (eps - ref).abs().max().item()
        rel = ((eps - ref).norm() / ref.norm()).item()
        print(f"{name} t={t} eps max-abs {err:.3e} rel-fro {rel:.3e} ref-max {ref.abs().max().item():.3f}")
        assert err < EPS_TOL, (name, t, err, rel)


def test_eps_vs_reference_golden_reduced_width_inpaint():
    _check_golden("tiny_sd21_inpaint", TINY21_INPAINT)


def test_eps_vs_reference_golden_full_sd2_inpaint_512():
    """stabilityai/stable-diffusion-2-inpainting topology at 512x512 (64x64 latents), 1 image + CFG, one SD2.1
    ControlNet, L = 77, at the first / middle / last timestep of the 50-step DDIM table; golden eps from the
    reference's own cldm modules (oracle/make_golden_inpaint.py --full)."""
    _check_golden("sd2_inpaint_512", SD2_INPAINT)


STEPS, GS = 8, 5.0


def _close(a, b, what):
    err = (a - b).abs().max().item()
    rel = ((a - b).norm() / b.norm()).item()
    print(f"{what}: max-abs {err:.3e} rel-fro {rel:.3e}")
    assert rel < 3e-2 and err < 0.15, (what, err, rel)


@pytest.mark.parametrize("sched", ["ddim", "unipc"])
def test_pipeline_9ch_on_cuda_matches_reference_branch(sched):
    usd = make_state_dict(TINY21_INPAINT, "unet", 81)
    csds = [make_state_dict(TINY21, "controlnet", 82)]
    pipe = StableDiffusionControlNetInpaintPipeline(DenoiseEngine(TINY21_INPAINT, usd, csds, DEV), vae=RecordingVAE())
    if sched == "unipc":
        pipe.scheduler = UniPCMultistepScheduler.from_config(pipe.scheduler.config)
    g = torch.Generator().manual_seed(0)
    H, W = 128, 192
    image = torch.rand(1, 3, H, W, generator=g) * 2 - 1
    mask = torch.zeros(1, 1, H, W)
    mask[:, :, 32:96, 16:112] = 1.0
    conds = [torch.randint(0, 256, (1, 3, H, W), generator=g).float()]
    pe = torch.randn(1, 13, TINY21.context_dim, generator=g)
    ne = torch.randn(1, 13, TINY21.context_dim, generator=g)
    kw = dict(image=image, mask_image=mask, controlnet_conditioning_image=conds, height=H, width=W,
              num_inference_steps=STEPS, guidance_scale=GS, prompt_embeds=pe, negative_prompt_embeds=ne,
              controlnet_conditioning_scale=0.8, num_images_per_prompt=1, output_type="latent")
    lat = pipe(generator=torch.manual_seed(7), **kw).images
    assert lat.is_cuda and lat.shape == (1, 4, H // 8, W // 8)
    ref, _ = reference_loop_9ch(TINY21_INPAINT, usd, csds, image, mask, conds, pe, ne, steps=STEPS, gs=GS,
                                scales=[0.8], seed=7,
                                scheduler=UniPCMultistepScheduler.from_config(DDIMScheduler().config)
                                if sched == "unipc" else None)
    _close(lat.cpu(), ref, f"9-channel latents ({sched})")
    # a second request replays the captured step and is bit-identical
    g0 = pipe.engine._graph
    lat2 = pipe(generator=torch.manual_seed(7), **kw).images
    assert pipe.engine._graph is g0
    assert torch.equal(lat2, lat), (lat2 - lat).abs().max().item()


def test_app_sd2_inpainting_end_to_end_on_cuda(tmp_path, monkeypatch):
    from editanything_b200 import app
    from tests.test_app_cpu import FakeSam, _inputs
    from tests.test_inpaint9_cpu import SD2_INPAINTING, make_sd2_inpaint_root
    make_sd2_inpaint_root(str(tmp_path / "hub"))
    monkeypatch.setenv("EA_MODEL_ROOT", str(tmp_path / "hub"))
    monkeypatch.chdir(tmp_path)
    model = app.EditAnythingLoraModel(base_model_path=SD2_INPAINTING, controlmodel_name="LAION Pretrained(v0-4)-SD21",
                                      extra_inpaint=False, use_blip=False, lora_model_path=None,
                                      sam_generator=FakeSam(), mask_predictor=object())
    main, tile = model.pipe, model.tile_pipe
    assert main.engine.dev.type == "cuda" and main.engine.cfg.in_channels == 9
    assert tile.engine.cfg == TINY and tile.engine.unet is not main.engine.unet and tile.vae is not main.vae
    args, kwargs = _inputs()
    args = args[:8] + (128, 128, 20) + args[11:]       # image / detect resolution 128, 20 steps
    kwargs["refine_image_resolution"] = 256
    refined, output, masks, text = model.process(*args, **kwargs)
    assert text == args[5] and len(output) == 2 and len(refined) == 2
    assert all(isinstance(i, Image.Image) and i.size == (192, 128) for i in output)
    assert all(isinstance(i, Image.Image) and i.size == (384, 256) for i in refined)
    assert all(np.isfinite(np.array(i)).all() and np.array(i).std() > 0 for i in output + refined)
    g0 = main.engine._graph
    again = model.process(*args, **kwargs)
    assert main.engine._graph is g0 and len(again[1]) == 2
