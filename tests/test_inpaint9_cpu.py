"""9-channel inpainting UNets (stabilityai/stable-diffusion-2-inpainting) with the operators emulated on CPU
(tests/cpu_ops.py): the engine against the reference-generated golden vector, the launch sequence, the pipeline's
9-channel branch against a re-enactment of the reference's (tests/inpaint_ref.py), and loading + the application
from diffusers-layout checkpoints."""
import os
from dataclasses import replace

import numpy as np
import pytest
import torch
from PIL import Image

from editanything_b200 import _backend
from editanything_b200.denoise import DenoiseEngine, ddim_schedule
from editanything_b200.pipeline import StableDiffusionControlNetInpaintPipeline
from editanything_b200.unet_spec import TINY, TINY21, TINY21_INPAINT, make_state_dict
from editanything_b200.vae_spec import VaeConfig
from oracle.inputs import make_inputs
from tests import cpu_ops, synth_ckpt
from tests.inpaint_ref import RecordingVAE, apply_model_9ch, reference_loop_9ch

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CPU = torch.device("cpu")


def _golden_engine(n_cn=None):
    g = torch.load(os.path.join(GOLD, "tiny_sd21_inpaint.pt"))
    m = g["meta"]
    seeds = m["cn_seeds"] if n_cn is None else [m["cn_seeds"][0] + i for i in range(n_cn)]
    usd = make_state_dict(TINY21_INPAINT, "unet", m["unet_seed"])
    csds = [make_state_dict(TINY21, "controlnet", s) for s in seeds]
    eng = DenoiseEngine(TINY21_INPAINT, usd, csds, CPU, backend=cpu_ops)
    x, ctx, hints = make_inputs(TINY21_INPAINT, m["B"], m["lat"], m["L"], m["in_seed"], n_controlnets=len(csds))
    return g, m, eng, x, ctx, hints, usd, csds


def test_eps_matches_reference_golden_and_keeps_lockstep():
    g, m, eng, x, ctx, hints, _, _ = _golden_engine()
    assert x.shape[1] == 9 and [R.n for R in eng.runner.groups] == [2]
    eng.prepare(ctx, hints, m["scales"])
    for t in m["timesteps"]:
        eps = eng.eps(x, t)
        ref = g[f"eps_t{t}"]
        assert (eps - ref).abs().max().item() < 2e-4 * max(1.0, ref.abs().max().item()), t
    # the ControlNets are 4-channel nets; a 4-channel x on this engine is refused
    assert all(c.cfg.in_channels == 4 for c in eng.cns) and eng.unet.cfg.in_channels == 9
    with pytest.raises(ValueError):
        eng.eps(x[:, :4], m["timesteps"][0])


def test_two_controlnets_lockstep_matches_oracle():
    _, m, eng, x, ctx, hints, usd, csds = _golden_engine(n_cn=2)
    assert [R.n for R in eng.runner.groups] == [3]
    eng.prepare(ctx, hints, [0.5, 1.0])
    with torch.no_grad():
        ref = apply_model_9ch(usd, TINY21_INPAINT, csds, x, 601, ctx, hints, [0.5, 1.0])
    assert (eng.eps(x, 601) - ref).abs().max().item() < 2e-4 * max(1.0, ref.abs().max().item())


def test_engine_rejects_other_channel_counts():
    cfg = replace(TINY21, in_channels=5)
    with pytest.raises(ValueError):
        DenoiseEngine(cfg, make_state_dict(cfg, "unet", 1), [], CPU, backend=cpu_ops)
    eng = DenoiseEngine(TINY21, make_state_dict(TINY21, "unet", 1), [], CPU, backend=cpu_ops)
    with pytest.raises(ValueError):                   # a 4-channel UNet has no condition channels
        eng.set_unet_condition(torch.zeros(1, 1, 8, 8), torch.zeros(1, 4, 8, 8))
    with pytest.raises(ValueError):
        eng.eps(torch.zeros(2, 9, 8, 8), 1)


def test_fused_step_launch_count_and_ddim_formula():
    """One fused step of the 9-channel engine makes as many launches as the same engine with in_channels=4 (conv_in
    reads the precomputed condition through its `add`); the request's condition costs one launch."""
    _, m, eng9, x, ctx, hints, usd, csds = _golden_engine()
    usd4 = dict(usd)
    usd4["input_blocks.0.0.weight"] = usd["input_blocks.0.0.weight"][:, :4].contiguous()
    eng4 = DenoiseEngine(replace(TINY21_INPAINT, in_channels=4), usd4, csds, CPU, backend=cpu_ops)
    ts, a, ap = ddim_schedule(50)
    lat0 = x[:1, :4].clone()
    counts = []
    for eng in (eng9, eng4):
        eng.prepare(ctx, hints, m["scales"])
        if eng is eng9:
            n0 = cpu_ops.launch_count()
            eng.set_unet_condition(x[:1, 4:5], x[:1, 5:9])
            assert cpu_ops.launch_count() - n0 == 1
        eng.begin(lat0, guidance=5.0, use_graph=False)
        eng.step(int(ts[3]), float(a[3]), float(ap[3]))        # warm: time-embedding rows of t
        eng.begin(lat0, guidance=5.0, use_graph=False)
        n0 = cpu_ops.launch_count()
        eng.step(int(ts[3]), float(a[3]), float(ap[3]))
        counts.append(cpu_ops.launch_count() - n0)
    assert counts[0] == counts[1], counts
    # the step is the DDIM update of eps(cat[x, x; cond; cond])
    x9 = torch.cat([torch.cat([lat0] * 2), torch.cat([x[:1, 4:]] * 2)], 1)
    eps = eng9.eps(x9, int(ts[3]))
    e = eps[:1] + 5.0 * (eps[1:] - eps[:1])
    x0 = (lat0 - (1 - a[3]) ** 0.5 * e) / a[3] ** 0.5
    xp = ap[3] ** 0.5 * x0 + (1 - ap[3]) ** 0.5 * e
    assert (eng9.latents() - xp).abs().max().item() < 1e-4


# ------------------------------------------------------------------------------------------------ pipeline
def _pipe_setup(n_cn=1, H=64, W=64):
    usd = make_state_dict(TINY21_INPAINT, "unet", 81)
    csds = [make_state_dict(TINY21, "controlnet", 82 + i) for i in range(n_cn)]
    eng = DenoiseEngine(TINY21_INPAINT, usd, csds, CPU, backend=cpu_ops)
    vae = RecordingVAE()
    pipe = StableDiffusionControlNetInpaintPipeline(eng, vae=vae)
    g = torch.Generator().manual_seed(0)
    image = torch.rand(1, 3, H, W, generator=g) * 2 - 1
    mask = torch.zeros(1, 1, H, W)
    mask[:, :, H // 4:3 * H // 4, W // 8:5 * W // 8] = 1.0
    conds = [torch.randint(0, 256, (1, 3, H, W), generator=g).float(), torch.rand(1, 3, H, W, generator=g)][:n_cn]
    pe = torch.randn(1, 9, TINY21.context_dim, generator=g)
    ne = torch.randn(1, 9, TINY21.context_dim, generator=g)
    return usd, csds, pipe, vae, image, mask, conds, pe, ne


def _call(pipe, image, mask, conds, pe, ne, *, steps=4, gs=7.0, scales=None, seed=7, n_img=1, **kw):
    H, W = image.shape[2], image.shape[3]
    scales = scales if scales is not None else [1.0] * len(conds)
    return pipe(image=image, mask_image=mask, controlnet_conditioning_image=conds, height=H, width=W,
                num_inference_steps=steps, guidance_scale=gs, generator=torch.manual_seed(seed), prompt_embeds=pe,
                negative_prompt_embeds=ne, output_type="latent", controlnet_conditioning_scale=scales,
                num_images_per_prompt=n_img, **kw).images


@pytest.mark.parametrize("n_img,n_cn,H,W", [(1, 1, 64, 64), (2, 2, 64, 64), (1, 1, 64, 128)])
def test_pipeline_ddim_matches_reference_branch(n_img, n_cn, H, W):
    usd, csds, pipe, vae, image, mask, conds, pe, ne = _pipe_setup(n_cn, H, W)
    assert pipe.unet.config.in_channels == 9 and pipe.controlnet.config.in_channels == 4
    assert all(n.config.in_channels == 4 for n in pipe.controlnet.nets)
    scales = [0.5, 1.0][:n_cn]
    out = _call(pipe, image, mask, conds, pe, ne, scales=scales, n_img=n_img, alignment_ratio=0.5)
    ref, masked = reference_loop_9ch(TINY21_INPAINT, usd, csds, image, mask, conds, pe, ne, steps=4, gs=7.0,
                                     scales=scales, seed=7, n_img=n_img)
    assert out.shape == (n_img, 4, H // 8, W // 8)
    assert (out - ref).abs().max().item() < 2e-4, (out - ref).abs().max().item()
    # the VAE encodes image * (mask < 0.5) only (the unmasked image is not encoded in this branch)
    assert len(vae.seen) == 1 and torch.equal(vae.seen[0], masked)
    # no blend: alignment_ratio is ignored, 1.0 included (the 4-channel branch raises IndexError there)
    assert torch.equal(_call(pipe, image, mask, conds, pe, ne, scales=scales, n_img=n_img, alignment_ratio=1.0), out)


def test_pipeline_unipc_generic_scheduler_and_callback():
    from editanything_b200.pipeline import DDIMScheduler
    from editanything_b200.schedulers import UniPCMultistepScheduler
    usd, csds, pipe, vae, image, mask, conds, pe, ne = _pipe_setup()
    # UniPC, fused on the device
    pipe.scheduler = UniPCMultistepScheduler.from_config(pipe.scheduler.config)
    out = _call(pipe, image, mask, conds, pe, ne, steps=6)
    ref, _ = reference_loop_9ch(TINY21_INPAINT, usd, csds, image, mask, conds, pe, ne, steps=6, gs=7.0, scales=[1.0],
                                seed=7, scheduler=UniPCMultistepScheduler.from_config(DDIMScheduler().config))
    assert (out - ref).abs().max().item() < 5e-4, (out - ref).abs().max().item()

    # any other scheduler object: eng.eps on the concatenated 9-channel input + scheduler.step
    class OtherDDIM:
        order, init_noise_sigma = 1, 1.0

        def __init__(self):
            self._s = DDIMScheduler()

        def set_timesteps(self, n, device=None):
            self._s.set_timesteps(n)
            self.timesteps = self._s.timesteps

        def scale_model_input(self, x, t):
            return x

        def step(self, e, t, x, **kw):
            return self._s.step(e, t, x)
    pipe.scheduler = OtherDDIM()
    out = _call(pipe, image, mask, conds, pe, ne)
    ref, _ = reference_loop_9ch(TINY21_INPAINT, usd, csds, image, mask, conds, pe, ne, steps=4, gs=7.0, scales=[1.0],
                                seed=7)
    assert (out - ref).abs().max().item() < 2e-4

    # a callback sees the latents of every step
    pipe.scheduler = DDIMScheduler()
    seen, pre = [], []
    out = _call(pipe, image, mask, conds, pe, ne, callback=lambda i, t, x: seen.append(x.clone()))
    reference_loop_9ch(TINY21_INPAINT, usd, csds, image, mask, conds, pe, ne, steps=4, gs=7.0, scales=[1.0], seed=7,
                       pre=pre)
    assert len(seen) == 4 and all((a - b).abs().max().item() < 2e-4 for a, b in zip(seen, pre))


def test_check_inputs_channel_rule():
    _, _, pipe, _, image, mask, conds, pe, ne = _pipe_setup()
    pipe.unet.config.in_channels = 8                   # neither 4 nor 2 * latent_channels + 1 (:955-979)
    with pytest.raises(ValueError):
        _call(pipe, image, mask, conds, pe, ne, steps=1)


# ------------------------------------------------------------------------------------------------ loading + app
VCFG = VaeConfig(ch=64, ch_mult=(1, 1, 1, 1), num_res_blocks=1)
SD2_INPAINTING = "stabilityai/stable-diffusion-2-inpainting"


@pytest.fixture
def cpu_backend():
    _backend.OPS = cpu_ops
    yield
    _backend.OPS = None


def make_sd2_inpaint_root(root):
    """The checkpoints an SD2-inpainting EditAnythingLoraModel loads (editany_lora.py:72-79,352-405), test-sized:
    a 9-channel base, the SD2.1 EditAnything ControlNet, the SD1.5 base and tile ControlNet of the tile pass."""
    usd, _ = synth_ckpt.write_pipeline(os.path.join(root, *SD2_INPAINTING.split("/")), TINY21_INPAINT, VCFG, seed=71)
    cn = synth_ckpt.write_unet_like(os.path.join(root, "shgao", "edit-anything-v0-4-sd21"), TINY21, "controlnet", 72)
    synth_ckpt.write_pipeline(os.path.join(root, "runwayml", "stable-diffusion-v1-5"), TINY, VCFG, seed=51)
    synth_ckpt.write_unet_like(os.path.join(root, "lllyasviel", "control_v11f1e_sd15_tile"), TINY, "controlnet", 54)
    return usd, cn


def test_from_pretrained_9ch_and_controlnet_rules(tmp_path, monkeypatch, cpu_backend):
    from editanything_b200.loading import ControlNetModel2
    from editanything_b200.nets import PackedNet
    usd, cn_sd = make_sd2_inpaint_root(str(tmp_path))
    monkeypatch.setenv("EA_MODEL_ROOT", str(tmp_path))
    cn = ControlNetModel2.from_pretrained("shgao/edit-anything-v0-4-sd21")
    pipe = StableDiffusionControlNetInpaintPipeline.from_pretrained(SD2_INPAINTING, controlnet=[cn],
                                                                   torch_dtype=torch.float16, safety_checker=None)
    assert pipe.engine.cfg == TINY21_INPAINT and pipe.unet.config.in_channels == 9
    assert pipe.controlnet.config.in_channels == 4 and pipe.controlnet.nets[0].config.in_channels == 4
    ref = PackedNet(TINY21_INPAINT, "unet", usd, pipe.engine.dev)
    assert ref.w.keys() == pipe.engine.unet.w.keys() and "input_blocks.0.0.wc" in ref.w
    for k, v in ref.w.items():
        assert torch.equal(v, pipe.engine.unet.w[k]), k
    ref_cn = PackedNet(TINY21, "controlnet", cn_sd, pipe.engine.dev)
    for k, v in ref_cn.w.items():
        assert torch.equal(v, pipe.engine.cns[0].w[k]), k
    # a ControlNet of another topology, or a 9-channel one, is refused
    for name, cfg in (("bad/other-topology", TINY), ("bad/nine-channel", TINY21_INPAINT)):
        synth_ckpt.write_unet_like(os.path.join(str(tmp_path), *name.split("/")), cfg, "controlnet", 5)
        with pytest.raises(ValueError):
            StableDiffusionControlNetInpaintPipeline.from_pretrained(
                SD2_INPAINTING, controlnet=[ControlNetModel2.from_pretrained(name)], share_with=pipe)
    # share_with a pipeline of another UNet is refused
    with pytest.raises(ValueError):
        StableDiffusionControlNetInpaintPipeline.from_pretrained(
            "runwayml/stable-diffusion-v1-5", controlnet=ControlNetModel2.from_pretrained("lllyasviel/control_v11f1e_sd15_tile"),
            share_with=pipe)


def test_app_sd2_inpainting_end_to_end(tmp_path, monkeypatch, cpu_backend):
    from editanything_b200 import app
    from tests.test_app_cpu import FakeSam, _inputs
    make_sd2_inpaint_root(str(tmp_path / "hub"))
    monkeypatch.setenv("EA_MODEL_ROOT", str(tmp_path / "hub"))
    monkeypatch.chdir(tmp_path)
    model = app.EditAnythingLoraModel(base_model_path=SD2_INPAINTING, controlmodel_name="LAION Pretrained(v0-4)-SD21",
                                      extra_inpaint=False, use_blip=False, lora_model_path=None,
                                      sam_generator=FakeSam(), mask_predictor=object())
    main, tile = model.pipe, model.tile_pipe
    assert main.engine.cfg.in_channels == 9 and len(main.engine.cns) == 1
    # the tile pass runs on a separately loaded SD1.5 base (editany_lora.py:395-405): nothing is shared
    assert tile.engine.cfg == TINY and tile.engine.unet is not main.engine.unet
    assert tile.vae is not main.vae and tile.text_encoder is not main.text_encoder
    args, kwargs = _inputs()
    args = args[:10] + (20,) + args[11:]      # 20 steps: the 4-channel tile pass's alignment_ratio 0.95 needs them
    refined, output, masks, text = model.process(*args, **kwargs)
    assert text == args[5] and len(output) == 2 and len(refined) == 2
    assert all(isinstance(i, Image.Image) and i.size == (64, 64) for i in output)
    assert all(isinstance(i, Image.Image) and i.size == (128, 128) for i in refined)
    assert isinstance(masks[0], Image.Image) and isinstance(masks[1], Image.Image)
    assert all(np.array(i).std() > 0 for i in output)
