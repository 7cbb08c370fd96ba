"""-m gpu: `StableDiffusionControlNetInpaintPipeline.__call__` on CUDA - the API BASELINE.json's north_star
names - with `VaeEngine` behind `pipe.vae`, for alignment_ratio in {None, 0.5} (the reference's tile pass uses
0.95, editany_demo.py:123-130), against the oracle re-enactment of the reference loop
(utils/stable_diffusion_controlnet_inpaint.py:1131-1703) already used by tests/test_pipeline_cpu.py.

Tolerances (fp16 storage / fp32 accumulation vs the fp32 oracle; the per-step eps gate is 1e-2,
tests/test_gpu_parity.py): the DDIM update divides by sqrt(a_t) and CFG multiplies eps differences by the guidance
scale, so a per-step eps error of ~3e-3 grows to several 1e-2 over a short schedule (measured 7.6e-2 max-abs after
the 4-step, guidance-9 loop).  Gates: latents rel-Frobenius < 3e-2 and max-abs < 0.15 after 8 steps at guidance 5;
decoded image in [0, 1]: mean-abs < 1e-2."""
import pytest
import torch
import torch.nn.functional as F

from editanything_b200.denoise import DenoiseEngine
from editanything_b200.pipeline import DDIMScheduler, StableDiffusionControlNetInpaintPipeline
from editanything_b200.unet_spec import TINY, build_topology, make_state_dict
from editanything_b200.vae import VaeEngine, make_vae_state_dict
from editanything_b200.vae_spec import VaeConfig
from oracle import unet_oracle as O
from oracle import vae_oracle as V

pytestmark = pytest.mark.gpu
VCFG = VaeConfig(ch=64, ch_mult=(1, 1, 1, 1), num_res_blocks=1)          # f = 8 like kl-f8, test-sized


def _setup(n_cn=2, n_img=1):
    cfg = TINY
    dev = torch.device("cuda:0")
    usd = make_state_dict(cfg, "unet", 51)
    csds = [make_state_dict(cfg, "controlnet", 52 + i) for i in range(n_cn)]
    vsd = dict(make_vae_state_dict(VCFG, 61, part="encoder"))
    vsd.update(make_vae_state_dict(VCFG, 62))
    eng = DenoiseEngine(cfg, usd, csds, dev)
    pipe = StableDiffusionControlNetInpaintPipeline(eng, vae=VaeEngine(VCFG, vsd, dev))
    g = torch.Generator().manual_seed(0)
    H = W = 128
    image = torch.rand(1, 3, H, W, generator=g) * 2 - 1
    mask = torch.zeros(1, 1, H, W)
    mask[:, :, 32:96, 16:80] = 1.0
    conds = [torch.randint(0, 256, (1, 3, H, W), generator=g).float(), torch.rand(1, 3, H, W, generator=g)][:n_cn]
    pe = torch.randn(1, 13, cfg.context_dim, generator=g)
    ne = torch.randn(1, 13, cfg.context_dim, generator=g)
    return cfg, usd, csds, vsd, pipe, image, mask, conds, pe, ne


def _close(a, b, what):
    err = (a - b).abs().max().item()
    rel = ((a - b).norm() / b.norm()).item()
    print(f"{what}: max-abs {err:.3e} rel-fro {rel:.3e}")
    assert rel < 3e-2 and err < 0.15, (what, err, rel)


STEPS, GS = 8, 5.0


def _reenact(cfg, usd, csds, vsd, image, mask, conds, pe, ne, steps, gs, scales, seed, alignment_ratio, n_img):
    gen = torch.manual_seed(seed)
    h = image.shape[2] // 8
    lat = torch.randn((n_img, 4, h, h), generator=gen)                    # prepare_latents (:981-1014)
    noise = lat
    with torch.no_grad():                                                 # in_channels == 4: the source image (:1469-1476)
        mom = V.encode_moments(image, vsd, VCFG)
    mean, logvar = mom.chunk(2, 1)
    init = VCFG.scaling_factor * (mean + torch.exp(0.5 * logvar.clamp(-30, 20)) * torch.randn(mean.shape, generator=gen))
    init = init.repeat(n_img, 1, 1, 1)
    m = 1 - F.interpolate((mask >= 0.5).float(), (h, h), mode="nearest")
    sch = DDIMScheduler()
    sch.set_timesteps(steps)
    ts = sch.timesteps
    ctx = torch.cat([ne.repeat(n_img, 1, 1), pe.repeat(n_img, 1, 1)])
    hints = [torch.cat([c.repeat_interleave(n_img, 0)] * 2) for c in conds]
    ut, ct = build_topology(cfg), build_topology(cfg, with_decoder=False)
    pre = []
    for i, t in enumerate(ts):
        with torch.no_grad():
            e = O.apply_model(usd, ut, [(sd, ct) for sd in csds], torch.cat([lat] * 2), torch.full((2 * n_img,), int(t)),
                              ctx, hints, scales)
        lat = sch.step(e[:n_img] + gs * (e[n_img:] - e[:n_img]), t, lat).prev_sample
        pre.append(lat.clone())
        if alignment_ratio is not None and i < len(ts) * alignment_ratio:
            lat = sch.add_noise(init, noise, ts[i + 1]) * m + lat * (1 - m)
    if alignment_ratio is None or alignment_ratio == 1.0:
        lat = init * m + lat * (1 - m)
    return lat, pre


@pytest.mark.parametrize("alignment_ratio", [None, 0.5])
def test_pipeline_call_on_cuda_matches_reference_loop(alignment_ratio):
    cfg, usd, csds, vsd, pipe, image, mask, conds, pe, ne = _setup()
    kw = dict(image=image, mask_image=mask, controlnet_conditioning_image=conds, height=128, width=128,
              num_inference_steps=STEPS, guidance_scale=GS, prompt_embeds=pe, negative_prompt_embeds=ne,
              controlnet_conditioning_scale=[0.5, 1.0], alignment_ratio=alignment_ratio, num_images_per_prompt=1)
    lat = pipe(generator=torch.manual_seed(7), output_type="latent", **kw).images
    assert lat.is_cuda
    ref, _ = _reenact(cfg, usd, csds, vsd, image, mask, conds, pe, ne, STEPS, GS, [0.5, 1.0], 7, alignment_ratio, 1)
    _close(lat.cpu(), ref, f"latents alignment_ratio={alignment_ratio}")
    out = pipe(generator=torch.manual_seed(7), output_type="np", **kw)
    assert out.nsfw_content_detected is None
    with torch.no_grad():
        img = V.decode_latents(ref, vsd, VCFG).permute(0, 2, 3, 1).numpy()
    assert out.images.shape == img.shape == (1, 128, 128, 3)
    assert abs(out.images - img).mean() < 1e-2
    # a second image through the same pipeline object replays the captured step (no re-capture when the blend
    # window opens or closes: the blend buffers always exist)
    g0 = pipe.engine._graph
    lat2 = pipe(generator=torch.manual_seed(7), output_type="latent", **kw).images
    assert pipe.engine._graph is g0
    # bit-reproducible: GroupNorm statistics are per-CTA partials summed in a fixed order (no floating-point
    # atomics), split-K partial tiles are reduced in split order, the step runs on one stream
    assert torch.equal(lat2, lat), (lat2 - lat).abs().max().item()


def test_pipeline_callback_sees_unblended_latents_and_two_images_per_prompt():
    """The reference calls `callback(i, t, latents)` BEFORE the inpaint blend of step i (:1640-1656)."""
    cfg, usd, csds, vsd, pipe, image, mask, conds, pe, ne = _setup(n_cn=1)
    seen = []
    kw = dict(image=image, mask_image=mask, controlnet_conditioning_image=conds, height=128, width=128,
              num_inference_steps=STEPS, guidance_scale=GS, prompt_embeds=pe, negative_prompt_embeds=ne,
              controlnet_conditioning_scale=0.8, alignment_ratio=0.5, num_images_per_prompt=2, output_type="latent")
    lat = pipe(generator=torch.manual_seed(5), callback=lambda i, t, x: seen.append(x.detach().cpu().clone()), **kw).images
    ref, pre = _reenact(cfg, usd, csds, vsd, image, mask, conds, pe, ne, STEPS, GS, [0.8], 5, 0.5, 2)
    assert len(seen) == STEPS and lat.shape == (2, 4, 16, 16)
    for i, (a, b) in enumerate(zip(seen, pre)):
        _close(a, b, f"callback latents step {i}")
    _close(lat.cpu(), ref, "final latents")
    # and the fused-blend path (no callback) ends in the same place
    lat_f = pipe(generator=torch.manual_seed(5), **kw).images
    _close(lat_f.cpu(), lat.cpu(), "fused blend vs host-side blend")


def test_pipeline_with_unipc_scheduler_fused_update():
    """`pipe.scheduler = UniPCMultistepScheduler.from_config(pipe.scheduler.config)` (editany_lora.py:383,418): the
    fused device-side multistep update against the reference loop re-enacted with the scheduler object on the oracle
    networks (alignment_ratio 0.5: the blend re-noises with the scheduler's alpha_t / sigma_t)."""
    from editanything_b200.schedulers import UniPCMultistepScheduler
    cfg, usd, csds, vsd, pipe, image, mask, conds, pe, ne = _setup()
    pipe.scheduler = UniPCMultistepScheduler.from_config(pipe.scheduler.config)
    for ar in (None, 0.5):
        lat = pipe(image=image, mask_image=mask, controlnet_conditioning_image=conds, height=128, width=128,
                   num_inference_steps=STEPS, guidance_scale=GS, prompt_embeds=pe, negative_prompt_embeds=ne,
                   controlnet_conditioning_scale=[0.5, 1.0], alignment_ratio=ar, num_images_per_prompt=1,
                   generator=torch.manual_seed(7), output_type="latent").images
        gen = torch.manual_seed(7)
        x = torch.randn((1, 4, 16, 16), generator=gen)
        noise = x
        with torch.no_grad():
            mom = V.encode_moments(image, vsd, VCFG)
        mean, logvar = mom.chunk(2, 1)
        init = VCFG.scaling_factor * (mean + torch.exp(0.5 * logvar.clamp(-30, 20)) * torch.randn(mean.shape, generator=gen))
        m = 1 - F.interpolate((mask >= 0.5).float(), (16, 16), mode="nearest")
        sch = UniPCMultistepScheduler.from_config(DDIMScheduler().config)
        sch.set_timesteps(STEPS)
        ts = sch.timesteps
        ctx = torch.cat([ne, pe])
        hints = [torch.cat([c] * 2) for c in conds]
        ut, ct = build_topology(cfg), build_topology(cfg, with_decoder=False)
        for i, t in enumerate(ts):
            with torch.no_grad():
                e = O.apply_model(usd, ut, [(sd, ct) for sd in csds], torch.cat([x] * 2), torch.full((2,), int(t)), ctx, hints, [0.5, 1.0])
            x = sch.step(e[:1] + GS * (e[1:] - e[:1]), t, x).prev_sample
            if ar is not None and i < len(ts) * ar:
                x = sch.add_noise(init, noise, ts[i + 1]) * m + x * (1 - m)
        if ar is None:
            x = init * m + x * (1 - m)
        _close(lat.cpu(), x, f"UniPC latents alignment_ratio={ar}")
