"""Sampling without classifier-free guidance (guidance_scale <= 1) with the operators emulated on CPU
(tests/cpu_ops_unguided.py): the pipeline against a re-enactment of the reference's unguided loop
(utils/stable_diffusion_controlnet_inpaint.py:1329 `do_classifier_free_guidance = guidance_scale > 1.0` false: the
positive prompt alone, undoubled conditioning images and latents, `noise_pred` straight into the scheduler) on the
oracle networks, the engine's guided / unguided switching, odd batches, the out-conv update against the reference
sampler's own unguided p_sample_ddim (tests/golden/ddim_nocfg.pt) and EditAnythingLoraModel.process end to end."""
import math
import os

import pytest
import torch
import torch.nn.functional as F

from editanything_b200.denoise import DenoiseEngine, ddim_schedule
from editanything_b200.pipeline import DDIMScheduler, StableDiffusionControlNetInpaintPipeline
from editanything_b200.schedulers import UniPCMultistepScheduler
from editanything_b200.unet_spec import TINY, TINY21, TINY21_INPAINT, build_topology, make_state_dict
from oracle import unet_oracle as O
from oracle.inputs import make_inputs
from tests import cpu_ops_unguided as cpu_ops
from tests.inpaint_ref import RecordingVAE, apply_model_9ch
from tests.test_pipeline_cpu import FakeVAE

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CPU = torch.device("cpu")


def _setup(n_cn=2):
    """tests/test_pipeline_cpu.py's tiny pipeline and inputs, on the emulation that has ea_out_ddim."""
    cfg = TINY
    usd = make_state_dict(cfg, "unet", 51)
    csds = [make_state_dict(cfg, "controlnet", 52 + i) for i in range(n_cn)]
    eng = DenoiseEngine(cfg, usd, csds, CPU, backend=cpu_ops)
    pipe = StableDiffusionControlNetInpaintPipeline(eng, vae=FakeVAE())
    g = torch.Generator().manual_seed(0)
    H = W = 64
    image = torch.rand(1, 3, H, W, generator=g) * 2 - 1
    mask = torch.zeros(1, 1, H, W)
    mask[:, :, 16:48, 8:40] = 1.0
    conds = [torch.randint(0, 256, (1, 3, H, W), generator=g).float(), torch.rand(1, 3, H, W, generator=g)][:n_cn]
    pe = torch.randn(1, 9, cfg.context_dim, generator=g)
    ne = torch.randn(1, 9, cfg.context_dim, generator=g)
    return cfg, usd, csds, pipe, image, mask, conds, pe, ne


class OtherDDIM:
    """The built-in DDIM behind another class: the pipeline's non-fused path (engine.eps + scheduler.step)."""

    def __init__(self):
        self._s = DDIMScheduler()
        self.order, self.init_noise_sigma = 1, 1.0

    def set_timesteps(self, n, device=None):
        self._s.set_timesteps(n)
        self.timesteps = self._s.timesteps

    def scale_model_input(self, x, t):
        return x

    def step(self, e, t, x, **kw):
        return self._s.step(e, t, x)

    def add_noise(self, a, b, t):
        return self._s.add_noise(a, b, t)


def reference_loop_nocfg(cfg, usd, csds, image, mask, conds, pe, *, steps, scales, seed, alignment_ratio,
                         n_img=1, scheduler=None, seen=None):
    """The reference __call__ (in_channels == 4) with do_classifier_free_guidance false: ctx = the positive prompt
    embeddings, hints and latents undoubled, the network output used as is (:1627-1631 skipped)."""
    vae = FakeVAE()
    sch = scheduler if scheduler is not None else DDIMScheduler()
    sch.set_timesteps(steps)
    ts = sch.timesteps
    ctx = pe.repeat(n_img, 1, 1)
    hints = [c.repeat_interleave(n_img, 0) for c in conds]
    lat = torch.randn((n_img, 4, 8, 8), generator=torch.Generator().manual_seed(seed))
    noise = lat
    init = 0.18215 * vae.encode(image).latent_dist.sample().repeat(n_img, 1, 1, 1)
    m = 1 - F.interpolate((mask >= 0.5).float(), (8, 8), mode="nearest")
    ut, ct = build_topology(cfg), build_topology(cfg, with_decoder=False)
    for i, t in enumerate(ts):
        with torch.no_grad():
            e = O.apply_model(usd, ut, [(sd, ct) for sd in csds], lat, torch.full((n_img,), int(t)), ctx, hints, scales)
        lat = sch.step(e, t, lat).prev_sample
        if seen is not None:
            seen.append(lat.clone())
        if alignment_ratio is not None and i < len(ts) * alignment_ratio:
            lat = sch.add_noise(init, noise, ts[i + 1]) * m + lat * (1 - m)
    if alignment_ratio is None or alignment_ratio == 1.0:
        lat = init * m + lat * (1 - m)
    return lat


def _call(pipe, image, mask, conds, pe, ne, gs, *, steps=4, seed=7, n_img=1, scales=(0.5, 1.0), **kw):
    return pipe(image=image, mask_image=mask, controlnet_conditioning_image=conds, height=64, width=64,
                num_inference_steps=steps, guidance_scale=gs, generator=torch.manual_seed(seed), prompt_embeds=pe,
                negative_prompt_embeds=ne, output_type="latent", controlnet_conditioning_scale=list(scales)[:len(conds)],
                num_images_per_prompt=n_img, **kw).images


# ------------------------------------------------------------------------------------------------ 4-channel pipeline
@pytest.mark.parametrize("n_img", [1, 3])
@pytest.mark.parametrize("alignment_ratio", [None, 0.5])
@pytest.mark.parametrize("gs", [1.0, 0.5])
def test_call_matches_unguided_reference_loop(gs, alignment_ratio, n_img):
    cfg, usd, csds, pipe, image, mask, conds, pe, ne = _setup()
    out = _call(pipe, image, mask, conds, pe, ne, gs, alignment_ratio=alignment_ratio, n_img=n_img)
    ref = reference_loop_nocfg(cfg, usd, csds, image, mask, conds, pe, steps=4, scales=[0.5, 1.0], seed=7,
                               alignment_ratio=alignment_ratio, n_img=n_img)
    assert pipe.engine.B == n_img and not pipe.engine.guided            # the networks ran on the N images alone
    assert out.shape == (n_img, 4, 8, 8)
    assert (out - ref).abs().max().item() < 2e-4, (out - ref).abs().max().item()


def test_guidance_below_one_gives_exactly_the_latents_of_one():
    """Without guidance the scale is not used at all: 0.5 is not an extrapolation towards the negative prompt."""
    cfg, usd, csds, pipe, image, mask, conds, pe, ne = _setup()
    a = _call(pipe, image, mask, conds, pe, ne, 1.0, alignment_ratio=0.5)
    b = _call(pipe, image, mask, conds, pe, ne, 0.5, alignment_ratio=0.5)
    c = _call(pipe, image, mask, conds, pe, None, 0.5, alignment_ratio=0.5)    # no negative prompt needed
    assert torch.equal(a, b) and torch.equal(a, c)


def test_callback_sees_unblended_latents_and_host_blend_matches():
    cfg, usd, csds, pipe, image, mask, conds, pe, ne = _setup()
    seen = []
    out = _call(pipe, image, mask, conds, pe, ne, 1.0, alignment_ratio=0.5,
                callback=lambda i, t, x: seen.append(x.clone()))
    pre = []
    ref = reference_loop_nocfg(cfg, usd, csds, image, mask, conds, pe, steps=4, scales=[0.5, 1.0], seed=7,
                               alignment_ratio=0.5, seen=pre)
    assert len(seen) == 4 and (out - ref).abs().max().item() < 2e-4
    for s, p in zip(seen, pre):
        assert (s - p).abs().max().item() < 2e-4
    assert (seen[0] - out).abs().max().item() > 1e-3


@pytest.mark.parametrize("alignment_ratio", [None, 0.5])
def test_fused_ddim_fused_unipc_and_scheduler_objects_agree(alignment_ratio):
    """Fused DDIM == the non-fused path with a DDIM object; fused UniPC == the reference loop driven by the UniPC
    scheduler object."""
    cfg, usd, csds, pipe, image, mask, conds, pe, ne = _setup()
    fused = _call(pipe, image, mask, conds, pe, ne, 1.0, alignment_ratio=alignment_ratio)
    pipe.scheduler = OtherDDIM()
    generic = _call(pipe, image, mask, conds, pe, ne, 1.0, alignment_ratio=alignment_ratio)
    assert (fused - generic).abs().max().item() < 1e-4
    pipe.scheduler = UniPCMultistepScheduler.from_config(DDIMScheduler().config)
    unipc = _call(pipe, image, mask, conds, pe, ne, 1.0, steps=6, alignment_ratio=alignment_ratio)
    ref = reference_loop_nocfg(cfg, usd, csds, image, mask, conds, pe, steps=6, scales=[0.5, 1.0], seed=7,
                               alignment_ratio=alignment_ratio,
                               scheduler=UniPCMultistepScheduler.from_config(DDIMScheduler().config))
    assert (unipc - ref).abs().max().item() < 5e-4, (unipc - ref).abs().max().item()


# ------------------------------------------------------------------------------------------------ 9-channel pipeline
@pytest.mark.parametrize("fused", [True, False])
def test_nine_channel_unguided_matches_reference_branch(fused):
    """in_channels == 9 without guidance: the UNet reads cat([x, mask, masked-image latents]) on the N rows alone."""
    n_img, steps, seed = 3, 4, 7
    usd = make_state_dict(TINY21_INPAINT, "unet", 81)
    csds = [make_state_dict(TINY21, "controlnet", 82)]
    eng = DenoiseEngine(TINY21_INPAINT, usd, csds, CPU, backend=cpu_ops)
    pipe = StableDiffusionControlNetInpaintPipeline(eng, vae=RecordingVAE())
    if not fused:
        pipe.scheduler = OtherDDIM()
    g = torch.Generator().manual_seed(0)
    image = torch.rand(1, 3, 64, 64, generator=g) * 2 - 1
    mask = torch.zeros(1, 1, 64, 64)
    mask[:, :, 16:48, 8:40] = 1.0
    conds = [torch.randint(0, 256, (1, 3, 64, 64), generator=g).float()]
    pe = torch.randn(1, 9, TINY21.context_dim, generator=g)
    out = pipe(image=image, mask_image=mask, controlnet_conditioning_image=conds, height=64, width=64,
               num_inference_steps=steps, guidance_scale=1.0, generator=torch.manual_seed(seed), prompt_embeds=pe,
               output_type="latent", controlnet_conditioning_scale=1.0, num_images_per_prompt=n_img).images
    # re-enactment (tests/inpaint_ref.reference_loop_9ch without the doubling and the combine)
    vae, sch, gen = RecordingVAE(), DDIMScheduler(), torch.manual_seed(seed)
    sch.set_timesteps(steps)
    lat = torch.randn((n_img, 4, 8, 8), generator=gen)
    mbin = (mask >= 0.5).float()
    mask_lat = F.interpolate(mbin, size=(8, 8)).repeat(n_img, 1, 1, 1)
    masked_lat = (0.18215 * vae.encode(image * (mbin < 0.5)).latent_dist.sample(generator=gen)).repeat(n_img, 1, 1, 1)
    for t in sch.timesteps:
        with torch.no_grad():
            e = apply_model_9ch(usd, TINY21_INPAINT, csds, torch.cat([lat, mask_lat, masked_lat], 1), t,
                                pe.repeat(n_img, 1, 1), [conds[0].repeat_interleave(n_img, 0)], [1.0])
        lat = sch.step(e, t, lat).prev_sample
    assert eng.B == n_img and (not fused or eng.cond_in.shape[0] == n_img)
    assert (out - lat).abs().max().item() < 2e-4, (out - lat).abs().max().item()


# ------------------------------------------------------------------------------------------------ engine
def _tiny_engine(n_cn=2, unet_packed=None, seed=51):
    usd = None if unet_packed is not None else make_state_dict(TINY, "unet", seed)
    csds = [make_state_dict(TINY, "controlnet", seed + 1 + i) for i in range(n_cn)]
    return DenoiseEngine(TINY, usd, csds, CPU, backend=cpu_ops, unet_packed=unet_packed)


def _request(eng, guided, n_img, seed, steps=4):
    """One request on `eng`: prepare + begin + a few fused steps; returns the latents."""
    x, ctx, hints = make_inputs(TINY, 2 * n_img, 8, 7, seed, n_controlnets=len(eng.cns))
    if not guided:
        ctx, hints = ctx[n_img:], [h[n_img:] for h in hints]       # the positive half only
    ts, a, ap = ddim_schedule(steps)
    eng.prepare(ctx, hints, [0.5, 1.0][:len(eng.cns)], cfg_duplicated=False, guided=guided)
    eng.set_schedule(ts, a, ap)
    eng.begin(x[:n_img, :4], guidance=6.0, use_graph=False)
    for _ in ts:
        eng.step()
    return eng.latents()


def test_switching_guided_and_unguided_on_one_engine_and_a_shared_tile_engine():
    """guided -> unguided -> guided on one engine, and on a tile engine sharing its packed UNet, equals fresh engines:
    the buffers are re-sized and nothing of the previous mode leaks into the next request."""
    main = _tiny_engine()
    tile = _tiny_engine(n_cn=1, unet_packed=main.unet)
    seq = [(True, 1, 3), (False, 1, 4), (False, 3, 5), (True, 2, 6), (False, 2, 7), (True, 1, 3)]
    for k, (guided, n_img, seed) in enumerate(seq):
        for eng, n_cn in ((main, 2), (tile, 1)):
            got = _request(eng, guided, n_img, seed + 10 * n_cn)
            fresh = _request(_tiny_engine(n_cn) if n_cn == 2 else _tiny_engine(1, unet_packed=_tiny_engine(0).unet),
                             guided, n_img, seed + 10 * n_cn)
            assert got.shape == (n_img, 4, 8, 8)
            assert torch.equal(got, fresh), (k, guided, n_img, n_cn)


def test_eps_returns_every_row_for_any_batch():
    """eps() of B = 1, 2, 3 rows (unguided) and B = 2 (guided) against the oracle networks."""
    usd = make_state_dict(TINY, "unet", 51)
    csds = [make_state_dict(TINY, "controlnet", 52 + i) for i in range(2)]
    eng = DenoiseEngine(TINY, usd, csds, CPU, backend=cpu_ops)
    ut, ct = build_topology(TINY), build_topology(TINY, with_decoder=False)
    x, ctx, hints = make_inputs(TINY, 3, 8, 7, 9)
    for B, guided in ((1, False), (3, False), (2, False), (2, True)):
        eng.prepare(ctx[:B], [h[:B] for h in hints], [0.5, 1.0], guided=guided)
        eps = eng.eps(x[:B], 601)
        with torch.no_grad():
            ref = O.apply_model(usd, ut, [(sd, ct) for sd in csds], x[:B], torch.full((B,), 601), ctx[:B],
                                [h[:B] for h in hints], [0.5, 1.0])
        assert eps.shape == (B, 4, 8, 8)
        assert (eps - ref).abs().max().item() < 2e-4, (B, guided)


def test_engine_rejects_rows_that_do_not_fit_the_mode():
    eng = _tiny_engine()
    x, ctx, hints = make_inputs(TINY, 3, 8, 7, 9)
    with pytest.raises(ValueError):                                 # guided needs [negative; positive]
        eng.prepare(ctx, hints, [0.5, 1.0])
    with pytest.raises(ValueError):
        eng.prepare(ctx, hints, [0.5, 1.0], cfg_duplicated=True, guided=False)
    eng.prepare(ctx[:2], [h[:2] for h in hints], [0.5, 1.0])
    with pytest.raises(ValueError):                                 # 2 latents would need 4 guided rows
        eng.begin(x[:2, :4], guidance=5.0, use_graph=False)
    eng.prepare(ctx, hints, [0.5, 1.0], guided=False)
    with pytest.raises(ValueError):
        eng.begin(x[:1, :4], guidance=5.0, use_graph=False)
    eng.begin(x[:, :4], guidance=5.0, use_graph=False)
    eng.step(501, 0.3, 0.4)
    assert torch.isfinite(eng.latents()).all()


# ------------------------------------------------------------------------------------------------ operator level
def _eps_as_out_conv(e_nhwc):
    """(xn, w, bias) whose out conv gives back e: xn = [hi | lo] with hi = half(e), lo = half(e - hi) (the storage type
    of the CPU emulation is fp32: lo is 0 there), w = the centre tap adding channels o and o + 4 into output o."""
    h = cpu_ops.half_dtype()
    hi = e_nhwc.to(h)
    lo = (e_nhwc - hi.float()).to(h)
    xn = torch.cat([hi, lo], -1).contiguous()
    w = torch.zeros(4, 3, 3, 8)
    for o in range(4):
        w[o, 1, 1, o] = w[o, 1, 1, o + 4] = 1.0
    return xn, w, torch.zeros(4)


def test_out_ddim_emulation_matches_reference_unguided_p_sample():
    """The update ea_out_ddim implements == the reference sampler's p_sample_ddim at unconditional_guidance_scale 1
    (one model evaluation, cldm/ddim_hacked.py:187-188,203-230), batch of 3."""
    g = torch.load(os.path.join(GOLD, "ddim_nocfg.pt"))["p_sample"]
    N = g["x"].shape[0]
    xn, w, bias = _eps_as_out_conv(g["e"].permute(0, 2, 3, 1).float())
    lat = g["x"].permute(0, 2, 3, 1).contiguous().float()
    a, ap = g["a_t"], g["a_prev"]
    coef = torch.tensor([math.sqrt(a), math.sqrt(1 - a), math.sqrt(ap), math.sqrt(1 - ap)] + [0.0] * 12)
    lat_half = torch.zeros(N, 8, 8, 4)
    eps_out = torch.zeros(N, 8, 8, 4)
    cpu_ops.out_ddim(xn, w, bias, latents=lat, eps_out=eps_out, coef=coef, lat_half_out=lat_half, Nimg=N, H=8, W=8,
                     C_=8)
    ref = g["x_prev"].permute(0, 2, 3, 1)
    assert (eps_out - g["e"].permute(0, 2, 3, 1)).abs().max().item() < 1e-6
    assert (lat - ref).abs().max().item() < 1e-5
    assert torch.equal(lat_half, lat)


def test_out_buffers_are_checked_against_the_entry_point():
    """N-row buffers handed to the guided entry point (which reads row img + Nimg and writes eps / lat_half at
    gw + npix) are refused before any launch, and 2N-row buffers handed to the unguided one likewise."""
    from editanything_b200 import ops
    N, H, W, C = 3, 4, 4, 8
    xn, w, bias = torch.zeros(N, H, W, C), torch.zeros(4, 3, 3, C), torch.zeros(4)
    lat, coef = torch.zeros(N, H, W, 4), torch.zeros(16)
    with pytest.raises(ValueError, match="xn"):
        ops.out_cfg_ddim(xn, w, bias, latents=lat, coef=coef, Nimg=N, H=H, W=W, C_=C)
    with pytest.raises(ValueError, match="lat_half_out"):
        ops.out_ddim(xn, w, bias, latents=lat, coef=coef, lat_half_out=torch.zeros(2 * N, H, W, 4), Nimg=N, H=H,
                     W=W, C_=C)
    with pytest.raises(ValueError, match="eps_out"):
        ops.out_ddim(xn, w, bias, eps_out=torch.zeros(2 * N, H, W, 4), Nimg=N, H=H, W=W, C_=C)
    with pytest.raises(ValueError, match="coef"):
        ops.out_ddim(xn, w, bias, latents=lat, coef=coef[:8], hist=torch.zeros(3, N, H, W, 4), Nimg=N, H=H, W=W,
                     C_=C)
    with pytest.raises(ValueError, match="positive"):
        ops.out_ddim(xn[:0], w, bias, eps_out=torch.zeros(0, H, W, 4), Nimg=0, H=H, W=W, C_=C)


# ------------------------------------------------------------------------------------------------ application
@pytest.mark.parametrize("scale", [1.0, 0.5])
def test_process_without_guidance_with_the_tile_pass(scale, tmp_path, monkeypatch):
    """EditAnythingLoraModel.process(scale <= 1) end to end on tiny engines, tile pass included (N = 1 per tile
    call): images come back, and scale 0.5 gives exactly what 1.0 gives."""
    from editanything_b200 import app
    from editanything_b200.vae import VaeEngine, make_vae_state_dict
    from editanything_b200.vae_spec import VaeConfig
    from tests.test_app_cpu import FakeSam, _Enc, _inputs, _Tok
    monkeypatch.chdir(tmp_path)
    monkeypatch.setenv("EA_SAVE_INPUT", "0")
    vcfg = VaeConfig(ch=64, ch_mult=(1, 1, 1, 1), num_res_blocks=1)
    vsd = dict(make_vae_state_dict(vcfg, 61, part="encoder"))
    vsd.update(make_vae_state_dict(vcfg, 62))
    vae = VaeEngine(vcfg, vsd, CPU, backend=cpu_ops)
    main_eng = _tiny_engine(seed=51)
    tile_eng = DenoiseEngine(TINY, None, [make_state_dict(TINY, "controlnet", 54)], CPU, backend=cpu_ops,
                             unet_packed=main_eng.unet)
    tok, enc = _Tok(), _Enc(TINY.context_dim)

    def mk(eng):
        p = StableDiffusionControlNetInpaintPipeline(eng, vae=vae, text_encoder=enc, tokenizer=tok)
        p.scheduler = UniPCMultistepScheduler.from_config(p.scheduler.config)
        return p
    model = app.EditAnythingLoraModel(base_model_path="base", lora_model_path=None, use_blip=False,
                                      sam_generator=FakeSam(), mask_predictor=object(), tile_model=mk(tile_eng),
                                      pipe=mk(main_eng))
    args, kwargs = _inputs()
    args = args[:10] + (6,) + args[11:12] + (scale,) + args[13:]          # 6 steps, guidance scale
    kwargs = dict(kwargs, refine_alignment_ratio=0.5)
    refined, output, _, _ = model.process(*args, **kwargs)
    assert len(output) == 2 and len(refined) == 2
    assert all(i.size == (64, 64) for i in output) and all(i.size == (128, 128) for i in refined)
    assert main_eng.B == 2 and tile_eng.B == 1 and not main_eng.guided and not tile_eng.guided
    import numpy as np
    key = [np.array(i) for i in output + refined]
    if scale != 1.0:
        again = model.process(*(args[:12] + (1.0,) + args[13:]), **kwargs)
        assert all(np.array_equal(a, np.array(b)) for a, b in zip(key, again[1] + again[0]))
    assert all(a.std() > 0 for a in key)
