"""Text-to-image ControlNet pipelines (all-region generation) with the operators emulated on CPU
(tests/cpu_ops_vpred.py): StableDiffusionControlNetPipeline / StableDiffusionControlNetPipeline2 against a line-by-line
re-enactment of the reference's Pipeline2.__call__ (utils/stable_diffusion_controlnet.py:465-662) on the oracle
networks - guess mode with guidance re-enacted as two oracle calls, the unconditional rows without ControlNets and the
conditional rows with them (:579-602) - the reference sampler's own guess-mode step (tests/golden/t2i_guess.pt),
EditAnythingLoraModel.process(enable_all_generate=True) and the rejections."""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from editanything_b200 import _backend, app
from editanything_b200.denoise import DenoiseEngine
from editanything_b200.pipeline import (DDIMScheduler, StableDiffusionControlNetInpaintPipeline,
                                        StableDiffusionControlNetPipeline, StableDiffusionControlNetPipeline2,
                                        randn_tensor)
from editanything_b200.schedulers import UniPCMultistepScheduler
from editanything_b200.unet_spec import TINY, TINY21, TINY21_INPAINT, build_topology, make_state_dict
from oracle import unet_oracle as O
from tests import cpu_ops_vpred as cpu_ops
from tests.test_app_cpu import SpyPipe, _Enc, _inputs, _model, _Tok
from tests.test_nocfg_cpu import OtherDDIM
from tests.test_pipeline_cpu import FakeVAE

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CPU = torch.device("cpu")
TOL = 2e-4


def _pipe(cfg=TINY, n_cn=1, cls=StableDiffusionControlNetPipeline2, seed=51, **kw):
    usd = make_state_dict(cfg, "unet", seed)
    csds = [make_state_dict(cfg if cfg.in_channels == 4 else TINY21, "controlnet", seed + 1 + i) for i in range(n_cn)]
    eng = DenoiseEngine(cfg, usd, csds, CPU, backend=cpu_ops)
    return cls(eng, vae=FakeVAE(), **kw), usd, csds


def _cond(n=1, seed=0, hw=64):
    g = torch.Generator().manual_seed(seed)
    c = torch.randint(0, 256, (n, 3, hw, hw), generator=g).float()
    c[:, 2] = 0
    return c


class _ListTok(_Tok):
    """tests/test_app_cpu._Tok over a list of prompts."""

    def __call__(self, text, **kw):
        rows = [super(_ListTok, self).__call__(t, **kw).input_ids for t in ([text] if isinstance(text, str) else text)]
        return SimpleNamespace(input_ids=torch.cat(rows))


def _embeds(cfg, n_prompts=1, L=9, seed=3):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n_prompts, L, cfg.context_dim, generator=g), torch.randn(n_prompts, L, cfg.context_dim, generator=g)


def _apply(usd, ut, cns, x_unet, x_cn, t, ctx, hints, scales, guess):
    """oracle.unet_oracle.apply_model with the ControlNets reading their own input x_cn (:579-582)."""
    if not cns:
        return O.unet_forward(usd, ut, x_unet, t, ctx, None)
    if x_cn is x_unet:
        return O.apply_model(usd, ut, cns, x_unet, t, ctx, hints, scales, guess_mode=guess)
    control = None
    for (sd, ct), hint, s in zip(cns, hints, scales):
        outs = O.controlnet_forward(sd, ct, x_cn, hint, t, ctx)
        f = torch.logspace(-1, 0, len(outs)) * s if guess else [s] * len(outs)
        outs = [o * float(fi) for o, fi in zip(outs, f)]
        control = outs if control is None else [a + b for a, b in zip(control, outs)]
    return O.unet_forward(usd, ut, x_unet, t, ctx, control)


def reference_t2i(cfg, usd, csds, pe, ne, images, scales, *, steps, guidance, guess, generator, nipp=1,
                  scheduler=None, seen=None):
    """Pipeline2.__call__ (:465-627) on the oracle networks.  pe / ne: the prompt embeddings of the batch_size
    prompts; images: one [1 or batch_size, 3, H, W] tensor per net; scales: one float or map per net (the map already
    multiplied in, :490-495)."""
    sch = scheduler if scheduler is not None else DDIMScheduler()
    bs = pe.shape[0]
    N = bs * nipp
    do_cfg = guidance > 1.0
    pos = pe.repeat(1, nipp, 1).view(N, *pe.shape[1:])                                   # _encode_prompt
    neg = ne.repeat(1, nipp, 1).view(N, *ne.shape[1:])
    hints = [im.repeat_interleave(N if im.shape[0] == 1 else nipp, 0) for im in images]   # prepare_image
    sch.set_timesteps(steps)
    H, W = images[0].shape[-2:]
    lat = randn_tensor((N, 4, H // 8, W // 8), generator=generator) * sch.init_noise_sigma
    ut, ct = build_topology(cfg), build_topology(cfg, with_decoder=False)
    cns = [(sd, ct) for sd in csds]
    for i, t in enumerate(sch.timesteps):
        tt = torch.full((N,), int(t))
        x_in = sch.scale_model_input(torch.cat([lat] * 2) if do_cfg else lat, t)          # :568-570
        with torch.no_grad():
            if do_cfg and guess:
                # :579-602: the ControlNets read the UNSCALED latents with the positive prompt; the unconditional rows
                # get zeros as residuals, i.e. the UNet alone
                e_u = _apply(usd, ut, [], x_in[:N], None, tt, neg, [], [], False)
                e_c = _apply(usd, ut, cns, x_in[N:], lat, tt, pos, hints, scales, True)
            elif do_cfg:
                t2 = torch.full((2 * N,), int(t))
                e = O.apply_model(usd, ut, cns, x_in, t2, torch.cat([neg, pos]), [torch.cat([h, h]) for h in hints],
                                  scales)
                e_u, e_c = e.chunk(2)
            else:
                e = O.apply_model(usd, ut, cns, x_in, tt, pos, hints, scales, guess_mode=guess)
        if do_cfg:
            e = e_u + guidance * (e_c - e_u)
        lat = sch.step(e, t, lat).prev_sample
        if seen is not None:
            seen.append(lat.clone())
    return lat


def _run(pipe, pe, ne, images, scale, *, steps=4, guidance=7.5, guess=False, seed=7, **kw):
    return pipe(prompt_embeds=pe, negative_prompt_embeds=ne, image=images, num_inference_steps=steps,
                guidance_scale=guidance, generator=torch.manual_seed(seed), output_type="latent",
                controlnet_conditioning_scale=scale, guess_mode=guess, **kw).images


# ------------------------------------------------------------------------------------------------ the pipeline
@pytest.mark.parametrize("guess", [False, True])
@pytest.mark.parametrize("guidance", [7.5, 1.0])
def test_matches_reference_call(guidance, guess):
    pipe, usd, csds = _pipe()
    pe, ne = _embeds(TINY)
    c = _cond()
    out = _run(pipe, pe, ne, [c], [0.7], guidance=guidance, guess=guess)
    ref = reference_t2i(TINY, usd, csds, pe, ne, [c], [0.7], steps=4, guidance=guidance, guess=guess,
                        generator=torch.manual_seed(7))
    eng = pipe.engine
    assert eng.guided == (guidance > 1) and eng.B == (2 if guidance > 1 else 1)
    assert eng.hints[0].shape[0] == eng.B                       # the hint stack ran once and was stacked on the device
    assert out.shape == (1, 4, 8, 8)
    assert (out - ref).abs().max().item() < TOL, (out - ref).abs().max().item()


def test_guess_mode_leaves_the_unconditional_rows_without_control():
    """eps() of a request prepared with controlnet_rows="conditional": the unconditional rows equal the UNet alone,
    the conditional rows the UNet with the guess-mode-weighted residuals."""
    pipe, usd, csds = _pipe(n_cn=2)
    eng = pipe.engine
    g = torch.Generator().manual_seed(4)
    N = 3
    x = torch.randn(N, 4, 8, 8, generator=g)
    ctx = torch.randn(2 * N, 9, TINY.context_dim, generator=g)
    hints = [_cond(N, 1), _cond(N, 2)]
    eng.prepare(ctx, hints, [0.5, 1.0], guess_mode=True, controlnet_rows="conditional")
    eps = eng.eps(torch.cat([x, x]), 601)
    ut, ct = build_topology(TINY), build_topology(TINY, with_decoder=False)
    tt = torch.full((N,), 601)
    with torch.no_grad():
        e_u = O.apply_model(usd, ut, [], x, tt, ctx[:N], [], [])
        e_c = O.apply_model(usd, ut, [(sd, ct) for sd in csds], x, tt, ctx[N:], hints, [0.5, 1.0], guess_mode=True)
    assert (eps[:N] - e_u).abs().max().item() < TOL
    assert (eps[N:] - e_c).abs().max().item() < TOL


def test_scale_map_pipeline2():
    """sketch2image.py:140-175: one ControlNet (not a list), a float scale times an [H, W] map."""
    pipe, usd, csds = _pipe()
    pe, ne = _embeds(TINY)
    c = _cond()
    smap = torch.linspace(0, 1, 64)[None, :].expand(64, 64).contiguous()
    out = pipe(prompt_embeds=pe, negative_prompt_embeds=ne, image=c, num_inference_steps=4, guidance_scale=5.0,
               generator=torch.manual_seed(7), output_type="latent", controlnet_conditioning_scale=0.9,
               controlnet_conditioning_scale_map=smap).images
    ref = reference_t2i(TINY, usd, csds, pe, ne, [c], [0.9 * smap], steps=4, guidance=5.0, guess=False,
                        generator=torch.manual_seed(7))
    assert (out - ref).abs().max().item() < TOL
    plain = _run(pipe, pe, ne, c, 0.9, guidance=5.0)
    assert (out - plain).abs().max().item() > 1e-3                                       # the map did something


@pytest.mark.parametrize("sched", ["unipc", "generic"])
def test_schedulers_guess_mode_guided(sched):
    pipe, usd, csds = _pipe()
    mk = (lambda: UniPCMultistepScheduler.from_config(DDIMScheduler().config)) if sched == "unipc" else OtherDDIM
    pipe.scheduler = mk()
    pe, ne = _embeds(TINY)
    c = _cond()
    out = _run(pipe, pe, ne, [c], [1.0], steps=4, guidance=6.0, guess=True)
    ref = reference_t2i(TINY, usd, csds, pe, ne, [c], [1.0], steps=4, guidance=6.0, guess=True,
                        generator=torch.manual_seed(7), scheduler=mk())
    assert (out - ref).abs().max().item() < 5e-4, (out - ref).abs().max().item()


class HalvingDDIM(OtherDDIM):
    """The built-in DDIM update behind a scale_model_input that halves the network input, as the sigma-based
    schedulers scale it by 1 / sqrt(sigma^2 + 1): a generic scheduler whose scale_model_input is not the identity."""

    def scale_model_input(self, x, t):
        return x * 0.5


@pytest.mark.parametrize("guidance,guess", [(6.0, False), (1.0, True)])
def test_scheduler_that_scales_the_input(guidance, guess):
    """Without guess mode, and in guess mode without guidance, every network reads scale_model_input(latents)
    (:583-584): the engine runs it."""
    pipe, usd, csds = _pipe()
    pipe.scheduler = HalvingDDIM()
    pe, ne = _embeds(TINY)
    c = _cond()
    out = _run(pipe, pe, ne, [c], [1.0], guidance=guidance, guess=guess)
    ref = reference_t2i(TINY, usd, csds, pe, ne, [c], [1.0], steps=4, guidance=guidance, guess=guess,
                        generator=torch.manual_seed(7), scheduler=HalvingDDIM())
    ident = reference_t2i(TINY, usd, csds, pe, ne, [c], [1.0], steps=4, guidance=guidance, guess=guess,
                          generator=torch.manual_seed(7), scheduler=OtherDDIM())
    assert (out - ref).abs().max().item() < TOL, (out - ref).abs().max().item()
    assert (ref - ident).abs().max().item() > 1e-2                    # the scaling matters


def test_guess_mode_with_guidance_refuses_a_scheduler_that_scales_the_input():
    """Guess mode with guidance feeds the ControlNet the unscaled latents and the UNet the scaled ones (:579-582); the
    engine's networks read one input, so such a scheduler is refused before anything runs, rather than giving the
    ControlNet the scaled latents."""
    pipe, usd, csds = _pipe()
    pipe.scheduler = HalvingDDIM()
    pe, ne = _embeds(TINY)
    with pytest.raises(NotImplementedError, match="scale_model_input"):
        _run(pipe, pe, ne, [_cond()], [1.0], guidance=6.0, guess=True)
    assert not hasattr(pipe.engine, "B")                                 # nothing was prepared or launched


@pytest.mark.parametrize("guess", [False, True])
def test_tiny21_v_prediction(guess):
    pipe, usd, csds = _pipe(cfg=TINY21, seed=61)
    pipe.scheduler = DDIMScheduler(prediction_type="v_prediction")
    pe, ne = _embeds(TINY21)
    c = _cond()
    out = _run(pipe, pe, ne, [c], [0.8], guidance=7.0, guess=guess)
    ref = reference_t2i(TINY21, usd, csds, pe, ne, [c], [0.8], steps=4, guidance=7.0, guess=guess,
                        generator=torch.manual_seed(7), scheduler=DDIMScheduler(prediction_type="v_prediction"))
    assert pipe.engine.prediction_type == "v_prediction"
    assert (out - ref).abs().max().item() < TOL, (out - ref).abs().max().item()


@pytest.mark.parametrize("guess", [False, True])
def test_prompt_strings_images_per_prompt_and_an_image_batch(guess):
    """sketch2image.py's call: a list of k prompts, num_images_per_prompt = k and k control images -> k * k rows."""
    tok, enc = _ListTok(), _Enc(TINY.context_dim)
    pipe, usd, csds = _pipe(cls=StableDiffusionControlNetPipeline2, text_encoder=enc, tokenizer=tok)
    k = 2
    prompts, negs = ["a cat, best quality"] * k, ["lowres"] * k
    c = torch.cat([_cond(1, 5), _cond(1, 6)])
    out = pipe(prompt=prompts, negative_prompt=negs, image=c, num_images_per_prompt=k, num_inference_steps=4,
               guidance_scale=7.5, generator=torch.manual_seed(7), output_type="latent",
               controlnet_conditioning_scale=1.0, guess_mode=guess).images
    pe = enc(tok(prompts, padding="max_length", max_length=tok.model_max_length).input_ids)[0]
    ne = enc(tok(negs, padding="max_length", max_length=pe.shape[1]).input_ids)[0]
    ref = reference_t2i(TINY, usd, csds, pe, ne, [c], [1.0], steps=4, guidance=7.5, guess=guess, nipp=k,
                        generator=torch.manual_seed(7))
    assert out.shape == (k * k, 4, 8, 8) and pipe.engine.B == 2 * k * k
    assert (out - ref).abs().max().item() < TOL


def test_generator_list_callbacks_and_output_types():
    pipe, usd, csds = _pipe()
    pe, ne = _embeds(TINY)
    c = _cond()
    n = 2
    gens = lambda: [torch.Generator().manual_seed(20 + i) for i in range(n)]      # noqa: E731
    seen = []
    out = pipe(prompt_embeds=pe, negative_prompt_embeds=ne, image=[c], num_images_per_prompt=n,
               num_inference_steps=4, guidance_scale=6.0, generator=gens(), output_type="latent",
               controlnet_conditioning_scale=[1.0], guess_mode=True, callback=lambda i, t, x: seen.append((i, x.clone())),
               callback_steps=2).images
    pre = []
    ref = reference_t2i(TINY, usd, csds, pe, ne, [c], [1.0], steps=4, guidance=6.0, guess=True, nipp=n,
                        generator=gens(), seen=pre)
    assert (out - ref).abs().max().item() < TOL
    assert [i for i, _ in seen] == [0, 2]
    for (i, x) in seen:
        assert (x - pre[i]).abs().max().item() < TOL
    kw = dict(prompt_embeds=pe, negative_prompt_embeds=ne, image=[c], num_inference_steps=2, guidance_scale=6.0,
              controlnet_conditioning_scale=[1.0])
    lat = pipe(generator=torch.manual_seed(3), output_type="latent", **kw).images
    arr = pipe(generator=torch.manual_seed(3), output_type="numpy", **kw).images
    pil, nsfw = pipe(generator=torch.manual_seed(3), output_type="pil", return_dict=False, **kw)
    expect = pipe.decode_latents(lat)
    assert isinstance(arr, np.ndarray) and arr.shape == (1, 64, 64, 3) and np.allclose(arr, expect)
    assert nsfw is None and len(pil) == 1 and pil[0].size == (64, 64)
    assert np.array_equal(np.array(pil[0]), (expect[0] * 255).round().astype("uint8"))


def test_the_latents_are_the_only_draw():
    """Nothing but the latents draws from the generator: the generator's state after the call is the state after one
    randn of the latent shape (the tile pass shares it, editany_lora.py:885-936)."""
    pipe, _, _ = _pipe()
    pe, ne = _embeds(TINY)
    g2 = torch.Generator().manual_seed(11)
    pipe(prompt_embeds=pe, negative_prompt_embeds=ne, image=[_cond()], num_inference_steps=2, generator=g2,
         output_type="latent", controlnet_conditioning_scale=[1.0])
    g3 = torch.Generator().manual_seed(11)
    torch.randn((1, 4, 8, 8), generator=g3)
    assert torch.equal(g2.get_state(), g3.get_state())


# ------------------------------------------------------------------------------------------------ the golden
def test_reference_guess_mode_step_golden():
    """The reference's own guided p_sample_ddim in guess mode (c_concat = None on the unconditional call), TINY
    networks: the engine's eps per half and the fused step."""
    g = torch.load(os.path.join(GOLD, "t2i_guess.pt"))
    m = g["meta"]
    usd = make_state_dict(TINY, "unet", m["unet_seed"])
    csd = make_state_dict(TINY, "controlnet", m["cn_seed"])
    eng = DenoiseEngine(TINY, usd, [csd], CPU, backend=cpu_ops)
    N = m["N"]
    eng.prepare(torch.cat([g["ctx_uncond"], g["ctx_cond"]]), [g["hint"]], [m["scale"]], guess_mode=True,
                controlnet_rows="conditional")
    eps = eng.eps(torch.cat([g["x"], g["x"]]), g["timestep"])
    assert (eps[:N] - g["e_uncond"]).abs().max().item() < TOL
    assert (eps[N:] - g["e_cond"]).abs().max().item() < TOL
    eng.begin(g["x"], m["guidance"], use_graph=False)
    eng.step(g["timestep"], g["a_t"], g["a_prev"])
    assert (eng.latents() - g["x_prev"]).abs().max().item() < 1e-3


# ------------------------------------------------------------------------------------------------ rejections
def test_rejections():
    pipe, _, _ = _pipe()
    pe, ne = _embeds(TINY)
    c = _cond()
    with pytest.raises(NotImplementedError):
        _run(pipe, pe, ne, [c], [1.0], eta=0.5)
    with pytest.raises(NotImplementedError):                     # guess mode with a map (the reference fails too)
        pipe(prompt_embeds=pe, negative_prompt_embeds=ne, image=c, controlnet_conditioning_scale=1.0,
             controlnet_conditioning_scale_map=torch.ones(64, 64), guess_mode=True, output_type="latent")
    pipe.controlnet.nets[0].config.global_pool_conditions = True
    with pytest.raises(NotImplementedError):
        _run(pipe, pe, ne, [c], [1.0])
    nine, _, _ = _pipe(cfg=TINY21_INPAINT, seed=81)
    with pytest.raises(NotImplementedError):
        _run(nine, _embeds(TINY21)[0], _embeds(TINY21)[1], [c], [1.0])
    two, _, _ = _pipe(n_cn=2)
    with pytest.raises(TypeError):
        _run(two, pe, ne, c, 1.0)                                # several nets take a list of images
    with pytest.raises(ValueError):
        _run(two, pe, ne, [c], [1.0, 1.0])
    with pytest.raises(ValueError):
        _run(two, pe, ne, [c, c], [1.0])
    single, _, _ = _pipe()
    with pytest.raises(TypeError):
        _run(single, pe, ne, c, 1)                               # one net: a float scale
    with pytest.raises(ValueError):
        _run(single, pe, ne, torch.cat([c, c, c]), 1.0)         # image batch neither 1 nor the prompt batch
    # nothing ran: every rejection comes before the engine is prepared
    assert not hasattr(pipe.engine, "B") and not hasattr(nine.engine, "B") and not hasattr(two.engine, "B")


def test_engine_rejects_conditional_rows_it_cannot_honour():
    pipe, _, _ = _pipe()
    eng = pipe.engine
    ctx = torch.randn(2, 9, TINY.context_dim)
    with pytest.raises(ValueError):
        eng.prepare(ctx[:1], [_cond()], [1.0], guided=False, controlnet_rows="conditional")
    with pytest.raises(NotImplementedError):
        eng.prepare(ctx, [_cond()], [torch.ones(64, 64)], controlnet_rows="conditional")
    with pytest.raises(ValueError):                              # the N images once, not doubled
        eng.prepare(ctx, [_cond(2)], [1.0], guess_mode=True, controlnet_rows="conditional")
    with pytest.raises(ValueError):
        eng.prepare(ctx, [_cond()], [1.0], controlnet_rows="unconditional")


def test_conditional_half_checks_alignment():
    from editanything_b200.nets import UNetRunner
    t = torch.zeros(2, 3, 3, 9, dtype=torch.float16)             # 81 halves per row: 162 bytes, not a multiple of 16
    with pytest.raises(ValueError, match="16"):
        UNetRunner.conditional_half(t)
    with pytest.raises(ValueError, match="even"):
        UNetRunner.conditional_half(torch.zeros(3, 2, 2, 8))
    v = UNetRunner.conditional_half(torch.zeros(4, 2, 2, 8, dtype=torch.float16))
    assert v.shape == (2, 2, 2, 8)


# ------------------------------------------------------------------------------------------------ application
def _spy_model(monkeypatch, extra_inpaint):
    built = []

    def fake_obtain(*a, **k):
        built.append((a, k))
        return SpyPipe()
    monkeypatch.setattr(app, "obtain_generation_model", fake_obtain)
    monkeypatch.setattr(torch.Tensor, "cuda", lambda self, *a, **k: self)
    monkeypatch.setenv("EA_SAVE_INPUT", "0")
    first = SpyPipe()
    model = _model(app.EditAnythingLoraModel, first, SpyPipe())
    model.extra_inpaint = extra_inpaint
    return model, first, built


@pytest.mark.parametrize("extra_inpaint", [True, False])
def test_process_all_region_generation_hands_the_pipelines_the_reference_arguments(monkeypatch, extra_inpaint):
    model, first, built = _spy_model(monkeypatch, extra_inpaint)
    args, kwargs = _inputs()
    args = (args[0], True) + args[2:]                           # enable_all_generate, no mask_image
    np.random.seed(5)
    tile, res, masks, prompt = model.process(*args, **kwargs)
    # rebuilt once for the mode (editany_lora.py:658-667): lora_weight not passed, the old pipeline shared
    assert len(built) == 1
    (a, k), = built
    assert a == ("base", None, app.config_dict["LAION Pretrained(v0-4)-SD15"], True, extra_inpaint)
    assert k == {"share_with": first} and model.defalut_enable_all_generate is True
    assert first.calls == [] and len(model.pipe.calls) == 1 and len(model.tile_pipe.calls) == 2
    call = model.pipe.calls[0]
    H = W = 64
    if extra_inpaint:                                           # :796-812, exactly these keywords
        assert set(call) == {"prompt_embeds", "negative_prompt_embeds", "num_images_per_prompt", "num_inference_steps",
                             "generator", "height", "width", "image", "controlnet_conditioning_scale",
                             "guidance_scale", "guess_mode", "generator_state"}
        assert call["controlnet_conditioning_scale"] == [0.5] and len(call["image"]) == 1
        assert call["image"][0].dtype == torch.float16 and call["image"][0].shape == (1, 3, H, W)
    else:
        assert np.array_equal(np.array(call["mask_image"]), np.full((H, W, 3), 255, np.uint8))
        assert call["controlnet_conditioning_scale"] == [0.5] and len(call["controlnet_conditioning_image"]) == 1
    assert (call["num_images_per_prompt"], call["num_inference_steps"], call["height"], call["width"],
            call["guidance_scale"], call["guess_mode"]) == (2, 4, H, W, 9.0, False)
    assert np.array(masks[1]).min() == 255                       # the all-white mask, also handed to the tile pass
    assert all(np.array(c["mask_image"]).min() == 255 for c in model.tile_pipe.calls)
    assert len(res) == 2 and len(tile) == 2
    # the same mode again: no rebuild; back to masked editing: rebuilt again
    model.process(*args, **kwargs)
    assert len(built) == 1
    model.process(*((args[0], False) + args[2:]), **kwargs)
    assert len(built) == 2 and built[1][0][3] is False and model.defalut_enable_all_generate is False


def test_a_mask_given_does_not_rebuild(monkeypatch):
    """With mask_image passed the reference does not rebuild the pipeline for the mode (editany_lora.py:658-678); the
    call is still chosen by enable_all_generate and extra_inpaint (:796), like there."""
    model, first, built = _spy_model(monkeypatch, True)
    args, kwargs = _inputs()
    mask = np.zeros((90, 120, 3), np.uint8)
    mask[10:40, 10:40] = 255
    model.process(*((args[0], True, mask) + args[3:]), **kwargs)
    assert built == [] and len(first.calls) == 1 and "mask_image" not in first.calls[0]
    model.process(*((args[0], False, mask) + args[3:]), **kwargs)
    assert built == [] and len(first.calls) == 2 and "mask_image" in first.calls[1]


@pytest.fixture
def vpred_backend():
    _backend.OPS = cpu_ops
    yield
    _backend.OPS = None


def test_toggle_rebuilds_from_checkpoints_and_shares_the_packed_unet(tmp_path, monkeypatch, vpred_backend):
    """obtain_generation_model on test-sized checkpoints: toggling all-region generation builds the text-to-image
    pipeline with the SAM ControlNet only, sharing the packed UNet, VAE and text encoder; toggling back builds the
    inpaint pipeline sharing them again; both generate images end to end, tile pass included."""
    from tests.test_nogradio_cpu import make_model_root
    from tests.test_app_cpu import FakeSam
    make_model_root(str(tmp_path / "hub"))
    monkeypatch.setenv("EA_MODEL_ROOT", str(tmp_path / "hub"))
    monkeypatch.setenv("EA_SAVE_INPUT", "0")
    monkeypatch.chdir(tmp_path)
    model = app.EditAnythingLoraModel(base_model_path="runwayml/stable-diffusion-v1-5", lora_model_path=None,
                                      use_blip=False, sam_generator=FakeSam(), mask_predictor=object(),
                                      extra_inpaint=True)
    main = model.pipe
    assert isinstance(main, StableDiffusionControlNetInpaintPipeline) and len(main.engine.cns) == 2
    args, kwargs = _inputs()
    args = (args[0], True) + args[2:]
    kwargs = dict(kwargs, refine_alignment_ratio=0.5)          # 4 steps: 0.95 would cover the last one
    tile, res, _, _ = model.process(*args, **kwargs)
    t2i = model.pipe
    assert isinstance(t2i, StableDiffusionControlNetPipeline) and len(t2i.engine.cns) == 1
    assert t2i.engine.unet is main.engine.unet and t2i.vae is main.vae and t2i.text_encoder is main.text_encoder
    assert len(res) == 2 and all(i.size == (64, 64) for i in res) and all(i.size == (128, 128) for i in tile)
    assert all(np.array(i).std() > 0 for i in res)
    model.process(*((args[0], False) + args[2:]), **kwargs)
    back = model.pipe
    assert isinstance(back, StableDiffusionControlNetInpaintPipeline) and len(back.engine.cns) == 2
    assert back.engine.unet is main.engine.unet
