"""The alpha-mixing inpaint pipeline (StableDiffusionControlNetInpaintMixingPipeline, editanything_b200/pipeline.py)
with the operators emulated on CPU (tests/cpu_ops_mixing.py): against the float64 restatement of the reference's
__call__ (tests/mixing_ref.py) over alpha_weight, alignment_ratio, DDIM / UniPC / a generic scheduler, guidance, two
images and the scale map; the 9-channel branch; the order of its random draws; its callback; the engine's extra
launch; EditAnythingLoraModel.process with mixing pipelines against the reference's own process
(tests/golden/host_mixing.pt); and the compat import."""
import os
import sys

import numpy as np
import pytest
import torch

from editanything_b200 import app, ops
from editanything_b200.denoise import DenoiseEngine
from editanything_b200.pipeline import (DDIMScheduler, StableDiffusionControlNetInpaintMixingPipeline,
                                        StableDiffusionControlNetInpaintPipeline)
from editanything_b200.schedulers import UniPCMultistepScheduler
from editanything_b200.unet_spec import TINY, TINY21, TINY21_INPAINT, make_state_dict
from tests import cpu_ops_mixing as cpu_ops
from tests.inpaint_ref import RecordingVAE, reference_loop_9ch
from tests.mixing_ref import mix_ref, reference_mixing
from tests.test_app_cpu import SpyPipe, _inputs, _model
from tests.test_nocfg_cpu import OtherDDIM

CPU = torch.device("cpu")
TOL = 1e-3
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "host_mixing.pt")


def _setup(n_cn=2, cfg=TINY, H=64, W=64):
    usd = make_state_dict(cfg, "unet", 51)
    ccfg = TINY21 if cfg is TINY21_INPAINT else cfg
    csds = [make_state_dict(ccfg, "controlnet", 52 + i) for i in range(n_cn)]
    eng = DenoiseEngine(cfg, usd, csds, CPU, backend=cpu_ops)
    pipe = StableDiffusionControlNetInpaintMixingPipeline(eng, vae=RecordingVAE())
    g = torch.Generator().manual_seed(0)
    image = torch.rand(1, 3, H, W, generator=g) * 2 - 1
    mask = torch.zeros(1, 1, H, W)
    mask[:, :, H // 4:3 * H // 4, W // 8:5 * W // 8] = 1.0
    conds = [torch.randint(0, 256, (1, 3, H, W), generator=g).float(), torch.rand(1, 3, H, W, generator=g)][:n_cn]
    pe = torch.randn(1, 9, ccfg.context_dim, generator=g)
    ne = torch.randn(1, 9, ccfg.context_dim, generator=g)
    return usd, csds, pipe, image, mask, conds, pe, ne


def _scale_map(H=64, W=64):
    return torch.linspace(0.2, 1.0, W)[None, None, None, :].expand(1, 1, H, W).contiguous()


def _call(pipe, image, mask, conds, pe, ne, *, steps=4, gs=7.0, scales=None, seed=7, n_img=1, **kw):
    H, W = image.shape[2], image.shape[3]
    scales = scales if scales is not None else [1.0] * len(conds)
    return pipe(image=image, mask_image=mask, controlnet_conditioning_image=conds, height=H, width=W,
                num_inference_steps=steps, guidance_scale=gs, generator=torch.manual_seed(seed), prompt_embeds=pe,
                negative_prompt_embeds=ne, output_type="latent", controlnet_conditioning_scale=scales,
                num_images_per_prompt=n_img, **kw).images


def _ref(usd, csds, image, mask, conds, pe, ne, *, steps=4, gs=7.0, scales=None, smap=None, seed=7, **kw):
    scales = scales if scales is not None else [1.0] * len(conds)
    if smap is not None:
        scales = [s * smap for s in scales]
    return reference_mixing(TINY, usd, csds, image, mask, conds, pe, ne, steps=steps, gs=gs, scales=scales, seed=seed,
                            vae=RecordingVAE(), **kw)


def _err(a, b):
    return (a.double() - b.double()).abs().max().item()


# ------------------------------------------------------------------------------------------------ the pipeline
@pytest.mark.parametrize("ratio", [0.95, 0.5, 1.0])
@pytest.mark.parametrize("alpha", [0.0, 0.5, 1.0])
def test_matches_reference_ddim(alpha, ratio):
    """4 steps: S * ratio = 3.8, 2.0 and 4.0 (every mix in the window, and no IndexError at ratio 1)."""
    usd, csds, pipe, image, mask, conds, pe, ne = _setup()
    out = _call(pipe, image, mask, conds, pe, ne, scales=[0.5, 1.0], alpha_weight=alpha, alignment_ratio=ratio)
    ref = _ref(usd, csds, image, mask, conds, pe, ne, scales=[0.5, 1.0], alpha=alpha, ratio=ratio)
    assert out.shape == (1, 4, 8, 8)
    assert _err(out, ref) < TOL, _err(out, ref)


@pytest.mark.parametrize("sched,gs,n_img,with_map,ratio", [
    ("unipc", 7.0, 2, True, 0.7),
    ("unipc", 1.0, 1, False, 0.95),
    ("ddim", 1.0, 2, True, 0.5),
    ("generic", 6.0, 2, True, 0.7),
    ("generic", 1.0, 1, False, 0.95),
])
def test_matches_reference_schedulers_guidance_batch_and_map(sched, gs, n_img, with_map, ratio):
    usd, csds, pipe, image, mask, conds, pe, ne = _setup()
    mk = {"ddim": DDIMScheduler, "generic": OtherDDIM,
          "unipc": lambda: UniPCMultistepScheduler.from_config(DDIMScheduler().config)}[sched]
    pipe.scheduler = mk()
    smap = _scale_map() if with_map else None
    out = _call(pipe, image, mask, conds, pe, ne, steps=5, gs=gs, scales=[0.5, 1.0], n_img=n_img, alpha_weight=0.3,
                alignment_ratio=ratio, controlnet_conditioning_scale_map=smap)
    ref = _ref(usd, csds, image, mask, conds, pe, ne, steps=5, gs=gs, scales=[0.5, 1.0], smap=smap, alpha=0.3,
               ratio=ratio, n_img=n_img, scheduler=mk())
    assert out.shape == (n_img, 4, 8, 8)
    assert pipe.engine.guided == (gs > 1.0)
    assert _err(out, ref) < TOL, _err(out, ref)
    if with_map:
        plain = _ref(usd, csds, image, mask, conds, pe, ne, steps=5, gs=gs, scales=[0.5, 1.0], alpha=0.3,
                     ratio=ratio, n_img=n_img, scheduler=mk())
        assert _err(plain, ref) > 1e-2                                       # the map changed the result


def test_single_controlnet_float_scale_times_map():
    usd, csds, pipe, image, mask, conds, pe, ne = _setup(n_cn=1)
    smap = _scale_map()[0, 0]                                                # an [H, W] map
    out = _call(pipe, image, mask, conds[0], pe, ne, scales=0.8, controlnet_conditioning_scale_map=smap)
    ref = _ref(usd, csds, image, mask, conds, pe, ne, scales=[0.8], smap=smap, alpha=0.5, ratio=0.95)
    assert _err(out, ref) < TOL, _err(out, ref)


def test_nine_channel_branch_has_no_mix():
    """A 9-channel UNet runs as in the inpaint pipeline (:1933-1953, :1996-1999): alpha_weight and alignment_ratio
    have no effect and nothing beyond the latents and the VAE sample is drawn."""
    usd, csds, pipe, image, mask, conds, pe, ne = _setup(n_cn=1, cfg=TINY21_INPAINT)
    outs = [_call(pipe, image, mask, conds, pe, ne, n_img=2, alpha_weight=a, alignment_ratio=r)
            for a, r in ((0.0, 0.95), (1.0, 0.5))]
    state = torch.default_generator.get_state()
    ref, _ = reference_loop_9ch(TINY21_INPAINT, usd, csds, image, mask, conds, pe, ne, steps=4, gs=7.0, scales=[1.0],
                                seed=7, n_img=2)
    assert torch.equal(torch.default_generator.get_state(), state)        # the restatement drew what the pipeline did
    assert torch.equal(outs[0], outs[1])
    assert _err(outs[0], ref) < TOL


# ------------------------------------------------------------------------------------------------ random draws
def test_predrawn_noise_table_equals_step_by_step_draws():
    """The fused loop draws the S - 1 mixes' noise before the first step; nothing else draws from the generator in
    between, so the table equals the draws the reference makes one per step."""
    init = torch.randn(2, 4, 8, 8)
    torch.manual_seed(123)
    table = torch.stack([torch.randn_like(init) for _ in range(5)])
    torch.manual_seed(123)
    steps = []
    x = init.clone()
    for _ in range(5):
        x = 0.9 * x + 0.1                                                    # the step's arithmetic draws nothing
        steps.append(torch.randn_like(init))
    assert torch.equal(table, torch.stack(steps))


@pytest.mark.parametrize("sched", ["ddim", "unipc", "generic"])
def test_draw_count_and_order(sched):
    """After the call the global generator is where the reference leaves it: the latents, the VAE sample, then
    1 + (S - 1) draws of the init latents' shape."""
    usd, csds, pipe, image, mask, conds, pe, ne = _setup()
    mk = {"ddim": DDIMScheduler, "generic": OtherDDIM,
          "unipc": lambda: UniPCMultistepScheduler.from_config(DDIMScheduler().config)}[sched]
    pipe.scheduler = mk()
    _call(pipe, image, mask, conds, pe, ne, steps=5, n_img=2)
    got = torch.default_generator.get_state()
    g = torch.manual_seed(7)
    torch.randn((2, 4, 8, 8), generator=g)
    torch.randn((1, 4, 8, 8), generator=g)                                   # RecordingVAE's sample of one image
    for _ in range(len(pipe.scheduler.timesteps)):
        torch.randn((2, 4, 8, 8))
    assert torch.equal(got, torch.default_generator.get_state())


def test_callback_sees_the_unmixed_latents():
    usd, csds, pipe, image, mask, conds, pe, ne = _setup()
    seen = []
    out = _call(pipe, image, mask, conds, pe, ne, steps=5, alpha_weight=0.4, alignment_ratio=0.5,
                callback=lambda i, t, x: seen.append((i, x.clone())), callback_steps=2)
    pre = []
    ref = _ref(usd, csds, image, mask, conds, pe, ne, steps=5, alpha=0.4, ratio=0.5, seen=pre)
    assert [i for i, _ in seen] == [0, 2, 4]
    for i, x in seen:
        assert _err(x, pre[i]) < TOL
    assert _err(out, ref) < TOL
    fused = _call(pipe, image, mask, conds, pe, ne, steps=5, alpha_weight=0.4, alignment_ratio=0.5)
    assert _err(out, fused) < 1e-5


# ------------------------------------------------------------------------------------------------ the engine
def _engine_pair():
    from oracle.inputs import make_inputs
    usd = make_state_dict(TINY, "unet", 61)
    csds = [make_state_dict(TINY, "controlnet", 62)]
    eng = DenoiseEngine(TINY, usd, csds, CPU, backend=cpu_ops)
    x, ctx, hints = make_inputs(TINY, 2, 8, 7, 5, n_controlnets=1)
    eng.prepare(ctx, hints, [1.0])
    return eng, x


def test_mixing_step_is_one_launch_longer_and_mixes_after_the_update():
    eng, x = _engine_pair()
    S = 3
    ts, a, ap = [801, 501, 201], [0.2, 0.5, 0.8], [0.5, 0.8, 0.95]
    g = torch.Generator().manual_seed(3)
    init, z = torch.randn(1, 4, 8, 8, generator=g), torch.randn(S - 1, 1, 4, 8, 8, generator=g)
    m = (torch.rand(1, 1, 8, 8, generator=g) > 0.5).float()
    eng.set_schedule(ts, a, ap, blend=([1.0] * S, [0.0] * S, [0.0] * S))
    eng.begin(x[:1], 7.0, known_nchw=init, mask_n1hw=m, use_graph=False)
    n0 = cpu_ops.launch_count()
    eng.step()
    plain = cpu_ops.launch_count() - n0
    upd = eng.latents()
    mix = ([0.9, 0.95, 1.0], [0.4, 0.3, 0.0], [1.0, 0.0, 1.0], [1.0, 1.0, 0.0])
    eng.set_schedule(ts, a, ap, mix=mix)
    eng.begin(x[:1], 7.0, known_nchw=init, mask_n1hw=m, use_graph=False, mix_alpha=0.25, mix_noise=z)
    lats = []
    for i in range(S):
        n0 = cpu_ops.launch_count()
        eng.step()
        assert cpu_ops.launch_count() - n0 == plain + 1
        lats.append(eng.latents())
    want = mix_ref(upd, init, m, z[0], 0.9, 0.4, True, 0.25)
    assert _err(lats[0], want) < 1e-5
    assert torch.equal(eng.x_half[:1], eng.x_half[1:]) and _err(eng.x_half[:1].permute(0, 3, 1, 2), lats[-1]) == 0.0


def test_engine_and_operator_rejections():
    eng, x = _engine_pair()
    with pytest.raises(ValueError, match="not both"):
        eng.set_schedule([501], [0.5], [0.8], blend=([1.0], [0.0], [1.0]), mix=([1.0], [0.0], [1.0], [0.0]))
    with pytest.raises(ValueError, match="one value per step"):
        eng.set_schedule([501, 201], [0.5, 0.8], [0.8, 0.9], mix=([1.0], [0.0], [1.0], [0.0]))
    eng.set_schedule([501, 201], [0.5, 0.8], [0.8, 0.9], mix=([1.0] * 2, [0.0] * 2, [1.0] * 2, [1.0, 0.0]))
    with pytest.raises(ValueError, match="mix_noise"):
        eng.begin(x[:1], 7.0, mix_alpha=0.5, mix_noise=torch.zeros(3, 1, 4, 8, 8))
    eng.begin(x[:1], 7.0, use_graph=False)
    with pytest.raises(RuntimeError, match="mix_alpha"):
        eng.step()
    px = 2 * 8 * 8
    lat, known, mask = torch.zeros(px * 4), torch.zeros(px * 4), torch.zeros(px)
    mix, ctr = torch.zeros(3, 4), torch.ones(1, dtype=torch.int32)
    ok = dict(alpha=0.5, step_counter=ctr, Nimg=2, H=8, W=8)
    cpu_ops.latent_mix(lat, known, mask, torch.zeros(3 * px * 4), mix, **ok)
    for bad in (dict(noise=torch.zeros(2 * px * 4)), dict(mask=torch.zeros(px + 1)), dict(mix=torch.zeros(3, 5)),
                dict(lat_half_out=torch.zeros(px * 4), copies=2), dict(copies=3)):
        kw = dict(latents=lat, known=known, mask=mask, noise=torch.zeros(3 * px * 4), mix=mix, **ok)
        kw.update(bad)
        with pytest.raises(ValueError):
            ops.latent_mix(**kw)                 # refused by the shared checks before the library is touched


def test_rejections():
    usd, csds, pipe, image, mask, conds, pe, ne = _setup()
    with pytest.raises(NotImplementedError):
        _call(pipe, image, mask, conds, pe, ne, eta=0.5)
    with pytest.raises(TypeError):
        _call(pipe, image, mask, conds, pe, ne, guess_mode=True)               # not in the reference's signature
    with pytest.raises(TypeError):
        _call(pipe, image, mask, conds, pe, ne, alignment_ratio=None)          # i < S * None, as in the reference


# ------------------------------------------------------------------------------------------------ process()
class SpyMixingPipe(StableDiffusionControlNetInpaintMixingPipeline):
    """tests/test_app_cpu.SpyPipe that is a mixing pipeline (process() takes its mixing branch)."""
    _execution_device = None                  # a plain attribute, set by SpyPipe.__init__
    __init__ = SpyPipe.__init__
    __call__ = SpyPipe.__call__


class SpyPlainPipe(StableDiffusionControlNetInpaintPipeline):
    """A SpyPipe with the plain inpaint pipeline's signature: alpha_weight is a TypeError."""
    _execution_device = None
    __init__ = SpyPipe.__init__

    def __call__(self, image=None, mask_image=None, controlnet_conditioning_image=None, height=None, width=None,
                 num_inference_steps=50, guidance_scale=7.5, num_images_per_prompt=1, generator=None,
                 prompt_embeds=None, negative_prompt_embeds=None, controlnet_conditioning_scale=1.0,
                 alignment_ratio=None, guess_mode=False):
        kw = {k: v for k, v in locals().items() if k != "self"}
        return SpyPipe.__call__(self, **kw)


def run_mixing_process(cls, use_scale_map, tile_cls=SpyMixingPipe):
    """process() of `cls` with mixing spy pipelines on tests/test_app_cpu's inputs, alpha_weight 0.3."""
    args, kwargs = _inputs()
    kwargs = dict(kwargs, alpha_weight=0.3, use_scale_map=use_scale_map)
    pipe, tile = SpyMixingPipe(), tile_cls()
    model = _model(cls, pipe, tile)
    np.random.seed(5)
    return pipe.calls, tile.calls, model.process(*args, **kwargs)


@pytest.mark.parametrize("use_scale_map", [False, True])
def test_process_hands_the_mixing_pipelines_exactly_what_the_reference_does(use_scale_map, monkeypatch):
    from tests.test_host_semantics_cpu import fingerprint
    monkeypatch.setenv("EA_SAVE_INPUT", "0")
    ref = torch.load(GOLD, weights_only=False)[f"scale_map={use_scale_map}"]
    calls, tile_calls, (o_tile, o_res, o_masks, o_prompt) = run_mixing_process(app.EditAnythingLoraModel,
                                                                               use_scale_map)
    assert len(calls) == len(ref["calls"]) == 1 and len(tile_calls) == len(ref["tile_calls"]) == 2
    for rc, oc in zip(ref["calls"] + ref["tile_calls"], calls + tile_calls):
        assert sorted(rc) == sorted(oc)
        for k in oc:
            assert fingerprint(oc[k]) == rc[k], k
    assert fingerprint(o_tile) == ref["results_tile"] and fingerprint(o_res) == ref["results"]
    assert fingerprint(o_masks) == ref["masks"] and o_prompt == ref["prompt"]
    main, tile = calls[0], tile_calls[0]
    assert main["alpha_weight"] == tile["alpha_weight"] == 0.3 and "guess_mode" not in main
    assert tile["alignment_ratio"] == 0.95
    smap = main["controlnet_conditioning_scale_map"]
    assert (smap is None) != use_scale_map
    if use_scale_map:                                   # the main pass's map, at the main pass's size, for the tile too
        assert smap.shape == (1, 1, 64, 64) and tile["controlnet_conditioning_scale_map"] is smap
        assert set(smap.unique().tolist()) == {0.0, 1.0}


def test_process_with_a_plain_tile_pipeline_raises_type_error(monkeypatch):
    monkeypatch.setenv("EA_SAVE_INPUT", "0")
    with pytest.raises(TypeError, match="alpha_weight"):
        run_mixing_process(app.EditAnythingLoraModel, False, tile_cls=SpyPlainPipe)


def test_alpha_mixing_constructor_argument_is_still_refused():
    with pytest.raises(NotImplementedError):
        app.EditAnythingLoraModel(alpha_mixing=True)


def test_compat_import():
    from editanything_b200 import compat
    root = os.path.dirname(os.path.abspath(compat.__file__))
    sys.path.insert(0, root)
    try:
        sys.modules.pop("utils", None)
        sys.modules.pop("utils.stable_diffusion_controlnet_inpaint", None)
        from utils.stable_diffusion_controlnet_inpaint import StableDiffusionControlNetInpaintMixingPipeline as M
    finally:
        sys.path.remove(root)
        sys.modules.pop("utils", None)
        sys.modules.pop("utils.stable_diffusion_controlnet_inpaint", None)
    assert M is StableDiffusionControlNetInpaintMixingPipeline
