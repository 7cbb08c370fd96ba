"""v-prediction base models (stabilityai/stable-diffusion-2-1, 768x768: the UNet predicts v = sqrt(a) eps -
sqrt(1-a) x0) with the operators emulated on CPU (tests/cpu_ops_vpred.py): the host DDIM scheduler and the emulated
fused update against the reference sampler's own v-mode p_sample_ddim (tests/golden/ddim_vpred.pt), UniPC in v mode
against UniPC in epsilon mode on the equivalent eps, loading the prediction type from a checkpoint, and a tiny
SD2.1-shaped pipeline against a re-enactment of the reference loop with v-mode schedulers."""
import math
import os

import pytest
import torch
import torch.nn.functional as F

from editanything_b200 import _backend
from editanything_b200.denoise import DenoiseEngine, ddim_schedule
from editanything_b200.pipeline import DDIMScheduler, StableDiffusionControlNetInpaintPipeline
from editanything_b200.schedulers import UniPCMultistepScheduler
from editanything_b200.unet_spec import TINY, TINY21, build_topology, make_state_dict
from editanything_b200.vae_spec import VaeConfig
from oracle import unet_oracle as O
from oracle.inputs import make_inputs
from tests import cpu_ops_vpred as cpu_ops
from tests import synth_ckpt
from tests.test_pipeline_cpu import FakeVAE

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CPU = torch.device("cpu")
V = "v_prediction"


def _golden(name):
    return torch.load(os.path.join(GOLD, "ddim_vpred.pt"))[name]


# ------------------------------------------------------------------------------------------------ host schedulers
@pytest.mark.parametrize("name", ["guided", "unguided"])
def test_host_ddim_v_step_matches_reference_p_sample(name):
    """DDIMScheduler(prediction_type="v_prediction").step on the combined v == the reference sampler's p_sample_ddim
    for a parameterization "v" model (cldm/ddim_hacked.py:187-230)."""
    g = _golden(name)
    sch = DDIMScheduler(prediction_type=V)
    sch.set_timesteps(50)
    a, ap = sch.coefficients(g["timestep"])
    assert abs(a - g["a_t"]) < 1e-12 and abs(ap - g["a_prev"]) < 1e-12
    out = sch.step(g["v"].double(), g["timestep"], g["x"].double())
    assert (out.prev_sample - g["x_prev"].double()).abs().max().item() < 1e-6
    assert (out.pred_original_sample - g["pred_x0"].double()).abs().max().item() < 1e-6


def _as_out_conv(e_nhwc):
    """(xn, w, bias) whose out conv gives back e: xn = [hi | lo] halves, w = the centre tap adding channels o and
    o + 4 into output o (lo is 0 on the CPU emulation, whose storage type is fp32)."""
    h = cpu_ops.half_dtype()
    hi = e_nhwc.to(h)
    lo = (e_nhwc - hi.float()).to(h)
    xn = torch.cat([hi, lo], -1).contiguous()
    w = torch.zeros(4, 3, 3, 8)
    for o in range(4):
        w[o, 1, 1, o] = w[o, 1, 1, o + 4] = 1.0
    return xn, w, torch.zeros(4)


@pytest.mark.parametrize("name", ["guided", "unguided"])
def test_emulated_v_update_matches_reference_p_sample(name):
    """The update ea_out_cfg_vpred / ea_out_vpred implement (guidance combine on v, then v -> x0, eps) == the
    reference sampler; eps_out is the raw network output of every row."""
    g = _golden(name)
    N = g["x"].shape[0]
    nhwc = lambda t: t.permute(0, 2, 3, 1).float().contiguous()       # noqa: E731
    guided = name == "guided"
    raw = torch.cat([nhwc(g["v_uncond"]), nhwc(g["v_cond"])]) if guided else nhwc(g["v"])
    xn, w, bias = _as_out_conv(raw)
    lat = nhwc(g["x"])
    a, ap = g["a_t"], g["a_prev"]
    coef = torch.tensor([math.sqrt(a), math.sqrt(1 - a), math.sqrt(ap), math.sqrt(1 - ap)] + [0.0] * 12)
    rows = raw.shape[0]
    eps_out, lat_half = torch.zeros(rows, 8, 8, 4), torch.zeros(rows, 8, 8, 4)
    kw = dict(latents=lat, eps_out=eps_out, coef=coef, lat_half_out=lat_half, Nimg=N, H=8, W=8, C_=8, prediction=V)
    if guided:
        cpu_ops.out_cfg_ddim(xn, w, bias, guidance=g["guidance"], **kw)
    else:
        cpu_ops.out_ddim(xn, w, bias, **kw)
    assert (eps_out - raw).abs().max().item() < 1e-6
    assert (lat - nhwc(g["x_prev"])).abs().max().item() < 1e-5
    assert torch.equal(lat_half, torch.cat([lat] * (2 if guided else 1)))


@pytest.mark.parametrize("solver_order", [1, 2])
def test_unipc_v_equals_unipc_eps_on_the_equivalent_eps(solver_order):
    """UniPC in v mode on outputs v == UniPC in epsilon mode on eps = alpha_t v + sigma_t x (x = that run's own
    sample), step for step in float64: the only difference between the modes is the x0 conversion."""
    base = DDIMScheduler().config
    sv = UniPCMultistepScheduler.from_config(base, prediction_type=V, solver_order=solver_order)
    se = UniPCMultistepScheduler.from_config(base, solver_order=solver_order)
    assert sv.config.prediction_type == V and se.config.prediction_type == "epsilon"
    for s in (sv, se):
        s.set_timesteps(15)
    g = torch.Generator().manual_seed(3)
    xv = xe = torch.randn(2, 4, 8, 8, generator=g, dtype=torch.float64)
    for t in sv.timesteps.tolist():
        v = torch.randn(2, 4, 8, 8, generator=g, dtype=torch.float64)
        ov = sv.step(v, t, xv)
        oe = se.step(float(se.alpha_t[t]) * v + float(se.sigma_t[t]) * xe, t, xe)
        assert (ov.pred_original_sample - oe.pred_original_sample).abs().max().item() < 1e-12
        assert (ov.prev_sample - oe.prev_sample).abs().max().item() < 1e-11, t
        xv, xe = ov.prev_sample, oe.prev_sample


def test_host_ddim_v_equals_eps_on_the_equivalent_eps():
    sv, se = DDIMScheduler(prediction_type=V), DDIMScheduler()
    for s in (sv, se):
        s.set_timesteps(10)
    g = torch.Generator().manual_seed(4)
    xv = xe = torch.randn(1, 4, 8, 8, generator=g, dtype=torch.float64)
    for t in sv.timesteps.tolist():
        v = torch.randn(1, 4, 8, 8, generator=g, dtype=torch.float64)
        a = sv.coefficients(t)[0]
        xv = sv.step(v, t, xv).prev_sample
        xe = se.step(math.sqrt(a) * v + math.sqrt(1 - a) * xe, t, xe).prev_sample
        assert (xv - xe).abs().max().item() < 1e-11


def test_schedulers_reject_what_they_cannot_run():
    for bad in ("sample", "v", "bogus"):
        with pytest.raises(NotImplementedError):
            DDIMScheduler(prediction_type=bad)
        with pytest.raises(NotImplementedError):
            UniPCMultistepScheduler(prediction_type=bad)
    with pytest.raises(NotImplementedError):
        UniPCMultistepScheduler(prediction_type=V, thresholding=True)
    assert DDIMScheduler().config.prediction_type == "epsilon"


def test_operators_reject_unknown_prediction_before_launch():
    from editanything_b200 import ops
    N, H, W, C = 1, 4, 4, 8
    xn, w, bias = torch.zeros(2 * N, H, W, C), torch.zeros(4, 3, 3, C), torch.zeros(4)
    lat, coef = torch.zeros(N, H, W, 4), torch.zeros(16)
    for fn, x in ((ops.out_cfg_ddim, xn), (ops.out_ddim, xn[:N]), (cpu_ops.out_cfg_ddim, xn), (cpu_ops.out_ddim, xn[:N])):
        with pytest.raises(ValueError, match="prediction"):
            fn(x, w, bias, latents=lat, coef=coef, Nimg=N, H=H, W=W, C_=C, prediction="sample")
    assert torch.equal(lat, torch.zeros_like(lat))


# ------------------------------------------------------------------------------------------------ loading
VCFG = VaeConfig(ch=64, ch_mult=(1, 1, 1, 1), num_res_blocks=1)
SD21 = "stabilityai/stable-diffusion-2-1"


def _write_sd21(root, prediction_type):
    """A diffusers-layout SD2.1-shaped base model whose scheduler_config.json names `prediction_type` like the real
    one's ("v_prediction" for the 768x768 model)."""
    import json
    path = os.path.join(root, *SD21.split("/"))
    usd, _ = synth_ckpt.write_pipeline(path, TINY21, VCFG, seed=91)
    sp = os.path.join(path, "scheduler", "scheduler_config.json")
    sc = json.load(open(sp))
    if prediction_type is not None:
        sc.update(_class_name="DDIMScheduler", prediction_type=prediction_type)
    json.dump(sc, open(sp, "w"))
    return usd


@pytest.fixture
def cpu_backend():
    _backend.OPS = cpu_ops
    yield
    _backend.OPS = None


def test_loader_reads_prediction_type(tmp_path, monkeypatch, cpu_backend):
    from editanything_b200.loading import ControlNetModel2
    _write_sd21(str(tmp_path), V)
    synth_ckpt.write_unet_like(os.path.join(str(tmp_path), "shgao", "edit-anything-v0-4-sd21"), TINY21, "controlnet", 92)
    monkeypatch.setenv("EA_MODEL_ROOT", str(tmp_path))
    cn = ControlNetModel2.from_pretrained("shgao/edit-anything-v0-4-sd21")
    pipe = StableDiffusionControlNetInpaintPipeline.from_pretrained(SD21, controlnet=[cn], torch_dtype=torch.float16,
                                                                   safety_checker=None)
    assert isinstance(pipe.scheduler, DDIMScheduler) and pipe.scheduler.config.prediction_type == V
    assert UniPCMultistepScheduler.from_config(pipe.scheduler.config).config.prediction_type == V
    # share_with: the tile-style pipeline of another (epsilon) base model keeps its own prediction type
    synth_ckpt.write_pipeline(os.path.join(str(tmp_path), "runwayml", "stable-diffusion-v1-5"), TINY, VCFG, seed=51)
    synth_ckpt.write_unet_like(os.path.join(str(tmp_path), "lllyasviel", "control_v11f1e_sd15_tile"), TINY,
                               "controlnet", 54)
    sd15 = StableDiffusionControlNetInpaintPipeline.from_pretrained(
        "runwayml/stable-diffusion-v1-5", controlnet=ControlNetModel2.from_pretrained("lllyasviel/control_v11f1e_sd15_tile"))
    assert sd15.scheduler.config.prediction_type == "epsilon"


@pytest.mark.parametrize("prediction_type", [None, "epsilon", "sample", "bogus"])
def test_loader_prediction_type_default_and_rejection(prediction_type, tmp_path, monkeypatch, cpu_backend):
    """Today's checkpoints (no prediction_type, or "epsilon") load as epsilon; a prediction type the sampler cannot run
    raises while loading."""
    from editanything_b200.loading import load_pipeline_parts
    _write_sd21(str(tmp_path), prediction_type)
    root = os.path.join(str(tmp_path), *SD21.split("/"))
    if prediction_type in (None, "epsilon"):
        sched = load_pipeline_parts(root, CPU)[-1]
        assert sched.config.prediction_type == "epsilon"
    else:
        with pytest.raises(NotImplementedError, match="prediction_type"):
            load_pipeline_parts(root, CPU)


# ------------------------------------------------------------------------------------------------ pipeline (TINY21)
def _setup(scheduler):
    cfg = TINY21
    usd = make_state_dict(cfg, "unet", 61)
    csds = [make_state_dict(cfg, "controlnet", 62)]
    eng = DenoiseEngine(cfg, usd, csds, CPU, backend=cpu_ops)
    pipe = StableDiffusionControlNetInpaintPipeline(eng, vae=FakeVAE(), scheduler=scheduler)
    g = torch.Generator().manual_seed(0)
    image = torch.rand(1, 3, 64, 64, generator=g) * 2 - 1
    mask = torch.zeros(1, 1, 64, 64)
    mask[:, :, 16:48, 8:40] = 1.0
    conds = [torch.randint(0, 256, (1, 3, 64, 64), generator=g).float()]
    pe = torch.randn(1, 9, cfg.context_dim, generator=g)
    ne = torch.randn(1, 9, cfg.context_dim, generator=g)
    return cfg, usd, csds, pipe, image, mask, conds, pe, ne


def _make_scheduler(kind):
    d = DDIMScheduler(prediction_type=V)
    return d if kind == "ddim" else UniPCMultistepScheduler.from_config(d.config)


def reference_loop_v(cfg, usd, csds, image, mask, conds, pe, ne, *, steps, gs, seed, alignment_ratio, scheduler):
    """The reference __call__ (in_channels == 4) on a v-prediction base model: the networks' output (v) combined for
    guidance (:1627-1631) and handed to the scheduler, whose step converts it (diffusers' prediction_type
    "v_prediction"); the blend as for any base model (:1647-1664)."""
    do_cfg = gs > 1.0
    copies = 2 if do_cfg else 1
    sch = scheduler
    sch.set_timesteps(steps)
    ts = sch.timesteps
    ctx = torch.cat([ne, pe]) if do_cfg else pe
    hints = [torch.cat([c] * copies) for c in conds]
    lat = torch.randn((1, 4, 8, 8), generator=torch.Generator().manual_seed(seed))
    noise = lat
    init = 0.18215 * FakeVAE().encode(image).latent_dist.sample()
    m = 1 - F.interpolate((mask >= 0.5).float(), (8, 8), mode="nearest")
    ut, ct = build_topology(cfg), build_topology(cfg, with_decoder=False)
    for i, t in enumerate(ts):
        with torch.no_grad():
            out = O.apply_model(usd, ut, [(sd, ct) for sd in csds], torch.cat([lat] * copies),
                                torch.full((copies,), int(t)), ctx, hints, [1.0])
        v = out[:1] + gs * (out[1:] - out[:1]) if do_cfg else out
        lat = sch.step(v, t, lat).prev_sample
        if alignment_ratio is not None and i < len(ts) * alignment_ratio:
            lat = sch.add_noise(init, noise, ts[i + 1]) * m + lat * (1 - m)
    if alignment_ratio is None or alignment_ratio == 1.0:
        lat = init * m + lat * (1 - m)
    return lat


def _call(pipe, image, mask, conds, pe, ne, gs, steps, alignment_ratio):
    return pipe(image=image, mask_image=mask, controlnet_conditioning_image=conds, height=64, width=64,
                num_inference_steps=steps, guidance_scale=gs, generator=torch.manual_seed(7), prompt_embeds=pe,
                negative_prompt_embeds=ne, output_type="latent", controlnet_conditioning_scale=1.0,
                alignment_ratio=alignment_ratio).images


@pytest.mark.parametrize("alignment_ratio", [None, 0.5])
@pytest.mark.parametrize("kind", ["ddim", "unipc"])
@pytest.mark.parametrize("gs", [7.5, 1.0])
def test_tiny21_v_pipeline_matches_reference_loop(gs, kind, alignment_ratio):
    steps = 4 if kind == "ddim" else 6
    cfg, usd, csds, pipe, image, mask, conds, pe, ne = _setup(_make_scheduler(kind))
    out = _call(pipe, image, mask, conds, pe, ne, gs, steps, alignment_ratio)
    assert pipe.engine.prediction_type == V and pipe.engine.guided == (gs > 1.0)
    ref = reference_loop_v(cfg, usd, csds, image, mask, conds, pe, ne, steps=steps, gs=gs, seed=7,
                           alignment_ratio=alignment_ratio, scheduler=_make_scheduler(kind))
    assert out.shape == (1, 4, 8, 8)
    assert (out - ref).abs().max().item() < 5e-4, (out - ref).abs().max().item()
    # the same weights read as an epsilon model sample something else: the prediction type reached the update
    eps_ref = reference_loop_v(cfg, usd, csds, image, mask, conds, pe, ne, steps=steps, gs=gs, seed=7,
                               alignment_ratio=alignment_ratio,
                               scheduler=DDIMScheduler() if kind == "ddim" else
                               UniPCMultistepScheduler.from_config(DDIMScheduler().config))
    assert (out - eps_ref).abs().max().item() > 1e-2


class _OtherScheduler:
    """A v-mode scheduler behind another class: the pipeline's non-fused path (engine.eps + scheduler.step)."""

    def __init__(self):
        self._s = DDIMScheduler(prediction_type=V)
        self.order, self.init_noise_sigma, self.config = 1, 1.0, self._s.config

    def set_timesteps(self, n, device=None):
        self._s.set_timesteps(n)
        self.timesteps = self._s.timesteps

    def scale_model_input(self, x, t):
        return x

    def step(self, e, t, x, **kw):
        return self._s.step(e, t, x)

    def add_noise(self, a, b, t):
        return self._s.add_noise(a, b, t)


@pytest.mark.parametrize("gs", [7.5, 1.0])
def test_fused_v_equals_the_non_fused_path(gs):
    cfg, usd, csds, pipe, image, mask, conds, pe, ne = _setup(DDIMScheduler(prediction_type=V))
    fused = _call(pipe, image, mask, conds, pe, ne, gs, 4, 0.5)
    pipe.scheduler = _OtherScheduler()
    generic = _call(pipe, image, mask, conds, pe, ne, gs, 4, 0.5)
    assert (fused - generic).abs().max().item() < 1e-4


# ------------------------------------------------------------------------------------------------ engine
def _request(eng, prediction_type, seed, guided=True, steps=4):
    x, ctx, hints = make_inputs(TINY21, 2, 8, 7, seed, n_controlnets=1)
    if not guided:
        ctx, hints = ctx[1:], [h[1:] for h in hints]
    ts, a, ap = ddim_schedule(steps)
    eng.prepare(ctx, hints, [1.0], guided=guided)
    eng.set_schedule(ts, a, ap, prediction_type=prediction_type)
    eng.begin(x[:1, :4], guidance=6.0, use_graph=False)
    for _ in ts:
        eng.step()
    return eng.latents()


def _engine():
    return DenoiseEngine(TINY21, make_state_dict(TINY21, "unet", 61), [make_state_dict(TINY21, "controlnet", 62)], CPU,
                         backend=cpu_ops)


def test_engine_switches_prediction_type_and_keeps_eps_raw():
    """epsilon -> v -> epsilon (guided and unguided) on one engine equals fresh engines; eps() returns the raw
    network output in either mode; an unknown prediction type is refused."""
    eng = _engine()
    for k, (pt, guided) in enumerate([("epsilon", True), (V, True), (V, False), ("epsilon", False), ("epsilon", True)]):
        got = _request(eng, pt, 20 + k, guided)
        assert eng.prediction_type == pt
        assert torch.equal(got, _request(_engine(), pt, 20 + k, guided)), (k, pt, guided)
    assert not torch.equal(_request(eng, V, 30), _request(eng, "epsilon", 30))
    x, ctx, hints = make_inputs(TINY21, 2, 8, 7, 9, n_controlnets=1)
    eng.prepare(ctx, hints, [1.0])
    eng.set_schedule(*ddim_schedule(4), prediction_type=V)
    ut, ct = build_topology(TINY21), build_topology(TINY21, with_decoder=False)
    usd, csd = make_state_dict(TINY21, "unet", 61), make_state_dict(TINY21, "controlnet", 62)
    with torch.no_grad():
        ref = O.apply_model(usd, ut, [(csd, ct)], x, torch.full((2,), 601), ctx, hints, [1.0])
    assert (eng.eps(x, 601) - ref).abs().max().item() < 2e-4
    with pytest.raises(ValueError, match="prediction_type"):
        eng.set_schedule(*ddim_schedule(4), prediction_type="sample")
