"""-m gpu: v-prediction base models (stabilityai/stable-diffusion-2-1, 768x768).

Ordered so that a kernel defect fails before any end-to-end run: first ea_out_cfg_vpred / ea_out_vpred against
float64 (the bounds of tests/test_gpu_kernels_fp64.py and tests/fp64_refs.py), against the reference sampler's own
v-mode p_sample_ddim (tests/golden/ddim_vpred.pt) and bit for bit against the epsilon exports' eps_out; then a TINY21
engine over several DDIM and UniPC steps against the host re-enactment, one engine switching epsilon -> v -> epsilon
through CUDA-graph re-capture, one full-size SD2.1 768x768 step (N = 4 + CFG) against the float64 v update of that
engine's own network output, and the pipeline with VaeEngine (the gates of tests/test_gpu_pipeline.py)."""
import math
import os

import pytest
import torch
import torch.nn.functional as F

from editanything_b200 import ops
from editanything_b200.denoise import DenoiseEngine, ddim_schedule
from editanything_b200.pipeline import DDIMScheduler, StableDiffusionControlNetInpaintPipeline
from editanything_b200.schedulers import UniPCMultistepScheduler
from editanything_b200.unet_spec import SD21, TINY21, build_topology, make_state_dict
from oracle import unet_oracle as O
from oracle.inputs import make_inputs
from tests import fp64_refs as R
from tests.test_gpu_kernels_fp64 import DEV, U, _close, _gen, _out_conv_inputs, _randn

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
V = "v_prediction"
KERNEL = {True: "ea_out_cfg_vpred", False: "ea_out_vpred"}


def _launch(guided, xn, w, bias, N, H, W, C, g=7.5, prediction=V, **kw):
    if guided:
        ops.out_cfg_ddim(xn, w, bias, guidance=g, Nimg=N, H=H, W=W, C_=C, prediction=prediction, **kw)
    else:
        ops.out_ddim(xn, w, bias, Nimg=N, H=H, W=W, C_=C, prediction=prediction, **kw)


def _inputs(guided, N, H, W, C, seed):
    xn, w, bias = _out_conv_inputs(N, H, W, C, seed)
    return (xn if guided else xn[:N].contiguous()), w, bias


def _m_ref(guided, eref, ebound, N, g):
    """The guidance-combined network output in float64 and its fp32 error bound."""
    if not guided:
        return eref, ebound
    eu, ec, bu, bc = eref[:N], eref[N:], ebound[:N], ebound[N:]
    return R.cfg(eu, ec, g), abs(1 - g) * bu + abs(g) * bc + 3 * U * (eu.abs() + abs(g) * (ec.abs() + eu.abs()))


def _v_x0_eps(cf, xt, m):
    """x0 = coef[0] x - coef[1] v, eps = coef[0] v + coef[1] x as (value, fp32 error bound) pairs."""
    x0 = R.ErrLin.lin([(cf[0], xt[0], xt[1]), (-cf[1], m[0], m[1])])
    e = R.ErrLin.lin([(cf[0], m[0], m[1]), (cf[1], xt[0], xt[1])])
    return x0, e


# ================================================ the v exports against float64 =================================
VD_CASES = {
    "cfg_8x8_c320_n1_blend_noise_half": dict(guided=True, N=1, H=8, W=8, C=320, blend=True, noise=True, half=True),
    "cfg_64x64_c640_n3": dict(guided=True, N=3, H=64, W=64, C=640),
    "cfg_128x128_c320_n1_half": dict(guided=True, N=1, H=128, W=128, C=320, half=True),
    "cfg_24x40_c320_n3_blend": dict(guided=True, N=3, H=24, W=40, C=320, blend=True),
    "cfg_eps_only_32x20_c640_n3": dict(guided=True, N=3, H=32, W=20, C=640, eps_only=True),
    "nocfg_8x8_c640_n3_blend_half": dict(guided=False, N=3, H=8, W=8, C=640, blend=True, half=True),
    "nocfg_128x128_c320_n1_blend_noise_half": dict(guided=False, N=1, H=128, W=128, C=320, blend=True, noise=True,
                                                   half=True),
    "nocfg_96x96_c320_n3_half": dict(guided=False, N=3, H=96, W=96, C=320, half=True),
    "nocfg_32x20_c640_n1": dict(guided=False, N=1, H=32, W=20, C=640),
    "nocfg_eps_only_8x8_c320_n1": dict(guided=False, N=1, H=8, W=8, C=320, eps_only=True),
}


@pytest.mark.parametrize("name", list(VD_CASES))
def test_vpred_ddim_fp64(name):
    c = VD_CASES[name]
    guided, N, H, W, C, g = c["guided"], c["N"], c["H"], c["W"], c["C"], 7.5
    kernel = KERNEL[guided]
    h = ops.half_dtype()
    rows = 2 * N if guided else N
    xn, w, bias = _inputs(guided, N, H, W, C, 81)
    eps_out = torch.full((rows, H, W, 4), 7.0, device=DEV)
    eref, mag = R.out_conv(xn.double(), w.double(), bias.double())
    ebound = (9 * C + 1) * U * mag
    if c.get("eps_only"):
        _launch(guided, xn, w, bias, N, H, W, C, eps_out=eps_out)
        _close(kernel, f"raw output {name}", eps_out, eref, ebound)
        return
    a_t, a_prev = 0.35, 0.62
    coef32 = torch.tensor([math.sqrt(a_t), math.sqrt(1 - a_t), math.sqrt(a_prev), math.sqrt(1 - a_prev),
                           0.8, 0.6, 1.0, 0.0] + [0.0] * 8, dtype=torch.float32, device=DEV)
    lat = _randn((N, H, W, 4), 82)
    lat0 = lat.double()
    known = _randn((N, H, W, 4), 83) if c.get("blend") else None
    noise = _randn((N, H, W, 4), 84) if c.get("noise") else None
    mask = None
    if known is not None:
        mask = (torch.rand(N, H, W, generator=_gen(85), device=DEV) < 0.4).float()
        mask[:, :2] = 0.37
    lat_half = torch.full((rows, H, W, 4), 7.0, device=DEV, dtype=h) if c.get("half") else None
    ctr = torch.zeros(1, device=DEV, dtype=torch.int32)
    _launch(guided, xn, w, bias, N, H, W, C, g=g, latents=lat, eps_out=eps_out, coef=coef32, known=known, noise=noise,
            mask=mask, lat_half_out=lat_half, step_counter=ctr)
    _close(kernel, f"raw output {name}", eps_out, eref, ebound)
    cf = [float(v) for v in coef32.double().cpu()]
    x0, e = _v_x0_eps(cf, (lat0, torch.zeros_like(lat0)), _m_ref(guided, eref, ebound, N, g))
    xp = R.ErrLin.lin([(cf[2], x0[0], x0[1]), (cf[3], e[0], e[1])])
    if known is not None:
        xp = R.blend_err(xp, known.double(), None if noise is None else noise.double(), mask.double(), cf)
    ref, err = xp
    _close(kernel, f"latents {name}", lat, ref, err)
    if lat_half is not None:
        _close(kernel, f"lat_half {name}", lat_half[:N], ref, R.ulp(ref, h) + err)
        if guided:
            assert torch.equal(lat_half[:N], lat_half[N:]), "the two CFG copies of the latents differ"
    assert int(ctr.item()) == 1


def _unipc_fused_v(rows_coef, outs, x, guidance, known=None, noise=None, mask=None):
    """fp64_refs.unipc_fused with the v conversion: x0 = coef[0] x - coef[1] m."""
    z = torch.zeros_like(x)
    m1, m2, last = (z, z), (z, z), (z, z)
    xt = (x, z)
    out = []
    for cf, (mu, mc) in zip(rows_coef, outs):
        cf = [float(v) for v in cf]
        m = (R.cfg(mu, mc, guidance), 3 * U * (mu.abs() + abs(guidance) * (mc.abs() + mu.abs())))
        x0, _ = _v_x0_eps(cf, xt, m)
        xc = R.ErrLin.lin([(cf[8], xt[0], xt[1]), (cf[9], last[0], last[1]), (cf[10], m1[0], m1[1]),
                           (cf[11], m2[0], m2[1]), (cf[12], x0[0], x0[1])])
        xp = R.ErrLin.lin([(cf[13], xc[0], xc[1]), (cf[14], x0[0], x0[1]), (cf[15], m1[0], m1[1])])
        m2, m1, last = m1, x0, xc
        if known is not None:
            xp = R.blend_err(xp, known, noise, mask, cf)
        xt = xp
        out.append(xp)
    return out


@pytest.mark.parametrize("blend", [False, True], ids=["plain", "blend_noise"])
@pytest.mark.parametrize("guided", [True, False], ids=["cfg", "nocfg"])
def test_vpred_unipc_schedule_fp64(guided, blend):
    """Mode 1 over a 14-step UniPC (order 2) schedule in v mode: the latents after every step against the v-mode
    scheduler.step() in float64, driven by the raw output the kernel reports through eps_out."""
    N, H, W, C, g = (1, 16, 24, 640, 7.5) if guided else (3, 16, 24, 320, 1.0)
    kernel = KERNEL[guided]
    sched = UniPCMultistepScheduler.from_config(DDIMScheduler(prediction_type=V).config, solver_order=2)
    sched.set_timesteps(14)
    ts = sched.timesteps.tolist()
    blend_rows = known = noise = mask = None
    if blend:
        on = [1.0 if (i < 9 and i % 4 != 2) else 0.0 for i in range(len(ts))]
        nxt = ts[1:] + [0]
        blend_rows = [(float(sched.alpha_t[t]), float(sched.sigma_t[t]), o) for t, o in zip(nxt, on)]
        known, noise = _randn((N, H, W, 4), 91), _randn((N, H, W, 4), 92)
        mask = (torch.rand(N, H, W, generator=_gen(93), device=DEV) < 0.5).float()
    rows = R.unipc_coef_rows(sched, blend_rows)
    coef_tab = torch.tensor(rows, device=DEV)
    if blend:
        blend_rows = [(float(r[4]), float(r[5]), float(r[6])) for r in rows]
    lat = _randn((N, H, W, 4), 94)
    x_init = lat.double()
    hist = torch.zeros(3, N, H, W, 4, device=DEV)
    eps_out = torch.empty((2 if guided else 1) * N, H, W, 4, device=DEV)
    coef = torch.empty(16, device=DEV)
    outs, lats = [], []
    for i in range(len(ts)):
        xn, w, bias = _inputs(guided, N, H, W, C, 300 + 7 * i)
        coef.copy_(coef_tab[i])
        _launch(guided, xn, w, bias, N, H, W, C, g=g, latents=lat, eps_out=eps_out, coef=coef, known=known,
                noise=noise, mask=mask, hist=hist)
        o = eps_out.double()
        outs.append((o[:N], o[N:]) if guided else (o, o))
        lats.append(lat.clone())
    kw = dict(known=None if known is None else known.double(), noise=None if noise is None else noise.double(),
              mask=None if mask is None else mask.double())
    ref = R.scheduler_trajectory(sched, outs, x_init, g, blend_rows, **kw)
    bounds = _unipc_fused_v(rows, outs, x_init, g, **kw)
    for i, (got, r, (_, err)) in enumerate(zip(lats, ref, bounds)):
        _close(kernel, f"UniPC v latents after step {i} (t={ts[i]})", got, r, err)


@pytest.mark.parametrize("name", ["guided", "unguided"])
def test_vpred_matches_reference_p_sample(name):
    """The reference sampler for a parameterization "v" model (cldm/ddim_hacked.py:187-230): the raw outputs handed
    to the kernel through an out conv that reproduces them ([hi | lo] halves through the centre tap)."""
    g = torch.load(os.path.join(GOLD, "ddim_vpred.pt"))[name]
    guided = name == "guided"
    N = g["x"].shape[0]
    nhwc = lambda t: t.permute(0, 2, 3, 1).float().contiguous()       # noqa: E731
    raw = torch.cat([nhwc(g["v_uncond"]), nhwc(g["v_cond"])]) if guided else nhwc(g["v"])
    raw = raw.to(DEV)
    h = ops.half_dtype()
    hi = raw.to(h)
    lo = (raw - hi.float()).to(h)
    xn = torch.cat([hi, lo], -1).contiguous()
    w = torch.zeros(4, 3, 3, 8, device=DEV)
    for o in range(4):
        w[o, 1, 1, o] = w[o, 1, 1, o + 4] = 1.0
    a, ap = g["a_t"], g["a_prev"]
    coef = torch.tensor([math.sqrt(a), math.sqrt(1 - a), math.sqrt(ap), math.sqrt(1 - ap)] + [0.0] * 12, device=DEV)
    lat = nhwc(g["x"]).to(DEV)
    eps_out = torch.empty(raw.shape, device=DEV)
    _launch(guided, xn, w, torch.zeros(4, device=DEV), N, 8, 8, 8, g=g["guidance"], latents=lat, eps_out=eps_out,
            coef=coef)
    assert (eps_out - raw).abs().max().item() < 1e-5
    err = (lat.cpu() - nhwc(g["x_prev"])).abs().max().item()
    assert err < 2e-5, err


@pytest.mark.parametrize("guided", [True, False], ids=["cfg", "nocfg"])
def test_raw_output_bit_identical_between_epsilon_and_v_exports(guided):
    N, H, W, C = 3, 24, 16, 320
    xn, w, bias = _inputs(guided, N, H, W, C, 71)
    rows = (2 if guided else 1) * N
    coef = torch.tensor([0.6, 0.8, 0.7, 0.71] + [0.0] * 12, device=DEV)
    outs = []
    for pred in ("epsilon", V):
        for with_latents in (False, True):
            eps_out = torch.empty(rows, H, W, 4, device=DEV)
            kw = dict(latents=_randn((N, H, W, 4), 72), coef=coef) if with_latents else {}
            _launch(guided, xn, w, bias, N, H, W, C, prediction=pred, eps_out=eps_out, **kw)
            outs.append(eps_out)
    assert all(torch.equal(outs[0], o) for o in outs[1:])


# ================================================ the engine =====================================================
def _tiny21_engine(unet_packed=None):
    usd = None if unet_packed is not None else make_state_dict(TINY21, "unet", 61)
    return DenoiseEngine(TINY21, usd, [make_state_dict(TINY21, "controlnet", 62)], DEV, unet_packed=unet_packed)


def _host_scheduler(kind, prediction_type):
    d = DDIMScheduler(prediction_type=prediction_type)
    return d if kind == "ddim" else UniPCMultistepScheduler.from_config(d.config)


def _run(eng, kind, prediction_type, seed, use_graph, steps=6, gs=6.0):
    x, ctx, hints = make_inputs(TINY21, 2, 16, 13, seed, n_controlnets=1)
    sch = _host_scheduler(kind, prediction_type)
    sch.set_timesteps(steps)
    ts = [int(t) for t in sch.timesteps]
    if kind == "ddim":
        coefs = [sch.coefficients(t) for t in ts]
        ms = None
    else:
        coefs = [(float(sch.alphas_cumprod[t]),) * 2 for t in ts]
        ms = sch.coefficient_rows()
    eng.prepare(ctx, hints, [1.0])
    eng.set_schedule(ts, [c[0] for c in coefs], [c[1] for c in coefs], multistep=ms, prediction_type=prediction_type)
    eng.begin(x[:1], guidance=gs, use_graph=use_graph)
    for _ in ts:
        eng.step()
    return eng.latents().cpu(), (x, ctx, hints, ts)


@pytest.mark.parametrize("kind", ["ddim", "unipc"])
def test_tiny21_engine_v_steps_match_host_reenactment(kind):
    eng = _tiny21_engine()
    steps = 6
    got, (x, ctx, hints, ts) = _run(eng, kind, V, 5, use_graph=True, steps=steps)
    usd, csd = make_state_dict(TINY21, "unet", 61), make_state_dict(TINY21, "controlnet", 62)
    ut, ct = build_topology(TINY21), build_topology(TINY21, with_decoder=False)
    sch, sch_e = _host_scheduler(kind, V), _host_scheduler(kind, "epsilon")
    for s in (sch, sch_e):
        s.set_timesteps(steps)                 # (the DDIM table of 6 steps has 7 entries, like the reference's)
    assert [int(t) for t in sch.timesteps] == ts
    lat, lat_e = x[:1].clone(), x[:1].clone()
    for t in ts:
        for s, which in ((sch, "v"), (sch_e, "e")):
            cur = lat if which == "v" else lat_e
            with torch.no_grad():
                o = O.apply_model(usd, ut, [(csd, ct)], torch.cat([cur, cur]), torch.full((2,), t), ctx, hints, [1.0])
            nxt = s.step(o[:1] + 6.0 * (o[1:] - o[:1]), t, cur).prev_sample
            if which == "v":
                lat = nxt
            else:
                lat_e = nxt
    err = (got - lat).abs().max().item()
    print(f"TINY21 {kind} v: {len(ts)} steps, latents max-abs {err:.3e}; "
          f"epsilon reading differs by {(got - lat_e).abs().max().item():.3e}")
    assert err < 5e-2, err
    assert (got - lat_e).abs().max().item() > 10 * max(err, 1e-3)


def test_engine_switches_epsilon_v_epsilon_with_graph_recapture():
    """One engine (and a tile engine sharing its packed UNet) switching epsilon -> v -> epsilon, DDIM and UniPC: every
    request equals the same request without a graph on a fresh engine, every change of prediction type re-captures,
    and repeating a request replays the captured step."""
    main = _tiny21_engine()
    tile = _tiny21_engine(unet_packed=main.unet)
    seq = [("ddim", "epsilon"), ("ddim", V), ("unipc", V), ("unipc", "epsilon"), ("ddim", "epsilon"), ("ddim", V)]
    prev = {}
    for k, (kind, pt) in enumerate(seq):
        for eng in (main, tile):
            got, _ = _run(eng, kind, pt, 40 + k, use_graph=True)
            g0 = eng._graph
            assert g0 is not None and eng.prediction_type == pt
            if k and seq[k - 1][1] != pt:
                assert g0 is not prev[id(eng)], (k, "a change of prediction type must re-capture")
            prev[id(eng)] = g0
            want, _ = _run(_tiny21_engine(), kind, pt, 40 + k, use_graph=False)
            err = (got - want).abs().max().item()
            assert err < 1e-4, (k, kind, pt, err)
            again, _ = _run(eng, kind, pt, 40 + k, use_graph=True)
            assert eng._graph is g0 and torch.equal(again, got)


def test_full_sd21_768_v_step_against_fp64_update():
    """One captured SD2.1 768x768 step (96x96 latents, N = 4 + CFG, one ControlNet: the sd21_768 configuration) in
    v mode against the float64 v update of the engine's own network output at the same latents and timestep."""
    g = torch.load(os.path.join(GOLD, "sd21_768.pt"))
    m = g["meta"]
    usd = make_state_dict(SD21, "unet", m["unet_seed"])
    csds = [make_state_dict(SD21, "controlnet", s) for s in m["cn_seeds"]]
    eng = DenoiseEngine(SD21, usd, csds, DEV)
    del usd, csds
    x, ctx, hints = make_inputs(SD21, m["B"], m["lat"], m["L"], m["in_seed"], n_controlnets=len(m["cn_seeds"]))
    eng.prepare(ctx, hints, m["scales"])
    N, gs = m["B"] // 2, 7.5
    lat = x[:N]
    ts, a, ap = ddim_schedule(50)
    i = 20
    t, a_t, a_p = int(ts[i]), float(a[i]), float(ap[i])
    raw = eng.eps(torch.cat([lat, lat]), t).double().cpu()          # [2N, 4, 96, 96]
    eng.set_schedule([t], [a_t], [a_p], prediction_type=V)
    eng.begin(lat, guidance=gs, use_graph=True)
    eng.step()
    got = eng.latents().double().cpu()
    assert eng.launches_per_step > 100
    v = raw[:N] + gs * (raw[N:] - raw[:N])
    x0 = math.sqrt(a_t) * lat.double() - math.sqrt(1 - a_t) * v
    e = math.sqrt(a_t) * v + math.sqrt(1 - a_t) * lat.double()
    ref = math.sqrt(a_p) * x0 + math.sqrt(1 - a_p) * e
    err = (got - ref).abs().max().item()
    eps_reading = math.sqrt(a_p) * (lat.double() - math.sqrt(1 - a_t) * v) / math.sqrt(a_t) + math.sqrt(1 - a_p) * v
    print(f"sd21_768 v step t={t}: max-abs {err:.3e}, |v| max {v.abs().max().item():.3f}, "
          f"epsilon reading differs by {(got - eps_reading).abs().max().item():.3e}")
    assert err < 1e-4 * (1 + v.abs().max().item()), err
    assert (got - eps_reading).abs().max().item() > 1e-2
    del eng
    torch.cuda.empty_cache()


# ================================================ the pipeline with VaeEngine ====================================
def _pipe_setup(kind):
    from editanything_b200.vae import VaeEngine, make_vae_state_dict
    from tests.test_gpu_pipeline import VCFG
    usd = make_state_dict(TINY21, "unet", 61)
    csds = [make_state_dict(TINY21, "controlnet", 62)]
    vsd = dict(make_vae_state_dict(VCFG, 63, part="encoder"))
    vsd.update(make_vae_state_dict(VCFG, 64))
    pipe = StableDiffusionControlNetInpaintPipeline(DenoiseEngine(TINY21, usd, csds, DEV),
                                                    vae=VaeEngine(VCFG, vsd, DEV),
                                                    scheduler=_host_scheduler(kind, V))
    gen = torch.Generator().manual_seed(0)
    image = torch.rand(1, 3, 128, 128, generator=gen) * 2 - 1
    mask = torch.zeros(1, 1, 128, 128)
    mask[:, :, 32:96, 16:80] = 1.0
    conds = [torch.randint(0, 256, (1, 3, 128, 128), generator=gen).float()]
    pe = torch.randn(1, 13, TINY21.context_dim, generator=gen)
    ne = torch.randn(1, 13, TINY21.context_dim, generator=gen)
    return usd, csds, vsd, pipe, image, mask, conds, pe, ne


@pytest.mark.parametrize("kind", ["ddim", "unipc"])
def test_pipeline_v_on_cuda_matches_reference_loop(kind):
    """guidance 5, 8 steps, alignment_ratio 0.5, VaeEngine on both sides, against the reference loop re-enacted with
    the v-mode scheduler object on the oracle networks."""
    from oracle import vae_oracle as VO
    from tests.test_gpu_pipeline import GS, STEPS, VCFG, _close as _close_lat
    usd, csds, vsd, pipe, image, mask, conds, pe, ne = _pipe_setup(kind)
    kw = dict(image=image, mask_image=mask, controlnet_conditioning_image=conds, height=128, width=128,
              num_inference_steps=STEPS, guidance_scale=GS, prompt_embeds=pe, negative_prompt_embeds=ne,
              controlnet_conditioning_scale=1.0, alignment_ratio=0.5)
    lat = pipe(generator=torch.manual_seed(7), output_type="latent", **kw).images
    assert lat.is_cuda and pipe.engine.prediction_type == V
    gen = torch.manual_seed(7)
    x = torch.randn((1, 4, 16, 16), generator=gen)
    noise = x
    with torch.no_grad():
        mom = VO.encode_moments(image, vsd, VCFG)
    mean, logvar = mom.chunk(2, 1)
    init = VCFG.scaling_factor * (mean + torch.exp(0.5 * logvar.clamp(-30, 20)) * torch.randn(mean.shape, generator=gen))
    m = 1 - F.interpolate((mask >= 0.5).float(), (16, 16), mode="nearest")
    sch = _host_scheduler(kind, V)
    sch.set_timesteps(STEPS)
    ts = sch.timesteps
    ut, ct = build_topology(TINY21), build_topology(TINY21, with_decoder=False)
    ctx, hints = torch.cat([ne, pe]), [torch.cat([conds[0]] * 2)]
    for i, t in enumerate(ts):
        with torch.no_grad():
            o = O.apply_model(usd, ut, [(csds[0], ct)], torch.cat([x, x]), torch.full((2,), int(t)), ctx, hints, [1.0])
        x = sch.step(o[:1] + GS * (o[1:] - o[:1]), t, x).prev_sample
        if i < len(ts) * 0.5:
            x = sch.add_noise(init, noise, ts[i + 1]) * m + x * (1 - m)
    _close_lat(lat.cpu(), x, f"v latents ({kind})")
    out = pipe(generator=torch.manual_seed(7), output_type="np", **kw)
    with torch.no_grad():
        img = VO.decode_latents(x, vsd, VCFG).permute(0, 2, 3, 1).numpy()
    assert out.images.shape == img.shape == (1, 128, 128, 3)
    assert abs(out.images - img).mean() < 1e-2
