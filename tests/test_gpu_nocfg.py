"""-m gpu: sampling without classifier-free guidance (guidance_scale <= 1).

Ordered so that a wrong shape fails as an assertion or an EA_ERR_* before any end-to-end run: first ea_out_ddim
against float64 (tests/fp64_refs.py, the gates of tests/test_gpu_kernels_fp64.py) and against the reference sampler's
own unguided p_sample_ddim (tests/golden/ddim_nocfg.pt), then the networks at the batch sizes only unguided requests
reach (B = 1 and B = 3: the batch rows of the reference networks are independent and oracle.inputs.make_inputs is
seeded, so rows of the existing goldens pin them under the 1e-2 max-abs gate), then the pipeline with VaeEngine
against the re-enacted unguided reference loop (the gates of tests/test_gpu_pipeline.py) and CUDA-graph re-capture
across guided and unguided requests."""
import math
import os

import pytest
import torch

from editanything_b200 import ops
from editanything_b200.denoise import DenoiseEngine, ddim_schedule
from editanything_b200.pipeline import DDIMScheduler
from editanything_b200.schedulers import UniPCMultistepScheduler
from editanything_b200.unet_spec import SD15, TINY, TINY21, make_state_dict
from oracle.inputs import make_inputs
from tests import fp64_refs as R
from tests.test_gpu_kernels_fp64 import DEV, U, _close, _gen, _out_conv_inputs, _randn

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
EPS_TOL = 1e-2


# ================================================ ea_out_ddim against float64 ===================================
def _rows(xn, N):
    return xn[:N].contiguous()          # _out_conv_inputs draws 2N rows; the unguided kernel reads N


OD_CASES = {
    "ddim_64x64_c320_n1_blend_noise_half": dict(Nimg=1, H=64, W=64, C=320, blend=True, noise=True, half_out=True),
    "ddim_24x40_c640_n3": dict(Nimg=3, H=24, W=40, C=640),
    "ddim_8x8_c320_n3_blend_half": dict(Nimg=3, H=8, W=8, C=320, blend=True, half_out=True),
    "ddim_128x128_c320_n1_half": dict(Nimg=1, H=128, W=128, C=320, half_out=True),
    "eps_only_32x20_c640_n3": dict(Nimg=3, H=32, W=20, C=640, eps_only=True),
    "eps_only_8x8_c320_n1": dict(Nimg=1, H=8, W=8, C=320, eps_only=True),
}


@pytest.mark.parametrize("name", list(OD_CASES))
def test_out_ddim_fp64(name):
    c = OD_CASES[name]
    h = ops.half_dtype()
    N, H, W, C = c["Nimg"], c["H"], c["W"], c["C"]
    xn, w, bias = _out_conv_inputs(N, H, W, C, 51)
    xn = _rows(xn, N)
    eps_out = torch.full((N, H, W, 4), 7.0, device=DEV)
    ref_e, mag = R.out_conv(xn.double(), w.double(), bias.double())
    e_bound = (9 * C + 1) * U * mag
    if c.get("eps_only"):
        ops.out_ddim(xn, w, bias, eps_out=eps_out, Nimg=N, H=H, W=W, C_=C)
        _close("ea_out_ddim", f"eps {name}", eps_out, ref_e, e_bound)
        return
    a_t, a_prev = 0.35, 0.62
    coef32 = torch.tensor([math.sqrt(a_t), math.sqrt(1 - a_t), math.sqrt(a_prev), math.sqrt(1 - a_prev),
                           0.8, 0.6, 1.0, 0.0] + [0.0] * 8, dtype=torch.float32, device=DEV)
    lat = _randn((N, H, W, 4), 52)
    lat0 = lat.double()
    known = _randn((N, H, W, 4), 53) if c.get("blend") else None
    noise = _randn((N, H, W, 4), 54) if c.get("noise") else None
    mask = None
    if known is not None:
        mask = (torch.rand(N, H, W, generator=_gen(55), device=DEV) < 0.4).float()
        mask[:, :2] = 0.37
    lat_half = torch.full((N, H, W, 4), 7.0, device=DEV, dtype=h) if c.get("half_out") else None
    ctr = torch.zeros(1, device=DEV, dtype=torch.int32)
    ops.out_ddim(xn, w, bias, latents=lat, eps_out=eps_out, coef=coef32, known=known, noise=noise, mask=mask,
                 lat_half_out=lat_half, step_counter=ctr, Nimg=N, H=H, W=W, C_=C)
    _close("ea_out_ddim", f"eps {name}", eps_out, ref_e, e_bound)
    cf = [float(v) for v in coef32.double().cpu()]
    z = torch.zeros_like(lat0)
    x0 = R.ErrLin.lin([(1.0 / cf[0], lat0, z), (-cf[1] / cf[0], ref_e, e_bound)])
    xp = R.ErrLin.lin([(cf[2], x0[0], x0[1]), (cf[3], ref_e, e_bound)])
    if known is not None:
        xp = R.blend_err(xp, known.double(), None if noise is None else noise.double(), mask.double(), cf)
    ref, err = xp
    _close("ea_out_ddim", f"latents {name}", lat, ref, err)
    if lat_half is not None:
        _close("ea_out_ddim", f"lat_half {name}", lat_half, ref, R.ulp(ref, h) + err)
    assert int(ctr.item()) == 1


def test_out_ddim_unipc_schedule_fp64():
    """Mode 1 over a 12-step UniPC (order 2) schedule with the blend, 3 images: the latents after every step against
    scheduler.step() in float64, driven by the eps the kernel reports (fp64_refs with the unguided eps as both
    halves at guidance 1: cfg(e, e, 1) = e)."""
    N, H, W, C = 3, 16, 24, 320
    sched = UniPCMultistepScheduler.from_config(DDIMScheduler().config, solver_order=2)
    sched.set_timesteps(12)
    ts = sched.timesteps.tolist()
    on = [1.0 if i < 7 else 0.0 for i in range(len(ts))]
    nxt = ts[1:] + [0]
    rows = R.unipc_coef_rows(sched, [(float(sched.alpha_t[t]), float(sched.sigma_t[t]), o) for t, o in zip(nxt, on)])
    blend_rows = [(float(r[4]), float(r[5]), float(r[6])) for r in rows]
    coef_tab = torch.tensor(rows, device=DEV)
    known, noise = _randn((N, H, W, 4), 61), _randn((N, H, W, 4), 62)
    mask = (torch.rand(N, H, W, generator=_gen(63), device=DEV) < 0.5).float()
    lat = _randn((N, H, W, 4), 64)
    x_init = lat.double()
    hist = torch.zeros(3, N, H, W, 4, device=DEV)
    eps_out = torch.empty(N, H, W, 4, device=DEV)
    coef = torch.empty(16, device=DEV)
    eps_list, lats = [], []
    for i in range(len(ts)):
        xn, w, bias = _out_conv_inputs(N, H, W, C, 200 + 7 * i)
        xn = _rows(xn, N)
        coef.copy_(coef_tab[i])
        ops.out_ddim(xn, w, bias, latents=lat, eps_out=eps_out, coef=coef, known=known, noise=noise, mask=mask,
                     hist=hist, Nimg=N, H=H, W=W, C_=C)
        e = eps_out.double()
        eps_list.append((e, e))
        lats.append(lat.clone())
    kw = dict(known=known.double(), noise=noise.double(), mask=mask.double())
    ref = R.scheduler_trajectory(sched, eps_list, x_init, 1.0, blend_rows, **kw)
    bounds = R.unipc_fused(rows, eps_list, x_init, 1.0, **kw)
    for i, (got, r, (_, err)) in enumerate(zip(lats, ref, bounds)):
        _close("ea_out_ddim", f"UniPC latents after step {i}", got, r, err)


def test_out_ddim_matches_reference_unguided_p_sample():
    """The reference sampler at unconditional_guidance_scale 1 (cldm/ddim_hacked.py:187-188): eps handed to the
    kernel through an out conv that reproduces it ([hi | lo] halves through the centre tap)."""
    g = torch.load(os.path.join(GOLD, "ddim_nocfg.pt"))["p_sample"]
    N = g["x"].shape[0]
    e = g["e"].permute(0, 2, 3, 1).float().to(DEV)
    h = ops.half_dtype()
    hi = e.to(h)
    lo = (e - hi.float()).to(h)
    xn = torch.cat([hi, lo], -1).contiguous()
    w = torch.zeros(4, 3, 3, 8, device=DEV)
    for o in range(4):
        w[o, 1, 1, o] = w[o, 1, 1, o + 4] = 1.0
    a, ap = g["a_t"], g["a_prev"]
    coef = torch.tensor([math.sqrt(a), math.sqrt(1 - a), math.sqrt(ap), math.sqrt(1 - ap)] + [0.0] * 12, device=DEV)
    lat = g["x"].permute(0, 2, 3, 1).contiguous().float().to(DEV)
    eps_out = torch.empty(N, 8, 8, 4, device=DEV)
    ops.out_ddim(xn, w, torch.zeros(4, device=DEV), latents=lat, eps_out=eps_out, coef=coef, Nimg=N, H=8, W=8, C_=8)
    assert (eps_out.cpu() - g["e"].permute(0, 2, 3, 1)).abs().max().item() < 1e-5
    err = (lat.cpu() - g["x_prev"].permute(0, 2, 3, 1)).abs().max().item()
    assert err < 2e-5, err


def test_unguided_eps_rows_equal_the_guided_kernels():
    """The out conv of ea_out_ddim over 2N rows gives bit for bit what ea_out_cfg_ddim gives for its two halves."""
    N, H, W, C = 2, 16, 16, 320
    xn, w, bias = _out_conv_inputs(N, H, W, C, 71)
    a = torch.empty(2 * N, H, W, 4, device=DEV)
    b = torch.empty(2 * N, H, W, 4, device=DEV)
    ops.out_cfg_ddim(xn, w, bias, eps_out=a, Nimg=N, H=H, W=W, C_=C)
    ops.out_ddim(xn, w, bias, eps_out=b, Nimg=2 * N, H=H, W=W, C_=C)
    assert torch.equal(a, b)


# ================================================ the networks at B = 1 and B = 3 ================================
CFGS = {"tiny_sd15": TINY, "tiny_sd21": TINY21, "tiny_sd15_32": TINY, "sd15_512": SD15, "sd15_512_b8": SD15}


def _eps_rows(name, rows):
    """eps of the golden's batch rows `rows` alone, on an engine prepared without guidance."""
    g = torch.load(os.path.join(GOLD, name + ".pt"))
    m = g["meta"]
    cfg = CFGS[name]
    usd = make_state_dict(cfg, "unet", m["unet_seed"])
    csds = [make_state_dict(cfg, "controlnet", s) for s in m["cn_seeds"]]
    eng = DenoiseEngine(cfg, usd, csds, torch.device("cuda:0"))
    del usd, csds
    x, ctx, hints = make_inputs(cfg, m["B"], m["lat"], m["L"], m["in_seed"], n_controlnets=len(m["cn_seeds"]))
    eng.prepare(ctx[rows], [h[rows] for h in hints], m["scales"], guided=False)
    for t in m["timesteps"]:
        eps = eng.eps(x[rows], t).cpu()
        ref = g[f"eps_t{t}"][rows]
        err = (eps - ref).abs().max().item()
        print(f"{name} rows {rows} t={t} eps max-abs {err:.3e}")
        assert eps.shape[0] == len(range(*rows.indices(m["B"])))
        assert err < EPS_TOL, (name, rows, t, err)
    del eng
    torch.cuda.empty_cache()


@pytest.mark.parametrize("name", ["tiny_sd15", "tiny_sd21", "tiny_sd15_32"])
def test_eps_batch1_reduced_width(name):
    _eps_rows(name, slice(1, 2))


def test_eps_batch1_sd15_512():
    _eps_rows("sd15_512", slice(1, 2))


def test_eps_batch3_sd15_512_b8():
    _eps_rows("sd15_512_b8", slice(0, 3))


# ================================================ pipeline and CUDA graphs =======================================
def test_pipeline_unguided_on_cuda_matches_reference_loop():
    """guidance_scale 1.0 (and 0.5: the same latents) with VaeEngine, 3 images per prompt, alignment_ratio 0.5."""
    import torch.nn.functional as F
    from editanything_b200.unet_spec import build_topology
    from oracle import unet_oracle as O
    from oracle import vae_oracle as V
    from tests.test_gpu_pipeline import STEPS, VCFG, _close as _close_lat, _setup
    cfg, usd, csds, vsd, pipe, image, mask, conds, pe, ne = _setup()
    n_img, ar = 3, 0.5
    kw = dict(image=image, mask_image=mask, controlnet_conditioning_image=conds, height=128, width=128,
              num_inference_steps=STEPS, prompt_embeds=pe, negative_prompt_embeds=ne,
              controlnet_conditioning_scale=[0.5, 1.0], alignment_ratio=ar, num_images_per_prompt=n_img)
    lat = pipe(generator=torch.manual_seed(7), output_type="latent", guidance_scale=1.0, **kw).images
    assert lat.is_cuda and lat.shape == (n_img, 4, 16, 16) and pipe.engine.B == n_img
    gen = torch.manual_seed(7)
    x = torch.randn((n_img, 4, 16, 16), generator=gen)
    noise = x
    with torch.no_grad():
        mom = V.encode_moments(image, vsd, VCFG)
    mean, logvar = mom.chunk(2, 1)
    init = VCFG.scaling_factor * (mean + torch.exp(0.5 * logvar.clamp(-30, 20)) * torch.randn(mean.shape, generator=gen))
    init = init.repeat(n_img, 1, 1, 1)
    m = 1 - F.interpolate((mask >= 0.5).float(), (16, 16), mode="nearest")
    sch = DDIMScheduler()
    sch.set_timesteps(STEPS)
    ts = sch.timesteps
    ut, ct = build_topology(cfg), build_topology(cfg, with_decoder=False)
    hints = [c.repeat_interleave(n_img, 0) for c in conds]
    for i, t in enumerate(ts):
        with torch.no_grad():
            e = O.apply_model(usd, ut, [(sd, ct) for sd in csds], x, torch.full((n_img,), int(t)), pe.repeat(n_img, 1, 1),
                              hints, [0.5, 1.0])
        x = sch.step(e, t, x).prev_sample
        if i < len(ts) * ar:
            x = sch.add_noise(init, noise, ts[i + 1]) * m + x * (1 - m)
    _close_lat(lat.cpu(), x, "unguided latents")
    lat_half = pipe(generator=torch.manual_seed(7), output_type="latent", guidance_scale=0.5, **kw).images
    assert torch.equal(lat_half, lat)
    out = pipe(generator=torch.manual_seed(7), output_type="np", guidance_scale=1.0, **kw)
    with torch.no_grad():
        img = V.decode_latents(x, vsd, VCFG).permute(0, 2, 3, 1).numpy()
    assert out.images.shape == img.shape == (n_img, 128, 128, 3)
    assert abs(out.images - img).mean() < 1e-2


def _tiny_engine(n_cn=2, unet_packed=None):
    usd = None if unet_packed is not None else make_state_dict(TINY, "unet", 51)
    csds = [make_state_dict(TINY, "controlnet", 52 + i) for i in range(n_cn)]
    return DenoiseEngine(TINY, usd, csds, torch.device("cuda:0"), unet_packed=unet_packed)


def _request(eng, guided, n_img, seed, use_graph):
    x, ctx, hints = make_inputs(TINY, 2 * n_img, 16, 13, seed, n_controlnets=len(eng.cns))
    if not guided:
        ctx, hints = ctx[n_img:], [h[n_img:] for h in hints]
    ts, a, ap = ddim_schedule(6)
    eng.prepare(ctx, hints, [0.5, 1.0][:len(eng.cns)], guided=guided)
    eng.set_schedule(ts, a, ap)
    eng.begin(x[:n_img, :4], guidance=6.0, use_graph=use_graph)
    for _ in ts:
        eng.step()
    return eng.latents().cpu()


def test_graph_recaptured_across_guided_and_unguided_requests():
    """guided -> unguided (N = 1, 2, 3) -> guided on one engine and on a tile engine sharing its packed UNet, with
    the captured step: every request equals the same request run without a graph, and every change of mode or
    batch re-captures."""
    main = _tiny_engine()
    tile = _tiny_engine(1, unet_packed=main.unet)
    plain_main, plain_tile = _tiny_engine(), _tiny_engine(1, unet_packed=None)
    seq = [(True, 1), (False, 1), (False, 2), (False, 3), (True, 2), (True, 1), (False, 1)]
    for k, (guided, n_img) in enumerate(seq):
        for eng, plain in ((main, plain_main), (tile, plain_tile)):
            got = _request(eng, guided, n_img, 40 + k, use_graph=True)
            g0 = eng._graph
            assert g0 is not None and eng.launches_per_step > 0
            want = _request(plain, guided, n_img, 40 + k, use_graph=False)
            err = (got - want).abs().max().item()
            assert got.shape == (n_img, 4, 16, 16) and err < 1e-4, (k, guided, n_img, err)
            again = _request(eng, guided, n_img, 40 + k, use_graph=True)       # same request: replayed, not re-captured
            assert eng._graph is g0 and torch.equal(again, got)
