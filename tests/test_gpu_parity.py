"""-m gpu: the CUDA path (through the C ABI) against the reference-generated golden vectors and
the CPU oracle, at reduced width (seconds) and at BASELINE.json configs[1] full size.

Tolerance (BASELINE.json north_star): per-step UNet eps max-abs < 1e-2 in fp16 storage / fp32
accumulation, against the fp32 reference at the same weights."""
import os

import pytest
import torch

from editanything_b200.denoise import DenoiseEngine, ddim_schedule
from editanything_b200.unet_spec import SD15, SD21, TINY, TINY21, build_topology, make_state_dict
from oracle import unet_oracle as O
from oracle.inputs import make_inputs

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CFGS = {"tiny_sd15": TINY, "tiny_sd21": TINY21, "tiny_sd15_32": TINY, "sd15_512": SD15, "sd21_768": SD21,
        "sd15_512_b8": SD15, "sd15_1024": SD15}
EPS_TOL = 1e-2


def _engine(name):
    g = torch.load(os.path.join(GOLD, name + ".pt"))
    m = g["meta"]
    cfg = CFGS[name]
    usd = make_state_dict(cfg, "unet", m["unet_seed"])
    csds = [make_state_dict(cfg, "controlnet", s) for s in m["cn_seeds"]]
    eng = DenoiseEngine(cfg, usd, csds, torch.device("cuda:0"))
    x, ctx, hints = make_inputs(cfg, m["B"], m["lat"], m["L"], m["in_seed"], n_controlnets=len(csds))
    eng.prepare(ctx, hints, m["scales"])
    if cfg.model_channels > 64:
        del usd, csds
        usd = csds = None
        torch.cuda.empty_cache()
    return g, m, eng, x, (cfg, usd, csds, ctx, hints)


@pytest.mark.parametrize("name", ["tiny_sd15", "tiny_sd21", "tiny_sd15_32"])
def test_eps_vs_reference_golden_reduced_width(name):
    g, m, eng, x, _ = _engine(name)
    for t in m["timesteps"]:
        eps = eng.eps(x, t).cpu()
        ref = g[f"eps_t{t}"]
        err = (eps - ref).abs().max().item()
        assert err < EPS_TOL, (name, t, err, ref.abs().max().item())


def _check_full(name):
    g, m, eng, x, _ = _engine(name)
    for t in m["timesteps"]:
        eps = eng.eps(x, t).cpu()
        ref = g[f"eps_t{t}"]
        if f"eps_t{t}_index" in g:       # the golden file keeps a fixed, seeded sample of the batch rows
            dim, idx = g[f"eps_t{t}_index"]
            eps = eps.index_select(dim, idx)
        err = (eps - ref).abs().max().item()
        rel = ((eps - ref).norm() / ref.norm()).item()
        print(f"{name} t={t} eps max-abs {err:.3e} rel-fro {rel:.3e} ref-max {ref.abs().max().item():.3f}")
        assert err < EPS_TOL, (name, t, err, rel)


def test_eps_vs_reference_golden_full_sd15_512():
    """BASELINE.json configs[1]: SD1.5, 512x512 (64x64 latents), 1 image + CFG, SAM + inpaint
    ControlNets, L = 77, at the first / middle / last timestep of the 50-step DDIM table.  Golden eps
    was produced by the reference's own cldm modules (oracle/make_golden.py --full)."""
    _check_full("sd15_512")


def test_eps_vs_reference_golden_full_sd21_768_batch4():
    """BASELINE.json configs[2]: SD2.1 (models/cldm_v21.yaml:21-55: 64-wide heads, linear proj_in/out,
    ctx 1024), 768x768 (96x96 latents, 9216-token self-attention), N = 4 + CFG => B = 8, 1 ControlNet."""
    _check_full("sd21_768")


def test_eps_vs_reference_golden_full_sd15_512_batch4():
    """BASELINE.json configs[3] per-GPU shard: SD1.5 512x512, 4 images + CFG => B = 8, SAM + inpaint
    ControlNets."""
    _check_full("sd15_512_b8")


def test_eps_vs_reference_golden_full_sd15_1024_tile():
    """BASELINE.json configs[4]: SD1.5 1024x1024 tile refinement (128x128 latents, 16384 tokens at the top
    level), N = 1 + CFG, one (tile) ControlNet."""
    _check_full("sd15_1024")


def test_eps_vs_cpu_oracle_fresh_inputs():
    cfg = TINY
    usd = make_state_dict(cfg, "unet", 11)
    csds = [make_state_dict(cfg, "controlnet", 12)]
    x, ctx, hints = make_inputs(cfg, 4, 16, 33, 99, n_controlnets=1)   # 2 images + CFG, ragged L
    eng = DenoiseEngine(cfg, usd, csds, torch.device("cuda:0"))
    eng.prepare(ctx, hints, [0.8])
    ut, ct = build_topology(cfg), build_topology(cfg, with_decoder=False)
    for t in (999, 500, 1):
        with torch.no_grad():
            ref = O.apply_model(usd, ut, [(csds[0], ct)], x, torch.full((4,), t), ctx, hints, [0.8])
        assert (eng.eps(x, t).cpu() - ref).abs().max().item() < EPS_TOL


@pytest.mark.parametrize("concurrent", ["1", "0"])
def test_three_controlnets_vs_cpu_oracle(concurrent, monkeypatch):
    """Three ControlNets are more networks than one grouped launch takes, so the encoder runs network by network: on
    one CUDA stream each with the zero-convs applied after the streams join (EA_CONCURRENT=1, the default), or one
    after another on the current stream (EA_CONCURRENT=0)."""
    monkeypatch.setenv("EA_CONCURRENT", concurrent)
    cfg = TINY
    usd = make_state_dict(cfg, "unet", 71)
    csds = [make_state_dict(cfg, "controlnet", 72 + i) for i in range(3)]
    x, ctx, hints = make_inputs(cfg, 2, 16, 13, 8)
    hints = hints + [hints[0].flip(-1)]
    scales = [0.5, 1.0, 0.7]
    eng = DenoiseEngine(cfg, usd, csds, torch.device("cuda:0"))
    assert not eng.runner.lockstep and eng.runner.concurrent == (concurrent == "1")
    eng.prepare(ctx, hints, scales)
    ut, ct = build_topology(cfg), build_topology(cfg, with_decoder=False)
    for t in (981, 501, 1):
        with torch.no_grad():
            ref = O.apply_model(usd, ut, [(sd, ct) for sd in csds], x, torch.full((2,), t), ctx, hints, scales)
        err = (eng.eps(x, t).cpu() - ref).abs().max().item()
        assert err < EPS_TOL, (concurrent, t, err)


@pytest.mark.parametrize("use_graph", [False, True])
def test_fused_ddim_loop_matches_oracle_loop(use_graph):
    """5 fused steps (ControlNets -> UNet -> CFG -> DDIM, with the inpaint blend) against the
    oracle loop; CUDA-graph replay must give the same latents as eager launches."""
    cfg = TINY
    usd = make_state_dict(cfg, "unet", 21)
    csds = [make_state_dict(cfg, "controlnet", 22), make_state_dict(cfg, "controlnet", 23)]
    x, ctx, hints = make_inputs(cfg, 2, 16, 13, 5)
    g = torch.Generator().manual_seed(3)
    lat0 = torch.randn(1, 4, 16, 16, generator=g)
    known = torch.randn(1, 4, 16, 16, generator=g)
    mask = (torch.rand(1, 1, 16, 16, generator=g) > 0.5).float()
    eng = DenoiseEngine(cfg, usd, csds, torch.device("cuda:0"))
    eng.prepare(ctx, hints, [0.5, 1.0])
    eng.begin(lat0, guidance=9.0, known_nchw=known, mask_n1hw=mask, use_graph=use_graph)
    ts, a, ap = ddim_schedule(50)
    ut, ct = build_topology(cfg), build_topology(cfg, with_decoder=False)
    lat = lat0.clone()
    for i in range(5):
        eng.step(int(ts[i]), float(a[i]), float(ap[i]))
        with torch.no_grad():
            xx = torch.cat([lat, lat])
            e = O.apply_model(usd, ut, [(sd, ct) for sd in csds], xx, torch.full((2,), int(ts[i])), ctx, hints,
                              [0.5, 1.0])
        lat, _ = O.ddim_step(lat, e[:1], e[1:], 9.0, float(a[i]), float(ap[i]))
        lat = known * mask + lat * (1 - mask)
    err = (eng.latents().cpu() - lat).abs().max().item()
    assert err < 5e-2, err
    if use_graph:
        assert eng.launches_per_step > 100


def test_guess_mode_and_spatial_scale_map_vs_oracle():
    """ControlNetModel2.forward scaling variants (utils/stable_diffusion_controlnet.py:777-802) on the CUDA path."""
    cfg = TINY
    usd = make_state_dict(cfg, "unet", 41)
    csds = [make_state_dict(cfg, "controlnet", 42), make_state_dict(cfg, "controlnet", 43)]
    x, ctx, hints = make_inputs(cfg, 2, 16, 11, 3)
    eng = DenoiseEngine(cfg, usd, csds, torch.device("cuda:0"))
    ut, ct = build_topology(cfg), build_topology(cfg, with_decoder=False)
    t = 601
    smap = torch.rand(16, 16, generator=torch.Generator().manual_seed(9))
    for scales, gm in (([0.7, 1.0], True), ([smap, 0.5], False), ([0.7, 1.0], False)):
        eng.prepare(ctx, hints, scales, guess_mode=gm)
        with torch.no_grad():
            ref = O.apply_model(usd, ut, [(sd, ct) for sd in csds], x, torch.full((2,), t), ctx, hints, scales, guess_mode=gm)
        assert (eng.eps(x, t).cpu() - ref).abs().max().item() < EPS_TOL
