"""-m gpu: text-to-image ControlNet pipelines (all-region generation) on the fused step.

First the zero-conv launches of guess mode with guidance (DenoiseEngine.prepare(controlnet_rows="conditional")): every
one has M = N*h*w rows and writes only the conditional rows of its slot, and the unconditional rows of every slot stay
bit for bit what the UNet stored there (snapshots taken around each launch).  Then the network output per step against
the oracle networks on the CPU under the 1e-2 max-abs gate of tests/test_gpu_nocfg.py, guess mode on and off, the
reference sampler's own guess-mode step (tests/golden/t2i_guess.pt), CUDA-graph replay against eager steps, and
EditAnythingLoraModel.process(enable_all_generate=True) end to end on test-sized checkpoints."""
import os

import numpy as np
import pytest
import torch

from editanything_b200 import ops
from editanything_b200.denoise import DenoiseEngine, ddim_schedule
from editanything_b200.unet_spec import SD15, SD21, TINY, build_topology, make_state_dict
from oracle import unet_oracle as O
from oracle.inputs import make_inputs

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
DEV = torch.device("cuda:0")
EPS_TOL = 1e-2


class _ZeroConvRecorder:
    """The operator table with every accumulating GEMM (the ControlNet zero-convs) recorded: its M, its output view and
    whether the rows in front of that view (the unconditional half of the slot) changed across the launch."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, k):
        return getattr(ops, k)

    def gemm(self, a, w, out=None, **kw):
        if not kw.get("accumulate"):
            return ops.gemm(a, w, out, **kw)
        n = out.shape[0]
        front = out.storage_offset() - n * out.stride(0)
        unc = torch.as_strided(out, out.shape, out.stride(), front) if front >= 0 else None
        before = unc.clone() if unc is not None else None
        r = ops.gemm(a, w, out, **kw)
        torch.cuda.synchronize()
        self.calls.append(dict(M=kw["M"], rows=n, hw=out.shape[1] * out.shape[2], a_rows=a.shape[0],
                               unchanged=unc is not None and torch.equal(unc, before)))
        return r


@pytest.mark.parametrize("n_img,n_cn", [(1, 1), (3, 2)])
def test_zero_convs_write_only_the_conditional_rows(n_img, n_cn):
    rec = _ZeroConvRecorder()
    usd = make_state_dict(TINY, "unet", 51)
    csds = [make_state_dict(TINY, "controlnet", 52 + i) for i in range(n_cn)]
    eng = DenoiseEngine(TINY, usd, csds, DEV, backend=rec)
    x, ctx, hints = make_inputs(TINY, 2 * n_img, 16, 13, 5, n_controlnets=n_cn)
    eng.prepare(ctx, [h[:n_img] for h in hints], [0.5, 1.0][:n_cn], guess_mode=True, controlnet_rows="conditional")
    eng.eps(x[:, :4], 501)
    n_zc = n_cn * (len(eng.unet.topo.input_blocks) + 1)
    assert len(rec.calls) == n_zc
    for c in rec.calls:
        assert c["rows"] == n_img and c["M"] == n_img * c["hw"] == c["a_rows"], c
        assert c["unchanged"], c
    rec.calls.clear()
    eng.prepare(ctx, hints, [0.5, 1.0][:n_cn], guess_mode=True)              # guess mode on both halves: 2N rows
    eng.eps(x[:, :4], 501)
    assert len(rec.calls) == n_zc and all(c["rows"] == 2 * n_img and c["M"] == 2 * n_img * c["hw"] for c in rec.calls)


# ================================================ the network output against the oracle =========================
CASES = {"tiny_n1": (TINY, 1, 8, 7), "tiny_n3": (TINY, 3, 8, 7), "sd15_512_n1": (SD15, 1, 64, 77),
         "sd15_512_n4": (SD15, 4, 64, 77), "sd21_768_n1": (SD21, 1, 96, 77)}


@pytest.mark.parametrize("guess", [False, True])
@pytest.mark.parametrize("name", list(CASES))
def test_eps_against_oracle(name, guess):
    cfg, n, lat, L = CASES[name]
    usd = make_state_dict(cfg, "unet", 101)
    csd = make_state_dict(cfg, "controlnet", 102)
    eng = DenoiseEngine(cfg, usd, [csd], DEV)
    x, ctx, hints = make_inputs(cfg, 2 * n, lat, L, 9, n_controlnets=1)
    x, hint = x[:n], hints[0][:n]
    t, s = 641, 0.9
    if guess:
        eng.prepare(ctx, [hint], [s], guess_mode=True, controlnet_rows="conditional")
    else:
        eng.prepare(ctx, [torch.cat([hint, hint])], [s], cfg_duplicated=True)
    eps = eng.eps(torch.cat([x, x]), t).cpu()
    del eng
    torch.cuda.empty_cache()
    ut, ct = build_topology(cfg), build_topology(cfg, with_decoder=False)
    tt = torch.full((n,), t)
    with torch.no_grad():
        if guess:
            e_u = O.apply_model(usd, ut, [], x, tt, ctx[:n], [], [])
            e_c = O.apply_model(usd, ut, [(csd, ct)], x, tt, ctx[n:], [hint], [s], guess_mode=True)
            ref = torch.cat([e_u, e_c])
        else:
            ref = O.apply_model(usd, ut, [(csd, ct)], torch.cat([x, x]), torch.full((2 * n,), t), ctx,
                                [torch.cat([hint, hint])], [s])
    err_u = (eps[:n] - ref[:n]).abs().max().item()
    err_c = (eps[n:] - ref[n:]).abs().max().item()
    print(f"{name} guess={guess} eps max-abs unconditional {err_u:.3e} conditional {err_c:.3e}")
    assert err_u < EPS_TOL and err_c < EPS_TOL, (err_u, err_c)


def test_reference_guess_mode_step_golden():
    g = torch.load(os.path.join(GOLD, "t2i_guess.pt"))
    m = g["meta"]
    eng = DenoiseEngine(TINY, make_state_dict(TINY, "unet", m["unet_seed"]),
                        [make_state_dict(TINY, "controlnet", m["cn_seed"])], DEV)
    N = m["N"]
    eng.prepare(torch.cat([g["ctx_uncond"], g["ctx_cond"]]), [g["hint"]], [m["scale"]], guess_mode=True,
                controlnet_rows="conditional")
    eps = eng.eps(torch.cat([g["x"], g["x"]]), g["timestep"]).cpu()
    assert (eps[:N] - g["e_uncond"]).abs().max().item() < EPS_TOL
    assert (eps[N:] - g["e_cond"]).abs().max().item() < EPS_TOL
    eng.begin(g["x"], m["guidance"], use_graph=True)
    eng.step(g["timestep"], g["a_t"], g["a_prev"])
    assert (eng.latents().cpu() - g["x_prev"]).abs().max().item() < EPS_TOL


# ================================================ CUDA graphs ===================================================
def _request(eng, guess, n_img, use_graph, seed=4):
    x, ctx, hints = make_inputs(TINY, 2 * n_img, 16, 13, seed, n_controlnets=1)
    if guess:
        eng.prepare(ctx, [hints[0][:n_img]], [0.8], guess_mode=True, controlnet_rows="conditional")
    else:
        eng.prepare(ctx, hints, [0.8], cfg_duplicated=True)
    ts, a, ap = ddim_schedule(6)
    eng.set_schedule(ts, a, ap)
    eng.begin(x[:n_img, :4], guidance=6.0, use_graph=use_graph)
    for _ in ts:
        eng.step()
    return eng.latents().cpu()


def test_graph_replay_equals_eager_and_guess_switch_recaptures():
    mk = lambda: DenoiseEngine(TINY, make_state_dict(TINY, "unet", 51), [make_state_dict(TINY, "controlnet", 52)], DEV)  # noqa: E731
    eng = mk()
    graphs = []
    for guess in (True, False, True):
        got = _request(eng, guess, 2, True)
        graphs.append(eng._graph)
        assert torch.equal(got, _request(mk(), guess, 2, False)), guess
    assert graphs[0] is not graphs[1] and graphs[1] is not graphs[2]
    # the same guess-mode request again keeps a valid graph and gives the same latents
    assert torch.equal(_request(eng, True, 2, True), _request(eng, True, 2, True))


# ================================================ the application ===============================================
@pytest.mark.parametrize("extra_inpaint", [True, False])
def test_process_all_region_generation_end_to_end(tmp_path, monkeypatch, extra_inpaint):
    from editanything_b200 import app
    from editanything_b200.pipeline import StableDiffusionControlNetInpaintPipeline, StableDiffusionControlNetPipeline
    from tests.test_app_cpu import FakeSam, _inputs
    from tests.test_nogradio_cpu import make_model_root
    make_model_root(str(tmp_path / "hub"))
    monkeypatch.setenv("EA_MODEL_ROOT", str(tmp_path / "hub"))
    monkeypatch.setenv("EA_SAVE_INPUT", "0")
    monkeypatch.chdir(tmp_path)
    model = app.EditAnythingLoraModel(base_model_path="runwayml/stable-diffusion-v1-5", lora_model_path=None,
                                      use_blip=False, sam_generator=FakeSam(), mask_predictor=object(),
                                      extra_inpaint=extra_inpaint)
    first = model.pipe
    args, kwargs = _inputs()
    args = (args[0], True) + args[2:10] + (6,) + args[11:]
    kwargs = dict(kwargs, refine_alignment_ratio=0.5)
    for guess in (False, True):
        a = args[:11] + (guess,) + args[12:]
        tile, res, masks, _ = model.process(*a, **kwargs)
        cls = StableDiffusionControlNetPipeline if extra_inpaint else StableDiffusionControlNetInpaintPipeline
        assert type(model.pipe) is cls and len(model.pipe.engine.cns) == 1
        assert model.pipe.engine.unet is first.engine.unet
        assert model.pipe.engine.B == 4
        assert len(res) == 2 and len(tile) == 2
        assert all(i.size == (64, 64) for i in res) and all(i.size == (128, 128) for i in tile)
        assert all(np.isfinite(np.array(i, dtype=np.float32)).all() and np.array(i).std() > 0 for i in res + tile)
        assert np.array(masks[1]).min() == 255
