"""-m gpu: the alpha-mixing inpaint pipeline on the H100.

ea_latent_mix per element against float64 (window on and off, the inactive last row, counters outside the table,
alpha 0 and 1, fractional masks, ragged and grid-stride pixel counts, lat_half_out rewritten in both copies) and its
rejections before any launch; then the kernel through the float64 launch audit (tests/launch_audit.py) on a mixing
step's production arguments; the launch counts of the captured steps; the SD1.5-shaped step with two ControlNets at
512x512 against an eager step (eng.eps, the DDIM update and the mix on the host); and the tiny pipeline, captured,
against the float64 restatement of the reference's __call__ (tests/mixing_ref.py) on the same noise."""
import ctypes as C
import math

import pytest
import torch

from editanything_b200 import _lib as L
from editanything_b200 import ops
from editanything_b200.denoise import DenoiseEngine, ddim_schedule
from editanything_b200.pipeline import DDIMScheduler, StableDiffusionControlNetInpaintMixingPipeline
from editanything_b200.schedulers import UniPCMultistepScheduler
from editanything_b200.unet_spec import SD15, TINY, make_state_dict
from oracle.inputs import make_inputs
from tests import fp64_refs as R
from tests import launch_audit as LA
from tests.inpaint_ref import RecordingVAE
from tests.mixing_ref import mix_ref, reference_mixing
from tests.test_gpu_kernels_fp64 import DEV, U, _close, _gen, _randn

pytestmark = pytest.mark.gpu


def _mix_bound(x, known, noise, k_init, k_noise):
    """fp32 evaluation of p = k_init known + k_noise noise and the two convex combinations: a few roundings of
    terms no larger than |x| + |p| each."""
    return 8 * U * (x.abs() + abs(k_init) * known.abs() + abs(k_noise) * noise.abs()) + 1e-30


# ================================================ ea_latent_mix against float64 =================================
CASES = {
    # name: (Nimg, H, W, copies, counter, rows [(k_init, k_noise, in_window, active)], alpha)
    "window_guided_64x64_n1": (1, 64, 64, 2, 1, [(0.9, 0.4, 1, 1), (0.8, 0.6, 0, 1), (1.0, 0.0, 0, 0)], 0.5),
    "outside_window_unguided_ragged_n3": (3, 7, 13, 1, 2, [(0.9, 0.4, 1, 1), (0.8, 0.6, 0, 1), (1.0, 0.0, 0, 0)], 0.3),
    "alpha0_window_n2": (2, 24, 40, 2, 1, [(0.95, 0.3, 1, 1), (1.0, 0.0, 0, 0)], 0.0),
    "alpha1_outside_n2": (2, 24, 40, 2, 1, [(0.7, 0.7, 0, 1), (1.0, 0.0, 0, 0)], 1.0),
    "inactive_last_row": (2, 16, 24, 2, 2, [(0.9, 0.4, 1, 1), (1.0, 0.0, 0, 0)], 0.5),
    "counter_zero": (1, 8, 8, 2, 0, [(0.9, 0.4, 1, 1)], 0.5),
    "counter_past_table": (1, 8, 8, 1, 4, [(0.9, 0.4, 1, 1), (0.9, 0.4, 1, 1)], 0.5),
    "grid_stride_784x800_n1": (1, 784, 800, 2, 1, [(0.9, 0.4, 0, 1), (1.0, 0.0, 0, 0)], 0.6),
}


@pytest.mark.parametrize("name", list(CASES))
def test_latent_mix_fp64(name):
    N, H, W, copies, ctr_v, rows, alpha = CASES[name]
    h = ops.half_dtype()
    n_rows = len(rows)
    lat = _randn((N, H, W, 4), 71)
    known = _randn((N, H, W, 4), 72, scale=0.8)
    noise = _randn((n_rows, N, H, W, 4), 73)
    mask = (torch.rand(N, H, W, generator=_gen(74), device=DEV) < 0.5).float()
    mask[:, :1] = 0.37                                             # a fractional row: both terms of every blend live
    mix = torch.tensor(rows, dtype=torch.float32, device=DEV)
    ctr = torch.full((1,), ctr_v, dtype=torch.int32, device=DEV)
    half = torch.full((copies * N, H, W, 4), 7.0, device=DEV, dtype=h)
    lat0, half0 = lat.clone(), half.clone()
    ops.latent_mix(lat, known, mask, noise, mix, alpha=alpha, step_counter=ctr, lat_half_out=half, copies=copies,
                   Nimg=N, H=H, W=W)
    torch.cuda.synchronize()
    assert int(ctr.item()) == ctr_v                                # read, never written
    r = ctr_v - 1
    if not (0 <= r < n_rows and rows[r][3]):
        assert torch.equal(lat, lat0) and torch.equal(half, half0)
        return
    ki, kn, win, _ = rows[r]
    x, kd, zd, md = lat0.double(), known.double(), noise[r].double(), mask.double()[..., None]
    ref = mix_ref(x, kd, md, zd, ki, kn, bool(win), alpha)
    bound = _mix_bound(x, kd, zd, ki, kn)
    _close("ea_latent_mix", f"latents {name}", lat, ref, bound)
    for c in range(copies):
        _close("ea_latent_mix", f"lat_half[{c}] {name}", half[c * N:(c + 1) * N], ref, bound + R.ulp(ref, h))
    assert torch.equal(half[:N], half[N:]) or copies == 1
    if alpha in (0.0, 1.0):                                        # the degenerate weights are exact selections
        p = ki * kd + kn * zd
        sel = (md == 0).expand_as(ref)
        want = (x if alpha == 0.0 else p)[sel]
        assert (lat.double()[sel] - want).abs().max().item() <= (8 * U * (x.abs() + p.abs()))[sel].max().item()


def test_latent_mix_rejections_before_launch():
    lib = L.lib()
    N, H, W = 1, 8, 8
    lat, known, noise = (torch.zeros(N * H * W * 4 + 4, device=DEV) for _ in range(3))
    mask, mix = torch.zeros(N * H * W, device=DEV), torch.zeros(1, 4, device=DEV)
    ctr = torch.ones(1, dtype=torch.int32, device=DEV)
    half = torch.zeros(2 * N * H * W * 4 + 4, device=DEV, dtype=ops.half_dtype())
    p = [t.data_ptr() for t in (lat, known, mask, noise, mix)]

    def call(latents=p[0], known_=p[1], mask_=p[2], noise_=p[3], mix_=p[4], ctr_=ctr.data_ptr(), half_=half.data_ptr(),
             copies=2, n=N, rows=1):
        return lib.ea_latent_mix(latents, known_, mask_, noise_, mix_, C.c_float(0.5), ctr_, rows, half_, copies, n, H,
                                 W, None)
    n0 = ops.launch_count()
    assert call(latents=None) == -1 and call(known_=None) == -1 and call(mask_=None) == -1
    assert call(noise_=None) == -1 and call(mix_=None) == -1 and call(ctr_=None) == -1
    assert call(copies=0) == -1 and call(copies=3) == -1
    assert call(n=0) == -2 and call(rows=0) == -2
    assert call(latents=p[0] + 4) == -2 and call(known_=p[1] + 8) == -2 and call(noise_=p[3] + 4) == -2
    assert call(half_=half.data_ptr() + 2) == -2
    assert ops.launch_count() == n0                                # nothing was launched
    assert call(half_=None) == 0 and ops.launch_count() == n0 + 1
    torch.cuda.synchronize()


# ================================================ the launch audit ==============================================
def h_latent_mix(be, a, hdt):
    N, H, W_, copies = a["Nimg"], a["H"], a["W"], a["copies"]
    n_rows = a["mix"].shape[0]
    px = (N, H, W_)
    o = [LA.dense("latents", a["latents"], px + (4,), "rw"), LA.dense("known", a["known"], px + (4,)),
         LA.dense("mask", a["mask"], px), LA.dense("noise", a["noise"], (n_rows,) + px + (4,)),
         LA.dense("mix", a["mix"], (n_rows, 4)), LA.dense("step_counter", a["step_counter"], (1,))]
    if a.get("lat_half_out") is not None:
        o.append(LA.dense("lat_half_out", a["lat_half_out"], (copies * N,) + px[1:] + (4,), "w"))

    def check(snap, got):
        snap = LA._whole(snap)
        r = int(snap("step_counter")[0]) - 1
        mix = snap("mix")
        x = snap("latents")
        yield "step_counter", got("step_counter"), snap("step_counter"), None
        if not (0 <= r < n_rows and float(mix[r, 3]) != 0.0):
            yield "latents", got("latents"), x, None
            if a.get("lat_half_out") is not None:
                yield "lat_half_out", got("lat_half_out"), snap("lat_half_out"), None
            return
        ki, kn, win = (float(v) for v in mix[r, :3])
        kd, zd = snap("known"), snap("noise")[r]
        ref = mix_ref(x, kd, snap("mask")[..., None], zd, ki, kn, win != 0.0, float(a["alpha"]))
        bound = _mix_bound(x, kd, zd, ki, kn)
        yield "latents", got("latents"), ref, bound
        if a.get("lat_half_out") is not None:
            lh = got("lat_half_out")
            for c in range(copies):
                yield f"lat_half_out[{c}]", lh[c * N:(c + 1) * N], ref, bound + R.ulp(ref, hdt)
    return LA.Spec("latent_mix", o, check)


def _mixing_request(eng, x, n_img, S=4, guided=True, alpha=0.4, use_graph=False, seed=5):
    g = torch.Generator().manual_seed(seed)
    ts, a, ap = ddim_schedule(S)
    n = len(ts)
    init = torch.randn(n_img, 4, x.shape[2], x.shape[3], generator=g)
    m = (torch.rand(n_img, 1, x.shape[2], x.shape[3], generator=g) > 0.5).float()
    z = torch.randn(n - 1, n_img, 4, x.shape[2], x.shape[3], generator=g)
    k = [(0.9 - 0.05 * i, 0.3 + 0.05 * i) for i in range(n)]
    mix = ([v[0] for v in k], [v[1] for v in k], [1.0 if i < 0.5 * n else 0.0 for i in range(n)],
           [1.0] * (n - 1) + [0.0])
    eng.set_schedule(ts, a, ap, mix=mix)
    eng.begin(x[:n_img, :4], 7.0 if guided else 1.0, known_nchw=init, mask_n1hw=m, mix_alpha=alpha, mix_noise=z,
              use_graph=use_graph)
    return (ts, a, ap), (init, m, z, mix)


def test_latent_mix_launch_audit():
    """Two eager mixing steps of the tiny engine (guided, then unguided with two images), every launch audited on
    its production arguments; latent_mix among them, once per step."""
    LA.HANDLERS["latent_mix"] = h_latent_mix
    LA.RETURNS["latent_mix"] = None
    try:
        usd = make_state_dict(TINY, "unet", 61)
        csds = [make_state_dict(TINY, "controlnet", 62), make_state_dict(TINY, "controlnet", 63)]
        aud = LA.Auditor(ops, "mixing step")
        eng = DenoiseEngine(TINY, usd, csds, DEV, backend=aud)
        x, ctx, hints = make_inputs(TINY, 4, 8, 7, 5, n_controlnets=2)
        for guided, n_img in ((True, 1), (False, 2)):
            c = ctx[:2 * n_img] if guided else ctx[:n_img]
            hs = [h[:2 * n_img] if guided else h[:n_img] for h in hints]
            eng.prepare(c, hs, [0.5, 1.0], guided=guided)
            _mixing_request(eng, x, n_img, guided=guided)
            eng.step()
            eng.step()
        counts = {op: n for (op, _), n in aud.counts.items()}
        assert counts["latent_mix"] == 4, aud.counts
        print("\n" + aud.report("mixing step"))
    finally:
        LA.HANDLERS.pop("latent_mix", None)
        LA.RETURNS.pop("latent_mix", None)


# ================================================ launch counts and SD1.5 parity ===============================
def _host_mix(x, init, m, z, row, alpha):
    ki, kn, win, act = row
    if not act:
        return x
    return mix_ref(x, init, m, z, ki, kn, bool(win), alpha).float()


@pytest.mark.parametrize("n_img", [1, 2])
def test_sd15_two_controlnets_captured_mixing_matches_eager(n_img):
    """SD1.5 at 512x512 with two ControlNets and guidance: the captured mixing step, over a 4-step schedule, against
    an eager loop of eng.eps + the DDIM update + the mix on the host; and the launch counts: the plain inpaint step
    and the text-to-image step are the same launches, the mixing step one more."""
    torch.manual_seed(0)
    eng = DenoiseEngine(SD15, make_state_dict(SD15, "unet", 201),
                        [make_state_dict(SD15, "controlnet", s) for s in (202, 203)], DEV)
    g = torch.Generator().manual_seed(3)
    ctx = torch.randn(2 * n_img, 77, SD15.context_dim, generator=g)
    hints = [torch.randint(0, 256, (n_img, 3, 512, 512), generator=g).float(), torch.rand(n_img, 3, 512, 512, generator=g)]
    eng.prepare(ctx, [torch.cat([h, h]) for h in hints], [1.0, 0.8], cfg_duplicated=True)
    x = torch.randn(n_img, 4, 64, 64, generator=g)
    ts, a, ap = ddim_schedule(4)
    # the plain inpaint step and the text-to-image step (no blend) as captured steps
    eng.set_schedule(ts, a, ap, blend=([0.9] * 4, [0.3] * 4, [1.0] * 4))
    eng.begin(x, 7.0, known_nchw=x, mask_n1hw=torch.ones(n_img, 1, 64, 64), noise_nchw=x)
    eng.step()
    plain = eng.launches_per_step
    eng.set_schedule(ts, a, ap)
    eng.begin(x, 7.0)
    eng.step()
    assert eng.launches_per_step == plain
    (ts, a, ap), (init, m, z, mix) = _mixing_request(eng, x, n_img, S=4, use_graph=True)
    n = len(ts)
    got = []
    for _ in range(n):
        eng.step()
        got.append(eng.latents().cpu())
    assert eng.launches_per_step == plain + 1
    lat = x.clone()
    rows = list(zip(*mix))
    worst = 0.0
    for i in range(n):
        e = eng.eps(torch.cat([lat, lat]), int(ts[i])).cpu()
        e = e[:n_img] + 7.0 * (e[n_img:] - e[:n_img])
        x0 = (lat - math.sqrt(1 - a[i]) * e) / math.sqrt(a[i])
        lat = math.sqrt(ap[i]) * x0 + math.sqrt(1 - ap[i]) * e
        lat = _host_mix(lat, init, m, z[i] if i < n - 1 else z[0], rows[i], 0.4)
        err = (got[i] - lat).abs().max().item()
        worst = max(worst, err)
        assert err < 1e-2, (i, err)
        lat = got[i]                     # each step from the same input: the per-step tolerance of the parity tests
    print(f"\nSD1.5 512 N={n_img}: captured mixing step vs eager, worst max-abs {worst:.2e}, "
          f"{plain} / {eng.launches_per_step} launches per plain / mixing step")


# ================================================ the pipeline ==================================================
@pytest.mark.parametrize("sched", ["ddim", "unipc"])
def test_tiny_pipeline_captured_matches_restatement(sched):
    """The tiny pipeline on the H100 with the captured step, two images, a scale map: its draws come from the CUDA
    default generator, which torch.manual_seed(7) (the call's `generator`, as process() makes it) seeds too, so the
    restatement is fed the same draws (re-seeded and drawn in the same order)."""
    usd = make_state_dict(TINY, "unet", 51)
    csds = [make_state_dict(TINY, "controlnet", 52), make_state_dict(TINY, "controlnet", 53)]
    eng = DenoiseEngine(TINY, usd, csds, DEV)
    pipe = StableDiffusionControlNetInpaintMixingPipeline(eng, vae=RecordingVAE())
    mk = DDIMScheduler if sched == "ddim" else (lambda: UniPCMultistepScheduler.from_config(DDIMScheduler().config))
    pipe.scheduler = mk()
    g = torch.Generator().manual_seed(0)
    image = torch.rand(1, 3, 64, 64, generator=g) * 2 - 1
    mask = torch.zeros(1, 1, 64, 64)
    mask[:, :, 16:48, 8:40] = 1.0
    conds = [torch.randint(0, 256, (1, 3, 64, 64), generator=g).float(), torch.rand(1, 3, 64, 64, generator=g)]
    pe, ne = torch.randn(1, 9, TINY.context_dim, generator=g), torch.randn(1, 9, TINY.context_dim, generator=g)
    smap = torch.linspace(0.2, 1.0, 64)[None, :].expand(64, 64).contiguous()
    out = pipe(image=image, mask_image=mask, controlnet_conditioning_image=conds, height=64, width=64,
               num_inference_steps=8, guidance_scale=5.0, generator=torch.manual_seed(7), prompt_embeds=pe,
               negative_prompt_embeds=ne, output_type="latent", controlnet_conditioning_scale=[0.5, 1.0],
               num_images_per_prompt=2, alignment_ratio=0.7, alpha_weight=0.4,
               controlnet_conditioning_scale_map=smap).images.cpu()
    assert eng._graph is not None and eng.mix_tab is not None
    n = len(pipe.scheduler.timesteps)
    torch.manual_seed(7)                  # generator=torch.manual_seed(7) seeded the CUDA generator as well
    draws = [torch.randn(2, 4, 8, 8, device=DEV).cpu() for _ in range(n)]
    real_randn_like = torch.randn_like
    it = iter(draws)
    try:
        torch.randn_like = lambda t, **k: next(it).to(t.dtype)
        ref = reference_mixing(TINY, usd, csds, image, mask, conds, pe, ne, steps=8, gs=5.0,
                               scales=[0.5 * smap, 1.0 * smap], seed=7, alpha=0.4, ratio=0.7, vae=RecordingVAE(),
                               n_img=2, scheduler=mk())
    finally:
        torch.randn_like = real_randn_like
    assert next(it, None) is None                                  # the restatement took exactly the pipeline's draws
    err = (out.double() - ref).abs().max().item()
    rel = ((out.double() - ref).norm() / ref.norm()).item()
    assert rel < 3e-2 and err < 0.15, (err, rel)                   # the gates of tests/test_gpu_pipeline.py
