"""-m gpu: the operators of ea_pointwise.cu, and the row_scale / out_f32 inputs of the ea_gemm epilogue, against
float64 references (tests/fp64_refs.py) at the shapes, strides and value ranges production reaches.

Every gate is per element:
  * layout / copy operators must match the reference bit for bit;
  * normalisations: 1 ulp of the storage dtype at the reference value, plus 16 fp32 ulps of each term of
    g (x - mu) r + b (an fp32 evaluation cannot do better where those terms cancel);
  * reductions: ulp_out(ref) + K u sum |a_i b_i| (u = 2^-24, K = reduction length, ulp_out = 0 for fp32 outputs),
    propagated through whatever formula is applied to the reduced value;
  * ea_softmax_rows (uses __expf): 1 ulp of the output plus 1e-5 |ref|.
A failure names the worst element (index, value, reference, bound)."""
import math

import numpy as np
import pytest
import torch

from editanything_b200 import _lib as L
from editanything_b200 import ops
from editanything_b200.pipeline import DDIMScheduler
from editanything_b200.schedulers import UniPCMultistepScheduler
from tests import fp64_refs as R

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
U = R.U32
NORM_K = 16.0          # fp32 ulps allowed on each term of the normalisations' affine map
WORST = {}             # kernel -> worst |err| / bound seen in this run


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if WORST:
        print("\nworst error / bound per kernel:")
        for k in sorted(WORST):
            print(f"  {k:24s} {WORST[k]:.3f}")


def _half():
    return ops.half_dtype()


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _randn(shape, seed, dtype=torch.float32, scale=1.0, offset=0.0):
    return (torch.randn(shape, generator=_gen(seed), device=DEV, dtype=torch.float32) * scale + offset).to(dtype)


def _close(kernel, what, got, ref, bound):
    """|got - ref| <= bound element-wise (NaN fails); records the worst ratio under `kernel`."""
    got = got.double()
    err = (got - ref).abs()
    ratio = torch.where(err == 0, torch.zeros_like(err), err / bound)
    ratio = torch.where(torch.isnan(err), torch.full_like(err, math.inf), ratio)
    i = int(torch.argmax(ratio.reshape(-1)))
    worst = float(ratio.reshape(-1)[i])
    WORST[kernel] = max(WORST.get(kernel, 0.0), worst)
    if not worst <= 1.0:
        idx = tuple(int(v) for v in np.unravel_index(i, tuple(ref.shape)))
        n_bad = int((~(err <= bound)).sum())
        raise AssertionError(f"{kernel} {what}: {n_bad} of {ref.numel()} elements out of bound; worst at {idx}: "
                             f"got {float(got.reshape(-1)[i])!r}, ref {float(ref.reshape(-1)[i])!r}, "
                             f"bound {float(bound.reshape(-1)[i]):.3e} (ratio {worst:.3g})")
    return worst


def _exact(kernel, what, got, ref):
    """Bitwise equality with the reference cast to the output dtype."""
    want = ref.to(got.dtype)
    if torch.equal(got, want):
        WORST[kernel] = max(WORST.get(kernel, 0.0), 0.0)
        return
    diff = (got != want) & ~(torch.isnan(got) & torch.isnan(want))
    i = int(torch.nonzero(diff.reshape(-1))[0])
    idx = tuple(int(v) for v in np.unravel_index(i, tuple(got.shape)))
    raise AssertionError(f"{kernel} {what}: {int(diff.sum())} elements differ; first at {idx}: "
                         f"got {float(got.reshape(-1)[i])!r}, ref {float(want.reshape(-1)[i])!r}")


def _untouched(kernel, what, region, sentinel):
    if not torch.equal(region, sentinel):
        raise AssertionError(f"{kernel} {what}: wrote outside its destination")


class _concurrent_lane:
    """The kernel variants without inter-CTA waits (two-pass GroupNorm, no_spin split-K), as used under concurrent
    streams; the default lane is always restored."""

    def __enter__(self):
        ops.set_lane(1, True)

    def __exit__(self, *exc):
        ops.set_lane(0, False)
        return False


# ================================================ GroupNorm ====================================================
GN_CASES = {
    # UNet levels (SD1.5 512^2, image + CFG)
    "unet64_c320": dict(B=2, HW=64 * 64, C=320),
    "unet32_c640": dict(B=2, HW=32 * 32, C=640),
    "unet16_c1280": dict(B=2, HW=16 * 16, C=1280),
    # decoder skip-concatenations, C1 not a multiple of the group size
    "unet8_c2560_cat": dict(B=2, HW=8 * 8, C=2560, C1=1280),
    "unet16_c1920_cat": dict(B=2, HW=16 * 16, C=1920, C1=1280),
    "unet64_c960_cat_strided": dict(B=2, HW=64 * 64, C=960, C1=640, xpad=16, opad=64),
    # SpatialTransformer norm: no SiLU, eps 1e-6, rows read from a wider buffer
    "transformer_norm": dict(B=2, HW=32 * 32, C=640, eps=1e-6, silu=False, xpad=64, opad=32),
    # VAE at 512^2: the 512^2 and 256^2 levels do not fit shared memory (uncached path), 64^2 does
    "vae512_c128": dict(B=1, HW=512 * 512, C=128, eps=1e-6),
    "vae256_c256": dict(B=1, HW=256 * 256, C=256, eps=1e-6),
    "vae64_c512": dict(B=1, HW=64 * 64, C=512, eps=1e-6),
    # SD2.1 768^2, 4 images + CFG, UNet + 2 ControlNets stacked: uncached, three affine sets
    "sd21_768_lockstep": dict(B=24, HW=96 * 96, C=320, n_nets=3),
    # groups whose variance is comparable to eps
    "small_variance": dict(B=2, HW=32 * 32, C=320, std=3.2e-3),
    # groups whose mean is far from zero relative to their spread (|mean| / std = 100, 256)
    "offset100": dict(B=2, HW=64 * 64, C=320, offset=25.0, std=0.25),
    "offset256": dict(B=2, HW=64 * 64, C=320, offset=64.0, std=0.25),
    "offset256_vae_uncached": dict(B=1, HW=256 * 256, C=256, offset=64.0, std=0.25, eps=1e-6),
}


def _gn_inputs(B, HW, C, C1=None, xpad=0, opad=0, n_nets=1, offset=0.0, std=1.0, seed=0, groups=32, **_):
    h = _half()
    # per-group mean (+-offset) and spread
    sign = torch.where(torch.rand(B, 1, groups, 1, generator=_gen(seed + 1), device=DEV) < 0.5, -1.0, 1.0)
    vals = _randn((B, HW, groups, C // groups), seed) * std + sign * offset
    vals = vals.reshape(B, HW, C).to(h)
    if C1 is None:
        x = torch.zeros(B, HW, C + xpad, device=DEV, dtype=h)
        x[..., :C] = vals
        srcs = dict(x=x, ldx=C + xpad)
    else:
        x = torch.zeros(B, HW, C1 + xpad, device=DEV, dtype=h)
        x2 = torch.zeros(B, HW, C - C1 + xpad, device=DEV, dtype=h)
        x[..., :C1], x2[..., :C - C1] = vals[..., :C1], vals[..., C1:]
        srcs = dict(x=x, ldx=C1 + xpad, x2=x2, ldx2=C - C1 + xpad, C1=C1)
    gam = [_randn((C,), seed + 10 + i, scale=0.5, offset=1.0) for i in range(n_nets)]
    bet = [_randn((C,), seed + 20 + i, scale=0.3) for i in range(n_nets)]
    out = torch.full((B, HW, C + opad), 7.0, device=DEV, dtype=h)
    return vals, srcs, gam, bet, out


def _gn_run(case, two_pass, silu=None, eps=None):
    c = dict(case)
    B, HW, C = c["B"], c["HW"], c["C"]
    silu = c.get("silu", True) if silu is None else silu
    eps = c.get("eps", 1e-5) if eps is None else eps
    n_nets = c.get("n_nets", 1)
    vals, srcs, gam, bet, out = _gn_inputs(**c)
    ws = ops.gn_workspace(B, DEV)
    x = srcs.pop("x")
    kw = dict(B=B, HW=HW, C_=C, eps=eps, silu=silu, workspace=ws, ldo=out.shape[-1], **srcs)
    g_arg, b_arg = (gam, bet) if n_nets > 1 else (gam[0], bet[0])
    outs = []
    for _ in range(2):
        if two_pass:
            with _concurrent_lane():
                ops.groupnorm(x, g_arg, b_arg, out, **kw)
        else:
            ops.groupnorm(x, g_arg, b_arg, out, **kw)
        torch.cuda.synchronize()
        assert not ws[:2 * B].view(torch.int32).any(), "workspace counters not left zero"
        outs.append(out.clone())
    assert torch.equal(outs[0], outs[1]), "two identical calls differ"
    if out.shape[-1] > C:
        _untouched("ea_groupnorm", "row padding", out[..., C:], torch.full_like(out[..., C:], 7.0))
    y, pre, terms = R.groupnorm(vals.double(), [g.double() for g in gam], [b.double() for b in bet], 32, eps, silu)
    e_aff = NORM_K * U * terms
    if silu:
        bound = R.ulp(y, _half()) + 1.1 * e_aff + R.silu_eval_err(pre)
    else:
        bound = R.ulp(y, _half()) + e_aff
    del terms, pre
    return _close("ea_groupnorm", f"{'two_pass' if two_pass else 'fused'}", out[..., :C], y, bound)


@pytest.mark.parametrize("two_pass", [False, True], ids=["fused", "two_pass"])
@pytest.mark.parametrize("name", list(GN_CASES))
def test_groupnorm(name, two_pass):
    _gn_run(GN_CASES[name], two_pass)


@pytest.mark.parametrize("two_pass", [False, True], ids=["fused", "two_pass"])
@pytest.mark.parametrize("eps", [1e-5, 1e-6])
@pytest.mark.parametrize("silu", [True, False])
def test_groupnorm_flags(silu, eps, two_pass):
    _gn_run(dict(B=2, HW=32 * 32, C=640, xpad=8, opad=8), two_pass, silu=silu, eps=eps)


# ================================================ LayerNorm ====================================================
@pytest.mark.parametrize("eps", [1e-5, 1e-6])
@pytest.mark.parametrize("C", [8, 72, 320, 1280, 2048])
def test_layernorm(C, eps):
    h = _half()
    M, xpad, opad = 301, 24, 16
    vals = _randn((M, C), 1)
    vals[0] = _randn((C,), 2, scale=0.25, offset=64.0)        # one row with |mean| / std = 256
    vals[1] = _randn((C,), 3, scale=3.2e-3)                    # one row whose variance is comparable to eps
    vals = vals.to(h)
    x = torch.zeros(M, C + xpad, device=DEV, dtype=h)
    x[:, :C] = vals
    gamma, beta = _randn((C,), 4, scale=0.5, offset=1.0), _randn((C,), 5, scale=0.3)
    out = torch.full((M, C + opad), 7.0, device=DEV, dtype=h)
    ops.layernorm(x, gamma, beta, out, M=M, C_=C, eps=eps, ldx=C + xpad, ldo=C + opad)
    _untouched("ea_layernorm", "row padding", out[:, C:], torch.full_like(out[:, C:], 7.0))
    y, terms = R.layernorm(vals.double(), gamma.double(), beta.double(), eps)
    _close("ea_layernorm", f"C={C}", out[:, :C], y, R.ulp(y, h) + NORM_K * U * terms)


# ================================================ conv_in ======================================================
@pytest.mark.parametrize("HW", [(64, 64), (1, 9), (7, 13)], ids=lambda s: f"{s[0]}x{s[1]}")
@pytest.mark.parametrize("Cout", [320, 128])
@pytest.mark.parametrize("Cin", [4, 8])
def test_conv_in(Cin, Cout, HW):
    h = _half()
    H, W = HW
    B = 2
    x = _randn((B, H, W, Cin), 11, h)
    w = _randn((3, 3, Cin, Cout), 12, scale=(9 * Cin) ** -0.5)
    bias = None if W == 9 else _randn((Cout,), 13)
    add = _randn((B, H, W, Cout), 14, h)
    ldo = Cout + 64
    out = torch.full((B, H, W, ldo), 7.0, device=DEV, dtype=h)
    slot = torch.full((B, H, W, 2 * Cout), 5.0, device=DEV, dtype=h)      # skip-concat slot: first Cout channels
    ops.conv_in(x, w, bias, out, B=B, H=H, W=W, Cin=Cin, Cout=Cout, out2=slot, add=add, ldo=ldo, ldo2=2 * Cout)
    _untouched("ea_conv_in", "out padding", out[..., Cout:], torch.full_like(out[..., Cout:], 7.0))
    _untouched("ea_conv_in", "out2 slot neighbours", slot[..., Cout:], torch.full_like(slot[..., Cout:], 5.0))
    assert torch.equal(out[..., :Cout], slot[..., :Cout]), "out and out2 differ"
    ref, mag = R.conv_nhwc(x.double(), w.double(), None if bias is None else bias.double())
    ref = ref + add.double()
    K = 9 * Cin + 2
    bound = R.ulp(ref, h) + K * U * (mag + add.double().abs())
    _close("ea_conv_in", f"{Cin}->{Cout} {H}x{W}", out[..., :Cout], ref, bound)


# ================================================ conv_direct ==================================================
CD_CASES = {
    "hint_3_16": dict(Hin=64, Win=64, Cin=3, Cout=16, k=3, s=1, silu=True),
    "hint_16_32_s2_odd": dict(Hin=33, Win=33, Cin=16, Cout=32, k=3, s=2, silu=True),
    "hint_96_256_s2_odd": dict(Hin=17, Win=15, Cin=96, Cout=256, k=3, s=2, silu=True),
    "hint_256_320_add": dict(Hin=8, Win=8, Cin=256, Cout=320, k=3, s=1, silu=False, add=True, ldo=640),
    "quant_conv_k1": dict(Hin=64, Win=64, Cin=8, Cout=8, k=1, s=1, ldo=16),
    "post_quant_k1_add": dict(Hin=32, Win=24, Cin=4, Cout=4, k=1, s=1, add=True),
    "k1_s2_odd_silu": dict(Hin=33, Win=31, Cin=16, Cout=32, k=1, s=2, silu=True, ldo=40),
}


@pytest.mark.parametrize("name", list(CD_CASES))
def test_conv_direct(name):
    c = CD_CASES[name]
    h = _half()
    B, k, s = 2, c["k"], c["s"]
    Hin, Win, Cin, Cout = c["Hin"], c["Win"], c["Cin"], c["Cout"]
    Ho, Wo = -(-Hin // s), -(-Win // s)
    ldo = c.get("ldo", Cout)
    silu = c.get("silu", False)
    x = _randn((B, Hin, Win, Cin), 21, h)
    w = _randn((k, k, Cin, Cout), 22, scale=(k * k * Cin) ** -0.5)
    bias = _randn((Cout,), 23)
    add = _randn((B, Ho, Wo, Cout), 24, h) if c.get("add") else None
    out = torch.full((B, Ho, Wo, ldo), 7.0, device=DEV, dtype=h)
    ops.conv_direct(x, w, bias, out, B=B, Hin=Hin, Win=Win, Cin=Cin, Cout=Cout, ksize=k, stride=s, silu=silu,
                    add=add, ldo=ldo)
    if ldo > Cout:
        _untouched("ea_conv_direct", "out padding", out[..., Cout:], torch.full_like(out[..., Cout:], 7.0))
    pre, mag = R.conv_nhwc(x.double(), w.double(), bias.double(), stride=s)
    K = k * k * Cin + 1
    e = K * U * mag
    if silu:
        y = R.silu(pre)
        e = 1.1 * e + R.silu_eval_err(pre)
    else:
        y = pre
    a = add.double() if add is not None else torch.zeros_like(y)
    ref = y + a
    bound = R.ulp(ref, h) + e + 2 * U * (y.abs() + a.abs())
    _close("ea_conv_direct", name, out[..., :Cout], ref, bound)


# ================================================ out_cfg_ddim =================================================
def _out_conv_inputs(Nimg, H, W, C, seed):
    h = _half()
    xn = _randn((2 * Nimg, H, W, C), seed, h)
    w = _randn((4, 3, 3, C), seed + 1, scale=(9 * C) ** -0.5)
    bias = _randn((4,), seed + 2, scale=0.1)
    return xn, w, bias


def _eps_check(xn, w, bias, eps_out, C, what):
    ref, mag = R.out_conv(xn.double(), w.double(), bias.double())
    bound = (9 * C + 1) * U * mag
    _close("ea_out_cfg_ddim", f"eps {what}", eps_out, ref, bound)
    return ref, bound


OC_CASES = {
    "ddim_64x64_c320_g7.5": dict(Nimg=1, H=64, W=64, C=320, g=7.5),
    "ddim_24x40_c640_g1_blend_noise_half": dict(Nimg=2, H=24, W=40, C=640, g=1.0, blend=True, noise=True,
                                                  half_out=True),
    "ddim_16x48_c320_g7.5_blend": dict(Nimg=1, H=16, W=48, C=320, g=7.5, blend=True, half_out=True),
    "eps_only_32x20_c640": dict(Nimg=2, H=32, W=20, C=640, g=7.5, eps_only=True),
}


@pytest.mark.parametrize("name", list(OC_CASES))
def test_out_cfg_ddim_mode0(name):
    c = OC_CASES[name]
    h = _half()
    N, H, W, C, g = c["Nimg"], c["H"], c["W"], c["C"], c["g"]
    xn, w, bias = _out_conv_inputs(N, H, W, C, 31)
    eps_out = torch.full((2 * N, H, W, 4), 7.0, device=DEV)
    if c.get("eps_only"):
        ops.out_cfg_ddim(xn, w, bias, latents=None, eps_out=eps_out, coef=None, guidance=g, Nimg=N, H=H, W=W, C_=C)
        _eps_check(xn, w, bias, eps_out, C, name)
        return
    a_t, a_prev = 0.35, 0.62
    coef32 = torch.tensor([math.sqrt(a_t), math.sqrt(1 - a_t), math.sqrt(a_prev), math.sqrt(1 - a_prev),
                           0.8, 0.6, 1.0, 0.0] + [0.0] * 8, dtype=torch.float32, device=DEV)
    lat = _randn((N, H, W, 4), 32)
    lat0 = lat.double()
    known = _randn((N, H, W, 4), 33) if c.get("blend") else None
    noise = _randn((N, H, W, 4), 34) if c.get("noise") else None
    mask = None
    if known is not None:
        mask = (torch.rand(N, H, W, generator=_gen(35), device=DEV) < 0.4).float()
        mask[:, :2] = 0.37                                                   # soft mask values too
    lat_half = torch.full((2 * N, H, W, 4), 7.0, device=DEV, dtype=h) if c.get("half_out") else None
    ops.out_cfg_ddim(xn, w, bias, latents=lat, eps_out=eps_out, coef=coef32, guidance=g, known=known, noise=noise,
                     mask=mask, lat_half_out=lat_half, Nimg=N, H=H, W=W, C_=C)
    eref, ebound = _eps_check(xn, w, bias, eps_out, C, name)
    cf = [float(v) for v in coef32.double().cpu()]
    eu, ec, bu, bc = eref[:N], eref[N:], ebound[:N], ebound[N:]
    e = R.cfg(eu, ec, g)
    e_err = abs(1 - g) * bu + abs(g) * bc + 3 * U * (eu.abs() + abs(g) * (ec.abs() + eu.abs()))
    z = torch.zeros_like(lat0)
    x0 = R.ErrLin.lin([(1.0 / cf[0], lat0, z), (-cf[1] / cf[0], e, e_err)])
    xp = R.ErrLin.lin([(cf[2], x0[0], x0[1]), (cf[3], e, e_err)])
    if known is not None:
        xp = R.blend_err(xp, known.double(), None if noise is None else noise.double(), mask.double(), cf)
    ref, err = xp
    _close("ea_out_cfg_ddim", f"latents {name}", lat, ref, err)
    if lat_half is not None:
        hb = R.ulp(ref, h) + err
        _close("ea_out_cfg_ddim", f"lat_half uncond {name}", lat_half[:N], ref, hb)
        assert torch.equal(lat_half[:N], lat_half[N:]), "the two CFG copies of the latents differ"


@pytest.mark.parametrize("blend", [False, True], ids=["plain", "blend_noise"])
def test_out_cfg_unipc_schedule(blend):
    """Mode 1 over a whole 20-step UniPC (order 2) schedule: the latents after every step against scheduler.step()
    in float64, driven by the eps the kernel reports through eps_out (so the check isolates the update).  The bound
    is the running fp32 error of the coefficient-row recurrence (fp64_refs.unipc_fused, (n + 2) u per linear
    combination of n terms), accumulated over the steps."""
    N, H, W, C, g = 2, 16, 24, 320, 7.5
    sched = UniPCMultistepScheduler.from_config(DDIMScheduler().config, solver_order=2)
    sched.set_timesteps(20)
    ts = sched.timesteps.tolist()
    blend_rows = None
    known = noise = mask = None
    if blend:
        on = [1.0 if (i < 12 and i % 5 != 3) else 0.0 for i in range(len(ts))]     # window with toggles
        nxt = ts[1:] + [0]
        blend_rows = [(float(sched.alpha_t[t]), float(sched.sigma_t[t]), o) for t, o in zip(nxt, on)]
        known, noise = _randn((N, H, W, 4), 41), _randn((N, H, W, 4), 42)
        mask = (torch.rand(N, H, W, generator=_gen(43), device=DEV) < 0.5).float()
    rows = R.unipc_coef_rows(sched, blend_rows)
    coef_tab = torch.tensor(rows, device=DEV)
    if blend:                    # the reference blends with the fp32 values the kernel reads
        blend_rows = [(float(r[4]), float(r[5]), float(r[6])) for r in rows]
    lat = _randn((N, H, W, 4), 44)
    x_init = lat.double()
    hist = torch.zeros(3, N, H, W, 4, device=DEV)
    eps_out = torch.empty(2 * N, H, W, 4, device=DEV)
    coef = torch.empty(16, device=DEV)
    eps_list, lats = [], []
    for i in range(len(ts)):
        xn, w, bias = _out_conv_inputs(N, H, W, C, 100 + 7 * i)
        coef.copy_(coef_tab[i])
        ops.out_cfg_ddim(xn, w, bias, latents=lat, eps_out=eps_out, coef=coef, guidance=g, known=known, noise=noise,
                         mask=mask, hist=hist, Nimg=N, H=H, W=W, C_=C)
        _eps_check(xn, w, bias, eps_out, C, f"step {i}")
        e = eps_out.double()
        eps_list.append((e[:N], e[N:]))
        lats.append(lat.clone())
    kw = dict(known=None if known is None else known.double(), noise=None if noise is None else noise.double(),
              mask=None if mask is None else mask.double())
    ref = R.scheduler_trajectory(sched, eps_list, x_init, g, blend_rows, **kw)
    bounds = R.unipc_fused(rows, eps_list, x_init, g, **kw)
    for i, (got, r, (_, err)) in enumerate(zip(lats, ref, bounds)):
        _close("ea_out_cfg_ddim", f"UniPC latents after step {i} (t={ts[i]})", got, r, err)


# ================================================ small_linear / timestep ======================================
@pytest.mark.parametrize("N", [1280, 1283])
@pytest.mark.parametrize("K", [320, 1280, 1288])
@pytest.mark.parametrize("M", [1, 2, 8, 16])
def test_small_linear(M, K, N):
    h = _half()
    silu_in = silu_out = (K != 320)          # time_embed[2] reads SiLU'd rows, emb_layers apply SiLU first
    x = _randn((M, K), 51, scale=2.0)
    w = _randn((N, K), 52, h, scale=K ** -0.5)
    bias = None if N == 1283 else _randn((N,), 53)
    y = torch.full((M, N), 7.0, device=DEV)
    ops.small_linear(x, w, bias, y, M=M, N=N, K=K, silu_in=silu_in, silu_out=silu_out)
    x64, w64 = x.double(), w.double()
    ref, pre, mag = R.small_linear(x64, w64, None if bias is None else bias.double(), silu_in, silu_out)
    e = (K + 1) * U * mag
    if silu_in:
        e = e + R.silu_eval_err(x64) @ w64.abs().T
    if silu_out:
        e = 1.1 * e + R.silu_eval_err(pre)
    _close("ea_small_linear", f"M={M} K={K} N={N}", y, ref, e)


@pytest.mark.parametrize("dim", [320, 256])
def test_timestep_embedding(dim):
    t = torch.tensor([0.0, 1.0, 0.5, 500.0, 981.0, 999.0], device=DEV)
    out = torch.full((t.numel(), dim), 7.0, device=DEV)
    ops.timestep_embedding(t, out, B=t.numel(), dim=dim)
    ref, arg, xf = R.timestep_embedding(t.double(), dim)
    # fp32 argument: the exponent ln(1e4) i / half is rounded (error ~ u |x|, amplified by exp), then exp, then t * f
    arg_err = (3 * xf[None].abs() + 4) * U * arg.abs()
    bound = torch.cat([arg_err, arg_err], dim=-1) + 4 * U
    _close("ea_timestep_embedding", f"dim={dim}", out, ref, bound)


# ================================================ SAM / VAE helpers ============================================
@pytest.mark.parametrize("case", [(1, 64, 16, 80, True), (4, 14, 16, 80, False)],
                         ids=["global_S64_fused_qkv", "window_S14"])
def test_sam_relpos(case):
    B, S, heads, d, fused = case
    h = _half()
    if fused:                   # q read straight out of the fused qkv projection [B, S^2, 3 heads d]
        qkv = _randn((B, S * S, 3 * heads * d), 61, h)
        q = qkv[..., :heads * d]
        q_bs, q_ns = S * S * 3 * heads * d, 3 * heads * d
    else:
        qkv = _randn((B, S * S, heads * d), 61, h)
        q = qkv
        q_bs, q_ns = S * S * heads * d, heads * d
    Rh, Rw = _randn((S, S, d), 62, scale=0.2), _randn((S, S, d), 63, scale=0.2)
    rel_h = torch.full((B * heads, S * S, S), 7.0, device=DEV)
    rel_w = torch.full_like(rel_h, 7.0)
    ops.sam_relpos(qkv, q_bs, q_ns, Rh, Rw, rel_h, rel_w, B=B, heads=heads, S=S, d=d)
    rh, rw, mh, mw = R.sam_relpos(q.reshape(B, S * S, heads, d).double(), Rh.double(), Rw.double())
    _close("ea_sam_relpos", "rel_h", rel_h, rh, (d + 1) * U * mh)
    _close("ea_sam_relpos", "rel_w", rel_w, rw, (d + 1) * U * mw)


@pytest.mark.parametrize("cols", [64, 1028, 4096])
def test_softmax_rows(cols):
    h = _half()
    rows, lds, ldp = 37, cols + 12, cols + 8
    s = torch.full((rows, lds), 1e30, device=DEV)           # padding must not be read
    logits = _randn((rows, cols), 71, scale=4.0)
    logits[0, cols // 3] = 60.0                              # one dominant logit
    logits[1] = 3.0                                          # all equal
    logits[2] = -50.0 + _randn((cols,), 72, scale=0.01)      # large negative, near equal
    s[:, :cols] = logits
    p = torch.full((rows, ldp), 7.0, device=DEV, dtype=h)
    ops.softmax_rows(s, p, rows=rows, cols=cols, lds=lds, ldp=ldp)
    _untouched("ea_softmax_rows", "row padding", p[:, cols:], torch.full_like(p[:, cols:], 7.0))
    ref = R.softmax_rows(logits.double())
    _close("ea_softmax_rows", f"cols={cols}", p[:, :cols], ref, R.ulp(ref, h) + 1e-5 * ref.abs())


def test_upsample2x_exact():
    h = _half()
    x = _randn((2, 16, 24, 320), 81, h)
    out = torch.empty(2, 32, 48, 320, device=DEV, dtype=h)
    ops.upsample2x(x, out, B=2, H=16, W=24, C_=320)
    _exact("ea_upsample2x", "16x24", out, R.upsample2x(x.double()))


@pytest.mark.parametrize("HWs", [(64, 64, 14), (20, 27, 8)], ids=["sam_64_ws14", "ragged_20x27_ws8"])
def test_window_partition_roundtrip_exact(HWs):
    h = _half()
    H, W, ws = HWs
    B, C = 2, 160
    x = _randn((B, H, W, C), 82, h)
    nW = -(-H // ws) * -(-W // ws)
    xw = torch.full((B * nW, ws, ws, C), 7.0, device=DEV, dtype=h)
    ops.window_partition(x, xw, B=B, H=H, W=W, C_=C, ws=ws)
    _exact("ea_window_partition", f"{H}x{W}", xw, R.window_partition(x.double(), ws))
    yw = _randn((B * nW, ws, ws, C), 83, h)
    out = torch.empty_like(x)
    ops.window_unpartition(yw, None, out, B=B, H=H, W=W, C_=C, ws=ws)
    _exact("ea_window_unpartition", f"{H}x{W}", out, R.window_unpartition(yw.double(), B, H, W, ws))
    res = _randn((B, H, W, C), 84, h)
    ops.window_unpartition(yw, res, out, B=B, H=H, W=W, C_=C, ws=ws)
    ref = R.window_unpartition(yw.double(), B, H, W, ws) + res.double()
    _close("ea_window_unpartition", f"+residual {H}x{W}", out, ref, 0.5 * R.ulp(ref, h) + U * ref.abs())


def test_nhwc_to_nchw_f32_exact():
    h = _half()
    B, HW, C = 2, 1000, 72
    x = _randn((B, HW, C), 85, h)
    out = torch.full((B, C, HW), 7.0, device=DEV)
    ops.nhwc_to_nchw_f32(x, out, B=B, HW=HW, C_=C)
    _exact("ea_nhwc_to_nchw_f32", "1000x72", out, R.nhwc_to_nchw(x.double()))


@pytest.mark.parametrize("shape", [(1, 1024), (2, 64)], ids=["1024sq", "64sq_b2"])
def test_sam_patchify_exact(shape):
    h = _half()
    B, S = shape
    ps = 16
    img = _randn((B, 3, S, S), 86, scale=2.0)
    out = torch.empty(B * (S // ps) ** 2, 3 * ps * ps, device=DEV, dtype=h)
    ops.sam_patchify(img, out, B=B, Cin=3, H=S, W=S, ps=ps)
    _exact("ea_sam_patchify", f"{S}^2", out, R.sam_patchify(img.double(), ps))


@pytest.mark.parametrize("affine", [(0.5, 0.5, 0.0, 1.0), (1.25, -0.25, -1.0, 2.0)], ids=["decode", "other"])
def test_image_out_exact(affine):
    h = _half()
    scale, shift, lo, hi = affine
    B, HW, C, ldx = 2, 64 * 48, 3, 8
    x = _randn((B, HW, ldx), 87, h, scale=1.5)
    out = torch.full((B, C, HW), 7.0, device=DEV)
    ops.image_out(x, out, B=B, HW=HW, C_=C, ldx=ldx, scale=scale, shift=shift, lo=lo, hi=hi)
    _exact("ea_image_out", str(affine), out, R.image_out(x.double(), C, scale, shift, lo, hi))


def test_step_gather_exact():
    n_rows = 5
    shapes = [(16,), (2, 1280), (7,)]
    tables = [_randn((n_rows,) + s, 88 + i) for i, s in enumerate(shapes)]
    dsts = [torch.full(s, 7.0, device=DEV) for s in shapes]
    ctr = torch.zeros(1, device=DEV, dtype=torch.int32)
    for c in (0, 3, 4, 9):
        ctr.fill_(c)
        ops.step_gather(ctr, n_rows, tables, dsts)
        for k, (t, d) in enumerate(zip(tables, dsts)):
            _exact("ea_step_gather", f"table {k} counter {c}", d, t[min(c, n_rows - 1)].double())
    assert int(ctr.item()) == 9, "ea_step_gather changed the counter"


# ================================================ GEMM epilogue inputs =========================================
@pytest.mark.parametrize("variant", ["default", "splits1", "no_spin"])
@pytest.mark.parametrize("MNK", [(128, 1280, 1280), (8192, 320, 320)], ids=["zero_conv_8x8", "zero_conv_64x64"])
def test_gemm_row_scale(MNK, variant):
    """ControlNet zero-conv with a spatial conditioning-scale map: slot += 0.7 * rs[m] * (A W^T + b), in a slot of
    a wider buffer (ldo = 2N)."""
    h = _half()
    M, N, K = MNK
    a = _randn((M, K), 91, h)
    w = _randn((N, K), 92, h, scale=K ** -0.5)
    bias = _randn((N,), 93, scale=0.1)
    rs = torch.rand(M, generator=_gen(94), device=DEV) * 2.0
    rs[::7] = 0.0
    buf = _randn((M, 2 * N), 95, h)
    old = buf[:, N:].double()
    left = buf[:, :N].clone()
    kw = dict(M=M, bias=bias, out_scale=0.7, row_scale=rs, accumulate=True, ldo=2 * N)
    if variant == "splits1":
        kw["force_splits"] = 1
    if variant == "no_spin":
        with _concurrent_lane():
            ops.gemm(a, w, buf[:, N:], **kw)
    else:
        ops.gemm(a, w, buf[:, N:], **kw)
    _untouched("ea_gemm row_scale", "left half of the slot", buf[:, :N], left)
    ref, t, mag = R.gemm_epilogue(a.double(), w.double(), bias.double(), 0.7, rs.double(), old)
    bound = R.ulp(ref, h) + (K + 1) * U * mag + 3 * U * (t.abs() + old.abs())
    _close("ea_gemm row_scale", f"M={M} {variant}", buf[:, N:], ref, bound)


def test_gemm_out_f32_vae_logits():
    """VAE AttnBlock logits: q and k side by side in one [HW, 2C] buffer, fp32 output scaled by C^-0.5."""
    M, C = 4096, 512
    qk = _randn((M, 2 * C), 96, _half())
    s = torch.full((M, M), 7.0, device=DEV)
    ops.gemm(qk, qk[:, C:], out_f32=s, K=C, lda=2 * C, ldw=2 * C, out_scale=C ** -0.5)
    ref, t, mag = R.gemm_epilogue(qk[:, :C].double(), qk[:, C:].double(), None, C ** -0.5)
    _close("ea_gemm out_f32", "4096x4096x512", s, ref, (C + 1) * U * mag + U * ref.abs())


def test_gemm_out_f32_accumulate_ragged():
    M, N, K = 300, 72, 128
    a = _randn((M, K), 97, _half())
    w = _randn((N, K), 98, _half(), scale=K ** -0.5)
    bias = _randn((N,), 99, scale=0.1)
    s = _randn((M, N), 100)
    old = s.double()
    ops.gemm(a, w, out_f32=s, bias=bias, out_scale=0.5, accumulate=True)
    ref, t, mag = R.gemm_epilogue(a.double(), w.double(), bias.double(), 0.5, None, old)
    _close("ea_gemm out_f32", "300x72 accumulate", s, ref, (K + 1) * U * mag + 2 * U * (t.abs() + old.abs()))


# ================================================ argument validation ==========================================
def _rejects(status, fn):
    n0 = ops.launch_count()
    with pytest.raises(RuntimeError, match=rf"\({status}\)"):
        fn()
    torch.cuda.synchronize()
    assert ops.launch_count() == n0, "a rejected call launched a kernel"


def test_rejected_arguments():
    h = _half()
    SHAPE, ARG = -2, -1          # EA_ERR_SHAPE, EA_ERR_ARG
    # conv_in: Cin must be 4 or 8
    x5 = torch.zeros(1, 8, 8, 5, device=DEV, dtype=h)
    w5 = torch.zeros(3, 3, 5, 64, device=DEV)
    o = torch.zeros(1, 8, 8, 64, device=DEV, dtype=h)
    _rejects(SHAPE, lambda: ops.conv_in(x5, w5, None, o, B=1, H=8, W=8, Cin=5, Cout=64))
    # layernorm: C <= 2048
    xl = torch.zeros(4, 2056, device=DEV, dtype=h)
    gl = torch.ones(2056, device=DEV)
    _rejects(SHAPE, lambda: ops.layernorm(xl, gl, gl, torch.empty_like(xl), M=4, C_=2056))
    # small_linear: M <= 16
    xs = torch.zeros(17, 64, device=DEV)
    ws_ = torch.zeros(64, 64, device=DEV, dtype=h)
    _rejects(SHAPE, lambda: ops.small_linear(xs, ws_, None, torch.empty(17, 64, device=DEV), M=17, N=64, K=64))
    # groupnorm: more images than SMs (every CTA of an image must be resident), C not divisible by groups
    n_sm = torch.cuda.get_device_properties(DEV).multi_processor_count
    Bg = n_sm + 1
    xg = torch.zeros(Bg, 8, 64, device=DEV, dtype=h)
    gg = torch.ones(64, device=DEV)
    _rejects(SHAPE, lambda: ops.groupnorm(xg, gg, gg, torch.empty_like(xg), B=Bg, HW=8, C_=64, groups=32))
    xg = torch.zeros(2, 8, 72, device=DEV, dtype=h)
    gg = torch.ones(72, device=DEV)
    _rejects(SHAPE, lambda: ops.groupnorm(xg, gg, gg, torch.empty_like(xg), B=2, HW=8, C_=72, groups=32))
    # softmax_rows: cols % 4 == 0
    sm = torch.zeros(4, 8, device=DEV)
    _rejects(SHAPE, lambda: ops.softmax_rows(sm, torch.empty(4, 8, device=DEV, dtype=h), rows=4, cols=6,
                                             lds=8, ldp=8))
    # gemm: row_scale cannot be combined with GEGLU
    a = torch.zeros(128, 64, device=DEV, dtype=h)
    wg = torch.zeros(256, 64, device=DEV, dtype=h)
    rs = torch.ones(128, device=DEV)
    _rejects(ARG, lambda: ops.gemm(a, wg, torch.empty(128, 128, device=DEV, dtype=h), act=L.EA_ACT_GEGLU,
                                   row_scale=rs))
