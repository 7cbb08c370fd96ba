"""The float64 references of tests/test_gpu_kernels_fp64.py (tests/fp64_refs.py), checked on the CPU against
torch.nn.functional / torch.nn modules, explicit loops and the schedulers, so the oracle is verified without a GPU."""
import math

import numpy as np
import torch
import torch.nn.functional as F

from editanything_b200.pipeline import DDIMScheduler
from editanything_b200.schedulers import UniPCMultistepScheduler
from tests import fp64_refs as R


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _rn(*shape, seed=0, dtype=torch.float64):
    return torch.randn(*shape, generator=_g(seed), dtype=dtype)


def test_ulp():
    h = torch.float16
    x = torch.tensor([1.0, 1.5, 0.75, -3.0, 0.0, 1e-7, 65504.0], dtype=torch.float64)
    want = (torch.nextafter(x.abs().to(h), torch.tensor(math.inf, dtype=h)).double() - x.abs().to(h).double())
    want[4] = want[5] = torch.finfo(h).tiny * torch.finfo(h).eps     # floored at the smallest normal
    want[6] = 32.0                                                   # spacing of the top binade
    assert torch.equal(R.ulp(x, h), want)
    assert float(R.ulp(torch.tensor([1.0], dtype=torch.float64), torch.bfloat16)) == 2.0 ** -7


def test_groupnorm_matches_nn_groupnorm():
    B, HW, C, G = 4, 12, 48, 8
    x = _rn(B, HW, C, seed=1) * 2 + 3
    gam = [_rn(C, seed=2), _rn(C, seed=3)]
    bet = [_rn(C, seed=4), _rn(C, seed=5)]
    y, pre, terms = R.groupnorm(x, gam, bet, G, 1e-6, True)
    for net in range(2):
        m = torch.nn.GroupNorm(G, C, eps=1e-6).double()
        with torch.no_grad():
            m.weight.copy_(gam[net])
            m.bias.copy_(bet[net])
        xs = x[2 * net:2 * net + 2].permute(0, 2, 1)
        want = m(xs).permute(0, 2, 1)
        assert torch.allclose(pre[2 * net:2 * net + 2], want, rtol=1e-12, atol=1e-12)
        assert torch.allclose(y[2 * net:2 * net + 2], F.silu(want), rtol=1e-12, atol=1e-12)
    assert (terms >= bet[0].abs().min()).all()


def test_layernorm_matches_nn_layernorm():
    x = _rn(7, 72, seed=6) + 10
    g, b = _rn(72, seed=7), _rn(72, seed=8)
    y, terms = R.layernorm(x, g, b, 1e-5)
    mu = x.mean(-1, keepdim=True)
    want = (x - mu) / torch.sqrt(((x - mu) ** 2).mean(-1, keepdim=True) + 1e-5) * g + b
    assert torch.allclose(y, want, rtol=1e-12, atol=1e-12)
    assert (terms > 0).all()


def _conv_loops(x, w, bias, stride):
    B, H, W, Cin = x.shape
    k, Cout = w.shape[0], w.shape[3]
    pad = k // 2
    Ho, Wo = -(-H // stride), -(-W // stride)
    out = np.zeros((B, Ho, Wo, Cout))
    xn, wn = x.numpy(), w.numpy()
    for b in range(B):
        for ho in range(Ho):
            for wo in range(Wo):
                acc = np.zeros(Cout) if bias is None else bias.numpy().copy()
                for kh in range(k):
                    for kw in range(k):
                        hi, wi = ho * stride + kh - pad, wo * stride + kw - pad
                        if 0 <= hi < H and 0 <= wi < W:
                            acc += xn[b, hi, wi] @ wn[kh, kw]
                out[b, ho, wo] = acc
    return torch.from_numpy(out)


def test_conv_matches_loops():
    for (H, W, Cin, Cout, k, s, bias) in [(5, 7, 3, 4, 3, 1, True), (7, 5, 4, 6, 3, 2, False), (5, 3, 2, 3, 1, 2, True)]:
        x = _rn(2, H, W, Cin, seed=H)
        w = _rn(k, k, Cin, Cout, seed=W)
        b = _rn(Cout, seed=9) if bias else None
        out, mag = R.conv_nhwc(x, w, b, s)
        assert torch.allclose(out, _conv_loops(x, w, b, s), rtol=1e-12, atol=1e-12)
        assert torch.allclose(mag, _conv_loops(x.abs(), w.abs(), None if b is None else b.abs(), s), rtol=1e-12)
    xn = _rn(2, 4, 5, 16, seed=10)
    w = _rn(4, 3, 3, 16, seed=11)
    b = _rn(4, seed=12)
    eps, _ = R.out_conv(xn, w, b)
    want = F.conv2d(xn.permute(0, 3, 1, 2), w.permute(0, 3, 1, 2), b, padding=1).permute(0, 2, 3, 1)
    assert torch.allclose(eps, want, rtol=1e-12, atol=1e-12)


def _im2col(x, mode):
    """[B, Hin, Win, C] -> [B, H, W, 9 C] in ea_gemm's K order (kh * 3 + kw) * C + c, by index arithmetic: tap (kh, kw)
    of output pixel (oh, ow) reads input pixel (s oh + kh - p, s ow + kw - p), zero outside the input."""
    B, Hin, Win, C = x.shape
    s, p = (1, 1) if mode == "s1" else (2, 1) if mode == "s2" else (2, 0)
    H, W = Hin // s, Win // s
    cols = []
    for kh in range(3):
        for kw in range(3):
            ih, iw = s * torch.arange(H) + kh - p, s * torch.arange(W) + kw - p
            ok = ((ih >= 0) & (ih < Hin))[:, None] & ((iw >= 0) & (iw < Win))[None, :]
            v = x[:, ih.clamp(0, Hin - 1)][:, :, iw.clamp(0, Win - 1)]
            cols.append(v * ok[None, :, :, None])
    return torch.cat(cols, dim=-1)


def test_conv_gemm_matches_im2col():
    """fp64_refs.conv_gemm (F.conv2d / F.pad) against the GEMM view of each mode, with and without the folded skip."""
    for mode, (Hin, Win), extra in [("s1", (5, 7), 0), ("s1", (4, 6), 3), ("s2", (6, 10), 0), ("s2a", (8, 6), 0),
                                    ("s2a", (10, 4), 0)]:
        x = _rn(2, Hin, Win, 4, seed=Hin + Win)
        s = 1 if mode == "s1" else 2
        w = _rn(5, 36 + extra, seed=Win)
        xe = _rn(2, Hin // s, Win // s, extra, seed=3) if extra else None
        cols = _im2col(x, mode)
        want, want_mag = cols @ w[:, :36].T, cols.abs() @ w[:, :36].abs().T
        if extra:
            want, want_mag = want + xe @ w[:, 36:].T, want_mag + xe.abs() @ w[:, 36:].abs().T
        out, mag = R.conv_gemm(x, w, mode, xe)
        assert out.shape == (2, Hin // s, Win // s, 5)
        assert torch.allclose(out, want, rtol=1e-12, atol=1e-12), mode
        assert torch.allclose(mag, want_mag, rtol=1e-12, atol=1e-12), mode


def test_small_linear_and_timestep_embedding():
    x, w, b = _rn(3, 16, seed=13), _rn(5, 16, seed=14), _rn(5, seed=15)
    y, pre, mag = R.small_linear(x, w, b, True, True)
    assert torch.allclose(y, F.silu(F.linear(F.silu(x), w, b)), rtol=1e-12, atol=1e-12)
    assert torch.allclose(mag, F.silu(x).abs() @ w.abs().T + b.abs())
    # ldm/modules/diffusionmodules/util.py:154-174, evaluated in fp32 as the reference runs it
    t = torch.tensor([0.0, 1.0, 0.5, 500.0, 981.0, 999.0])
    for dim in (320, 256):
        half = dim // 2
        freqs = torch.exp(-math.log(10000) * torch.arange(start=0, end=half, dtype=torch.float32) / half)
        args = t[:, None].float() * freqs[None]
        want = torch.cat([torch.cos(args), torch.sin(args)], dim=-1)
        got, arg, xf = R.timestep_embedding(t.double(), dim)
        assert torch.allclose(got.float(), want, atol=1e-3)
        assert torch.allclose(arg.float(), args, rtol=1e-5)


def test_sam_relpos_matches_loops():
    B, S, heads, d = 2, 3, 2, 4
    q = _rn(B, S * S, heads, d, seed=16)
    Rh, Rw = _rn(S, S, d, seed=17), _rn(S, S, d, seed=18)
    rh, rw, mh, mw = R.sam_relpos(q, Rh, Rw)
    for b in range(B):
        for h in range(heads):
            for qh in range(S):
                for qw in range(S):
                    for k in range(S):
                        qv = q[b, qh * S + qw, h]
                        assert abs(float(rh[b * heads + h, qh * S + qw, k] - qv @ Rh[qh, k])) < 1e-12
                        assert abs(float(rw[b * heads + h, qh * S + qw, k] - qv @ Rw[qw, k])) < 1e-12
                        assert abs(float(mw[b * heads + h, qh * S + qw, k] - qv.abs() @ Rw[qw, k].abs())) < 1e-12


def test_layout_helpers():
    x = _rn(2, 5, 7, 8, seed=19)
    assert torch.equal(R.upsample2x(x), F.interpolate(x.permute(0, 3, 1, 2), scale_factor=2.0,
                                                      mode="nearest").permute(0, 2, 3, 1))
    xw = R.window_partition(x, 3)
    assert xw.shape == (2 * 2 * 3, 3, 3, 8)
    assert torch.equal(xw[1, 0, 0], x[0, 0, 3]) and torch.equal(xw[5, 2, 2], torch.zeros(8, dtype=x.dtype))
    assert torch.equal(R.window_unpartition(xw, 2, 5, 7, 3), x)
    img = _rn(2, 3, 32, 16, seed=20)
    p = R.sam_patchify(img, 16)
    want = F.unfold(img, 16, stride=16).permute(0, 2, 1).reshape(-1, 3 * 256)    # (c, kh, kw) order per patch
    assert torch.equal(p, want)
    y = _rn(2, 10, 6, seed=21)
    assert torch.equal(R.nhwc_to_nchw(y), y.permute(0, 2, 1))
    assert torch.equal(R.image_out(y, 3, 0.5, 0.5, 0.0, 1.0), (y[..., :3] / 2 + 0.5).clamp(0, 1).permute(0, 2, 1))
    s = _rn(4, 12, seed=22) * 5
    assert torch.allclose(R.softmax_rows(s), F.softmax(s.float(), -1).double(), atol=1e-7)


def test_gemm_epilogue():
    a, w, b = _rn(6, 8, seed=23), _rn(5, 8, seed=24), _rn(5, seed=25)
    rs, old = _rn(6, seed=26).abs(), _rn(6, 5, seed=27)
    out, t, mag = R.gemm_epilogue(a, w, b, 0.7, rs, old)
    assert torch.allclose(out, F.linear(a, w, b) * 0.7 * rs[:, None] + old, rtol=1e-12, atol=1e-12)
    assert torch.allclose(mag, (a.abs() @ w.abs().T + b.abs()) * 0.7 * rs[:, None])


def test_gelu_matches_functional():
    y = torch.cat([torch.linspace(-12, 12, 4001, dtype=torch.float64), _rn(1000, seed=30) * 4])
    got = R.gelu(y)
    # F.gelu forms 1 + erf, which cancels in the negative tail: compare it where that costs < 1e-12 relative
    body = y > -3
    assert torch.allclose(got[body], F.gelu(y)[body], rtol=1e-12, atol=0)
    want = torch.tensor([0.5 * v * math.erfc(-v / math.sqrt(2.0)) for v in y.tolist()], dtype=torch.float64)
    assert torch.allclose(got, want, rtol=1e-13, atol=0)


def test_geglu_matches_interleave_loop():
    M, N = 3, 384
    y = _rn(M, N, seed=31) * 3
    want = torch.empty(M, N // 2, dtype=torch.float64)
    for m in range(M):
        for blk in range(N // 128):
            for i in range(64):
                x, g = float(y[m, blk * 128 + i]), float(y[m, blk * 128 + 64 + i])
                want[m, blk * 64 + i] = x * 0.5 * g * math.erfc(-g / math.sqrt(2.0))
    assert torch.allclose(R.geglu(y), want, rtol=1e-13, atol=1e-300)


def _gelu_erf_f32(y, pert):
    """The kernel's gelu_erf_f (ea_common.cuh) in fp32 numpy, with relative error `pert` applied to the results of
    rcp.approx and ex2.approx (fma as an fp32 multiply-add in float64, rounded once)."""
    f = np.float32

    def fma(a, b, c):
        return (a.astype(np.float64) * b + c).astype(np.float32)

    z = (np.abs(y) * f(0.70710678118654752)).astype(np.float32)
    t = (f(1) / fma(f(0.3275911), z, f(1))).astype(np.float32) * f(pert)
    poly = fma(f(1.061405429), t, f(-1.453152027))
    for c in (1.421413741, -0.284496736, 0.254829592):
        poly = fma(poly, t, f(c))
    arg = ((z * z).astype(np.float32) * f(-1.4426950408889634)).astype(np.float32)
    ex = np.exp2(arg.astype(np.float64)).astype(np.float32) * f(pert)
    e = fma((-poly * t).astype(np.float32), ex, f(1))
    return (f(0.5) * y * (f(1) + np.copysign(e, y)).astype(np.float32)).astype(np.float32)


def test_gelu_eval_err_bounds_fp32_emulation():
    """gelu_eval_err bounds the kernel's formula evaluated in fp32, with +-2^-22 on the two .approx results, over a
    dense grid of [-12, 12] and log-spaced points down to 1e-8 on both sides."""
    y = np.concatenate([np.linspace(-12, 12, 400001), -np.logspace(-8, 1.1, 4001),
                        np.logspace(-8, 1.1, 4001)]).astype(np.float32)
    yd = torch.from_numpy(y.astype(np.float64))
    ref, bound = R.gelu(yd), R.gelu_eval_err(yd)
    worst = 0.0
    for pert in (1 - 2.0 ** -22, 1.0, 1 + 2.0 ** -22):
        got = torch.from_numpy(_gelu_erf_f32(y, pert).astype(np.float64))
        err = (got - ref).abs()
        ratio = torch.where(err == 0, torch.zeros_like(err), err / bound)
        assert bool((err <= bound).all()), float(ratio.max())
        worst = max(worst, float(ratio.max()))
    assert worst > 0.05        # the bound is not vacuous


def test_ddim_update_matches_ddim_scheduler():
    s = DDIMScheduler()
    s.set_timesteps(20)
    t = int(s.timesteps[3])
    a, ap = s.coefficients(t)
    x, e = _rn(2, 4, 4, 4, seed=28), _rn(2, 4, 4, 4, seed=29)
    got, _ = R.ddim_update(x, e, [math.sqrt(a), math.sqrt(1 - a), math.sqrt(ap), math.sqrt(1 - ap)])
    assert torch.allclose(got, s.step(e, t, x).prev_sample, rtol=1e-12, atol=1e-12)


def _unipc_setup(blend):
    sched = UniPCMultistepScheduler.from_config(DDIMScheduler().config, solver_order=2)
    sched.set_timesteps(20)
    ts = sched.timesteps.tolist()
    blend_rows = None
    if blend:
        nxt = ts[1:] + [0]
        blend_rows = [(float(sched.alpha_t[t]), float(sched.sigma_t[t]), float(i % 3 != 1)) for i, t in enumerate(nxt)]
    rows = R.unipc_coef_rows(sched, blend_rows)
    shape = (2, 3, 5, 4)
    eps = [(_rn(*shape, seed=40 + 2 * i), _rn(*shape, seed=41 + 2 * i)) for i in range(len(ts))]
    kw = {}
    if blend:
        kw = dict(known=_rn(*shape, seed=90), noise=_rn(*shape, seed=91),
                  mask=(torch.rand(shape[:3], generator=_g(92)) < 0.5).double())
        blend_rows = [(float(r[4]), float(r[5]), float(r[6])) for r in rows]
    return sched, rows, eps, _rn(*shape, seed=93), blend_rows, kw


def test_unipc_recurrence_matches_scheduler_step():
    """The coefficient-row recurrence (the fused kernel's mode 1) reproduces UniPCMultistepScheduler.step() with and
    without the inpaint blend, and its fp32 error bound holds for an fp32 evaluation of the same recurrence."""
    for blend in (False, True):
        sched, rows, eps, x, blend_rows, kw = _unipc_setup(blend)
        ref = R.scheduler_trajectory(sched, eps, x, 7.5, blend_rows, **kw)
        fused = R.unipc_fused(rows, eps, x, 7.5, **kw)
        # the same recurrence in fp32, operation by operation as the kernel evaluates it
        f = lambda v: v.float()
        xt, m1, m2, last = f(x), torch.zeros_like(f(x)), torch.zeros_like(f(x)), torch.zeros_like(f(x))
        r32 = torch.tensor(rows, dtype=torch.float32)
        for i, (r, (val, err)) in enumerate(zip(ref, fused)):
            assert ((val - r).abs() <= err).all(), (blend, i)     # differ by the fp32 rounding of the coefficients
            assert float(err.max()) < 1e-4 * (1.0 + float(r.abs().max()))      # not vacuous
            c = r32[i]
            eu, ec = f(eps[i][0]), f(eps[i][1])
            e = eu + 7.5 * (ec - eu)
            x0 = (xt - c[1] * e) / c[0]
            xc = c[8] * xt + c[9] * last + c[10] * m1 + c[11] * m2 + c[12] * x0
            xp = c[13] * xc + c[14] * x0 + c[15] * m1
            m2, m1, last = m1, x0, xc
            if blend:
                mk = f(kw["mask"])[..., None] * c[6]
                kn = c[4] * f(kw["known"]) + c[5] * f(kw["noise"])
                xp = kn * mk + xp * (1.0 - mk)
            xt = xp
            assert ((xt.double() - r).abs() <= err).all(), (blend, i)
