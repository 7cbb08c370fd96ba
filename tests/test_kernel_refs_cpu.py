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
