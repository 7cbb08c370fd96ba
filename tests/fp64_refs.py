"""Float64 references of the library's non-GEMM operators (and the GEMM epilogue inputs row_scale / out_f32), written
from each operation's definition and independent of tests/cpu_ops.py and tools/gpu_probe_ops.py.

Every function takes the kernel's own inputs upcast to float64 (any device) and returns float64 results in the
kernel's layout (channels-last).  Reductions also return the sum of absolute products behind every output, which the
error bounds of tests/test_gpu_kernels_fp64.py are built from.  tests/test_kernel_refs_cpu.py checks these references
against torch.nn.functional and the schedulers on the CPU."""
import math

import numpy as np
import torch
import torch.nn.functional as F

U32 = 2.0 ** -24          # unit roundoff of fp32 (round to nearest)


def ulp(ref, dtype):
    """Spacing of `dtype` at |ref| (float64 tensor), floored at the dtype's smallest normal."""
    fi = torch.finfo(dtype)
    a = ref.abs().clamp_min(fi.tiny)
    _, e = torch.frexp(a)                      # a = m * 2**e, m in [0.5, 1)
    return torch.ldexp(torch.full_like(a, fi.eps), e - 1)


def silu(y):
    return y * torch.sigmoid(y)


def silu_eval_err(y):
    """Bound on the kernel's fp32 SiLU (ex2.approx + rcp.approx) at y, relative to |silu(y)|: the rounding of
    y * log2(e) is amplified by |y|, the two approximations add a few ulps."""
    return U32 * (8.0 + 2.0 * y.abs()) * silu(y).abs()


# ---- normalisations -------------------------------------------------------------------------------------------
def groupnorm(x, gammas, betas, groups, eps, silu_on):
    """x: [B, HW, C]; gammas / betas: one [C] vector per stacked network (B divisible by their count).
    Returns (y, pre, terms): y after affine (+ SiLU), the affine output before the SiLU, and the magnitudes
    (|x - mu| r + |mu| r + 1) |g| + |b| that an fp32 evaluation of g (x - mu) r + b is rounded against (the 1 stands
    for the rounding of the statistics themselves, in units of the group's standard deviation)."""
    B, HW, C = x.shape
    n = len(gammas)
    xc = x.permute(0, 2, 1)                                      # [B, C, HW]
    y = F.group_norm(xc, groups, eps=eps).permute(0, 2, 1)       # normalised, no affine
    xg = x.reshape(B, HW, groups, C // groups)
    mu = xg.mean(dim=(1, 3), keepdim=True)
    var = xg.var(dim=(1, 3), correction=0, keepdim=True)
    r = (var + eps).rsqrt()
    amu = (mu.abs() * r).expand_as(xg).reshape(B, HW, C)
    g = torch.stack(gammas).repeat_interleave(B // n, dim=0)[:, None, :]
    b = torch.stack(betas).repeat_interleave(B // n, dim=0)[:, None, :]
    out = y * g + b
    terms = (y.abs() + amu + 1.0) * g.abs() + b.abs()
    return (silu(out) if silu_on else out), out, terms


def layernorm(x, gamma, beta, eps):
    """x: [M, C].  Returns (y, terms) like groupnorm (no SiLU)."""
    y = F.layer_norm(x, (x.shape[-1],), gamma, beta, eps)
    mu = x.mean(dim=-1, keepdim=True)
    r = (x.var(dim=-1, correction=0, keepdim=True) + eps).rsqrt()
    xh = (x - mu) * r
    terms = (xh.abs() + mu.abs() * r + 1.0) * gamma.abs() + beta.abs()
    return y, terms


# ---- convolutions ---------------------------------------------------------------------------------------------
def conv_nhwc(x, w, bias, stride=1):
    """x: [B, H, W, Cin]; w: [k, k, Cin, Cout] (the library's layout); pad k // 2.  Returns (out NHWC, sum of |x w|
    + |bias|)."""
    k = w.shape[0]
    wt = w.permute(3, 2, 0, 1)
    xc = x.permute(0, 3, 1, 2)
    out = F.conv2d(xc, wt, bias, stride=stride, padding=k // 2).permute(0, 2, 3, 1)
    mag = F.conv2d(xc.abs(), wt.abs(), None if bias is None else bias.abs(), stride=stride,
                   padding=k // 2).permute(0, 2, 3, 1)
    return out, mag


def out_conv(xn, w, bias):
    """The out conv of ea_out_cfg_ddim: xn [2N, H, W, C], w [4, 3, 3, C] -> eps [2N, H, W, 4] and its |.| sums."""
    return conv_nhwc(xn, w.permute(1, 2, 3, 0), bias)


# ---- small linears / time embedding ---------------------------------------------------------------------------
def small_linear(x, w, bias, silu_in, silu_out):
    """y = act_out(W act_in(x) + b): x [M, K], w [N, K].  Returns (y, pre-activation, |.| sums)."""
    xi = silu(x) if silu_in else x
    pre = xi @ w.T
    mag = xi.abs() @ w.abs().T
    if bias is not None:
        pre = pre + bias
        mag = mag + bias.abs()
    return (silu(pre) if silu_out else pre), pre, mag


def timestep_embedding(t, dim, max_period=10000):
    """ldm/modules/diffusionmodules/util.py:154-174 (dim even): [cos(t f) | sin(t f)], f_i = max_period^(-i/half).
    Returns (emb, the argument t f, the exponent ln(max_period) i / half)."""
    half = dim // 2
    xf = math.log(max_period) * torch.arange(half, dtype=torch.float64, device=t.device) / half
    arg = t[:, None] * torch.exp(-xf)[None]
    return torch.cat([torch.cos(arg), torch.sin(arg)], dim=-1), arg, xf


# ---- SAM / VAE helpers ----------------------------------------------------------------------------------------
def sam_relpos(q, Rh, Rw):
    """q: [B, S*S, heads, d]; Rh, Rw: [S, S, d].  rel_h[b*heads + h, qh*S + qw, k] = sum_c q[b, (qh, qw), h, c]
    Rh[qh, k, c], rel_w likewise with Rw[qw].  Returns (rel_h, rel_w, |.| sums of each)."""
    B, SS, heads, d = q.shape
    S = Rh.shape[0]
    qq = q.reshape(B, S, S, heads, d)                  # x = qh, y = qw

    def rel(spec, qv, R):
        return torch.einsum(spec, qv, R).reshape(B * heads, SS, S)

    hs, ws = "bxyhc,xkc->bhxyk", "bxyhc,ykc->bhxyk"
    return (rel(hs, qq, Rh), rel(ws, qq, Rw), rel(hs, qq.abs(), Rh.abs()), rel(ws, qq.abs(), Rw.abs()))


def softmax_rows(s):
    return torch.softmax(s, dim=-1)


def upsample2x(x):
    """Nearest x2 on NHWC."""
    return x.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2)


def window_partition(x, ws):
    """[B, H, W, C] -> [B * nWh * nWw, ws, ws, C], zero padded at the bottom / right."""
    B, H, W, C = x.shape
    ph, pw = (-H) % ws, (-W) % ws
    xp = F.pad(x, (0, 0, 0, pw, 0, ph))
    Hp, Wp = H + ph, W + pw
    xw = xp.reshape(B, Hp // ws, ws, Wp // ws, ws, C).permute(0, 1, 3, 2, 4, 5)
    return xw.reshape(-1, ws, ws, C)


def window_unpartition(xw, B, H, W, ws):
    C = xw.shape[-1]
    Hp, Wp = H + (-H) % ws, W + (-W) % ws
    x = xw.reshape(B, Hp // ws, Wp // ws, ws, ws, C).permute(0, 1, 3, 2, 4, 5).reshape(B, Hp, Wp, C)
    return x[:, :H, :W]


def sam_patchify(img, ps):
    """fp32 NCHW [B, Cin, H, W] -> [B * gh * gw, Cin * ps * ps] with K index (c * ps + kh) * ps + kw."""
    B, Cin, H, W = img.shape
    p = img.reshape(B, Cin, H // ps, ps, W // ps, ps).permute(0, 2, 4, 1, 3, 5)
    return p.reshape(B * (H // ps) * (W // ps), Cin * ps * ps)


def nhwc_to_nchw(x):
    """[B, HW, C] -> [B, C, HW]."""
    return x.permute(0, 2, 1)


def image_out(x, C, scale, shift, lo, hi):
    """x: [B, HW, ldx] (first C channels used) -> [B, C, HW] = clamp(x * scale + shift, lo, hi)."""
    return (x[..., :C] * scale + shift).clamp(lo, hi).permute(0, 2, 1)


# ---- GEMM epilogue ---------------------------------------------------------------------------------------------
def gemm_epilogue(a, w, bias=None, out_scale=1.0, row_scale=None, old=None):
    """out = (A W^T + bias) * out_scale * row_scale[m] (+ old).  Returns (out, the scaled product term, the scaled
    |.| sums)."""
    acc = a @ w.T
    mag = a.abs() @ w.abs().T
    if bias is not None:
        acc = acc + bias
        mag = mag + bias.abs()
    s = torch.full((a.shape[0], 1), float(out_scale), dtype=a.dtype, device=a.device)
    if row_scale is not None:
        s = s * row_scale[:, None]
    t = acc * s
    return (t if old is None else t + old), t, mag * s.abs()


# ---- fused CFG + scheduler update ------------------------------------------------------------------------------
def cfg(eu, ec, g):
    return eu + g * (ec - eu)


def ddim_update(xt, e, coef):
    """cldm/ddim_hacked.py:215-230 (eta = 0) with coef = (sqrt a_t, sqrt(1-a_t), sqrt a_prev, sqrt(1-a_prev))."""
    sa, s1a, sap, s1ap = coef[:4]
    x0 = (xt - s1a * e) / sa
    return sap * x0 + s1ap * e, x0


def blend(xp, known, noise, mask, k_init, k_noise, on):
    """utils/stable_diffusion_controlnet_inpaint.py:1647-1656: keep the (re-noised) known latents where mask = 1."""
    kn = known if noise is None else k_init * known + k_noise * noise
    mk = mask[..., None] * on
    return kn * mk + xp * (1.0 - mk), kn


class ErrLin:
    """Forward error bound of fp32 linear combinations: y = sum c_i v_i evaluated in fp32 with fp32-rounded
    coefficients satisfies |y_fp32 - y| <= sum |c_i| err_i + (n + 2) u sum |c_i v_i|: one rounding per product and
    per addition, one per coefficient, and one more for a coefficient the kernel forms as a quotient of two
    (x0 = (x - sigma e) / alpha).  Values are carried in float64."""

    @staticmethod
    def lin(terms):
        val = sum(c * v for c, v, _ in terms)
        err = sum(abs(c) * e for c, _, e in terms) + (len(terms) + 2) * U32 * sum(abs(c) * v.abs() for c, v, _ in terms)
        return val, err


def blend_err(xp, known, noise, mask, cf):
    """The kernel's inpaint blend of (value, error bound) xp with its fp32 rounding: with `noise` the kept region is
    cf[4] known + cf[5] noise and the mask is gated by cf[6]."""
    z = torch.zeros_like(known)
    mk = mask[..., None] * (cf[6] if noise is not None else 1.0)
    kn = ErrLin.lin([(cf[4], known, z), (cf[5], noise, z)]) if noise is not None else (known, z)
    val = kn[0] * mk + xp[0] * (1.0 - mk)
    err = kn[1] * mk + xp[1] * (1.0 - mk) + 3 * U32 * (kn[0].abs() * mk + xp[0].abs() * (1.0 - mk) + val.abs())
    return val, err


def unipc_fused(rows_coef, eps_list, x, guidance, known=None, noise=None, mask=None):
    """The coefficient-row recurrence ea_out_cfg_ddim runs in mode 1 (include/editanything_b200.h), in float64 with a
    running fp32 error bound.  rows_coef: per step the 16 fp32 coef values (as tensors or floats); eps_list: per step
    (eu, ec).  Returns the list of (latents, error bound) after every step."""
    z = torch.zeros_like(x)
    m1, m2, last = (z, z), (z, z), (z, z)        # (value, error bound)
    xt = (x, z)
    out = []
    for cf, (eu, ec) in zip(rows_coef, eps_list):
        cf = [float(v) for v in cf]
        e = cfg(eu, ec, guidance)
        e_err = 3 * U32 * (eu.abs() + abs(guidance) * (ec.abs() + eu.abs()))
        x0 = ErrLin.lin([(1.0 / cf[0], xt[0], xt[1]), (-cf[1] / cf[0], e, e_err)])
        xc = ErrLin.lin([(cf[8], xt[0], xt[1]), (cf[9], last[0], last[1]), (cf[10], m1[0], m1[1]),
                         (cf[11], m2[0], m2[1]), (cf[12], x0[0], x0[1])])
        xp = ErrLin.lin([(cf[13], xc[0], xc[1]), (cf[14], x0[0], x0[1]), (cf[15], m1[0], m1[1])])
        m2, m1, last = m1, x0, xc
        if known is not None:
            xp = blend_err(xp, known, noise, mask, cf)
        xt = xp
        out.append(xp)
    return out


def scheduler_trajectory(sched, eps_list, x, guidance, blend_rows=None, known=None, noise=None, mask=None):
    """The reference loop: latents = scheduler.step(cfg(eps), t, latents).prev_sample (+ inpaint blend), float64."""
    lat = x
    out = []
    for i, (t, (eu, ec)) in enumerate(zip(sched.timesteps.tolist(), eps_list)):
        lat = sched.step(cfg(eu, ec, guidance), t, lat).prev_sample
        if known is not None:
            ki, kn_, on = blend_rows[i] if blend_rows is not None else (1.0, 0.0, 1.0)
            lat, _ = blend(lat, known, noise, mask, ki, kn_, on)
        out.append(lat)
    return out


def unipc_coef_rows(sched, blend_rows=None):
    """Per step the 16-float coef row of ea_out_cfg_ddim mode 1 from UniPCMultistepScheduler.coefficient_rows()."""
    rows = []
    for i, r in enumerate(sched.coefficient_rows()):
        ki, kn, on = blend_rows[i] if blend_rows is not None else (1.0, 0.0, 1.0)
        rows.append([r["alpha"], r["sigma"], 0.0, 0.0, ki, kn, on, 1.0,
                     r["kx"], r["kl"], r["k1"], r["k2"], r["k0"], r["px"], r["p0"], r["p1"]])
    return np.asarray(rows, dtype=np.float32)
