"""Float64 references of the library's non-GEMM operators (and the GEMM epilogue: activations, row_scale, out_f32), written
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


def gelu(y):
    """Exact-erf GELU, F.gelu's default: y / 2 (1 + erf(y / sqrt 2)), written as y / 2 erfc(-y / sqrt 2) so that
    the negative tail (fp16 subnormal outputs) keeps full relative precision."""
    return 0.5 * y * torch.erfc(-y * math.sqrt(0.5))


def gelu_eval_err(y):
    """Bound on the kernel's fp32 gelu_erf_f at y: erf from Abramowitz & Stegun 7.1.26 (stated |error| < 1.5e-7)
    scaled by |y| / 2, 32 fp32 ulps of |y| / 2 for evaluating it (ex2.approx, rcp.approx, the polynomial), and 8 ulps
    of the result."""
    return 0.5 * y.abs() * (1.5e-7 + 32.0 * U32) + 8.0 * U32 * gelu(y).abs()


def geglu_split(y):
    """[M, N] pre-activations in the weight layout nets packs for GEGLU (per 128 columns: 64 value | 64 gate) ->
    (value, gate), each [M, N / 2] in output column order."""
    M, N = y.shape
    v = y.reshape(M, N // 128, 2, 64)
    return v[:, :, 0].reshape(M, N // 2), v[:, :, 1].reshape(M, N // 2)


def geglu(y):
    """value * gelu(gate) (ldm/modules/attention.py:54-56) of pre-activations in the packed layout."""
    x, g = geglu_split(y)
    return x * gelu(g)


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


def gn_geometry(B, HW, C, groups, n_sm):
    """ea_groupnorm's launch geometry (ea_pointwise.cu, ea_groupnorm) as (chunks, ppc, lanes, parts): `chunks` CTAs
    per image of `ppc` pixels each, `lanes` pixel lanes per CTA (thread = lane x 8-channel vector), and the `parts`
    threads per statistic that sum the image's per-CTA partials."""
    chunks = max(1, min(n_sm // B, HW))
    ppc = -(-HW // chunks)
    chunks = -(-HW // ppc)
    nvec = C // 8
    threads = min(512, -(-((512 // nvec) * nvec) // 32) * 32)
    lanes = threads // nvec
    parts = max(1, min(threads // (2 * groups), lanes * (C // groups)))
    return chunks, ppc, lanes, parts


def _chain(v, dim):
    """A serial fp32 sum along `dim`, in float64: (sum of |partial sums|, the total).  The rounding error of the
    recursive sum is at most u times the sum of its partial sums' magnitudes (Higham, Accuracy and Stability of
    Numerical Algorithms, 2nd ed., (4.3)); zero padding at the end of a chain only adds to that sum."""
    cs = v.cumsum(dim)
    return cs.abs().sum(dim), cs.select(dim, -1)


def gn_cta_sums(d, lanes, groups):
    """One CTA's part of ea_groupnorm's statistics.  d: [n, C] float64, the CTA's pixels minus each channel's shift
    k_g.  The kernel sums d and d^2 in this order: thread (lane l, channel c) adds pixels l, l + lanes, ...; then one
    thread per (group, statistic) adds the lanes x cpg thread partials, lane-major.  Returns
    [2, groups] (the CTA totals, the sum of |partial sums| over both stages) for (sum d, sum d^2)."""
    n, C = d.shape
    cpg = C // groups
    T = -(-n // lanes)
    tot, run = [], []
    for v in (d, d * d):
        r1, t1 = _chain(torch.nn.functional.pad(v, (0, 0, 0, T * lanes - n)).reshape(T, lanes, C), 0)
        r2, t2 = _chain(t1.reshape(lanes, groups, cpg).permute(1, 0, 2).reshape(groups, lanes * cpg), 1)
        tot.append(t2)
        run.append(r1.reshape(lanes, groups, cpg).sum(dim=(0, 2)) + r2)
    return torch.stack(tot), torch.stack(run)


def gn_cross_cta(totals, parts):
    """The kernel's sum of one image's per-CTA totals [chunks, 2, groups]: thread pidx of each statistic adds CTAs
    pidx, pidx + parts, ... in order, then one thread adds the parts in order.  Returns the sum of |partial sums|
    [2, groups]."""
    chunks = totals.shape[0]
    rows = -(-chunks // parts)
    t = torch.nn.functional.pad(totals, (0, 0, 0, 0, 0, rows * parts - chunks)).reshape(rows, parts, *totals.shape[1:])
    r1, t1 = _chain(t, 0)
    r2, _ = _chain(t1, 0)
    return r1.sum(0) + r2


def gn_stats_err(run, abs_sum, sq_sum, n, mean_dev, var, eps):
    """Bounds on ea_groupnorm's fp32 statistics per (image, group) from their summation order: `run` [2, ...] the sum
    of |partial sums| of sum d and sum d^2 over every stage (gn_cta_sums, gn_cross_cta), abs_sum / sq_sum the sums of
    |d| and d^2 (the rounding of d = x - k and of d^2), n the pixels x channels of the group, mean_dev the mean of d,
    var the group's variance.  The sums are off by dS1 = u (run_1 + sum |d|) and dS2 = u (run_2 + 3 sum d^2) (x1.01 for
    the second-order terms); the kernel's dm = S1 inv_n (3 u) gives the mean's bound, and q inv_n - dm^2 the
    variance's: dS2 / n + 2 |dm| dS1 / n + 4 u E[d^2] + 8 u dm^2.  Returns (bound on the mean, relative bound on
    rstd = (var + eps)^-1/2: half the variance's relative error plus 2 u)."""
    dS1 = 1.01 * U32 * (run[0] + abs_sum)
    dS2 = 1.01 * U32 * (run[1] + 3 * sq_sum)
    m = mean_dev.abs()
    d_mean = dS1 / n + 3 * U32 * m
    d_var = dS2 / n + 2 * m * dS1 / n + 4 * U32 * sq_sum / n + 8 * U32 * m * m
    return d_mean, 0.5 * d_var / (var + eps) + 2 * U32


def gn_stats_bound(x, groups, eps, n_sm):
    """gn_stats_err for a whole [B, HW, C] float64 input (the kernel's fp16 values): per (image, group) the bound on
    the mean, the relative bound on rstd, and rstd itself, each [B, groups]."""
    B, HW, C = x.shape
    cpg = C // groups
    chunks, ppc, lanes, parts = gn_geometry(B, HW, C, groups, n_sm)
    xg = x.reshape(B, HW, groups, cpg)
    k = xg[:, 0, :, 0]
    d_mean, d_rstd, r = [], [], []
    for b in range(B):
        kc = k[b].repeat_interleave(cpg)
        cta = [gn_cta_sums(x[b, c * ppc:(c + 1) * ppc] - kc, lanes, groups) for c in range(chunks)]
        run = sum(r_ for _, r_ in cta) + gn_cross_cta(torch.stack([t for t, _ in cta]), parts)
        dk = xg[b] - k[b][None, :, None]
        var = xg[b].var(dim=(0, 2), correction=0)
        dm, dr = gn_stats_err(run, dk.abs().sum(dim=(0, 2)), (dk * dk).sum(dim=(0, 2)), HW * cpg,
                              dk.mean(dim=(0, 2)), var, eps)
        d_mean.append(dm)
        d_rstd.append(dr)
        r.append((var + eps).rsqrt())
    return torch.stack(d_mean), torch.stack(d_rstd), torch.stack(r)


def gn_stats_excess(y, gamma, r, d_mean, d_rstd, allowance):
    """What the statistics' rounding (gn_stats_err) can add to g (x - mean) rstd + b beyond `allowance` |g|, the unit
    the normalisation bound has always given them: |g| max(0, rstd d_mean + |y| d_rstd - allowance).  y: the
    normalised value; r / d_mean / d_rstd broadcast against it."""
    return gamma.abs() * (r * d_mean + y.abs() * d_rstd - allowance).clamp_min(0.0)


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


def conv_gemm(x, w, mode, extra=None):
    """ea_gemm's implicit-GEMM convolutions.  x: NHWC input [B, Hin, Win, Cin]; w: [Cout, 9 Cin (+ Cin_extra)] with K
    index (kh * 3 + kw) * Cin + c; mode "s1" (3x3, stride 1, pad 1), "s2" (stride 2, pad 1 on the 2H x 2W input) or
    "s2a" (F.pad(x, (0, 1, 0, 1)), then stride 2, pad 0); extra: [B, H, W, Cin_extra], the operand of the folded 1x1
    skip convolution (the last Cin_extra columns of w).  Returns (out [B, H, W, Cout], sum of |a w|), no bias."""
    cout, cin = w.shape[0], x.shape[-1]
    wt = w[:, :9 * cin].reshape(cout, 3, 3, cin).permute(0, 3, 1, 2)
    xc = x.permute(0, 3, 1, 2)
    if mode == "s2a":
        xc, kw = F.pad(xc, (0, 1, 0, 1)), dict(stride=2)
    else:
        kw = dict(stride=1 if mode == "s1" else 2, padding=1)
    out = F.conv2d(xc, wt, **kw).permute(0, 2, 3, 1)
    mag = F.conv2d(xc.abs(), wt.abs(), **kw).permute(0, 2, 3, 1)
    if extra is not None:
        we = w[:, 9 * cin:]
        out, mag = out + extra @ we.T, mag + extra.abs() @ we.abs().T
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


# ---- per-element gate -------------------------------------------------------------------------------------------
def worst_element(got, ref, bound):
    """(worst |got - ref| / bound, its flat index, number of elements out of bound) of got against a float64 reference;
    a NaN difference counts as infinitely far, an exact match as 0 whatever the bound."""
    err = (got.double() - ref).abs()
    ratio = torch.where(err == 0, torch.zeros_like(err), err / bound)
    ratio = torch.where(torch.isnan(err), torch.full_like(err, math.inf), ratio)
    i = int(torch.argmax(ratio.reshape(-1)))
    return float(ratio.reshape(-1)[i]), i, int((~(err <= bound)).sum())


# ---- GEMM epilogue ---------------------------------------------------------------------------------------------
def gemm_act(act, pre, e):
    """act(pre) and its error bound for an fp32 pre-activation `pre` (float64) whose error is bounded by `e`; act is
    "none", "silu", "gelu" or "geglu" (pre in the packed [value | gate] layout)."""
    if act == "none":
        return pre, e
    if act == "silu":
        return silu(pre), 1.1 * e + silu_eval_err(pre)
    if act == "gelu":
        return gelu(pre), 1.13 * e + gelu_eval_err(pre)
    x, g = geglu_split(pre)
    ex, eg = geglu_split(e)
    gg = gelu(g)
    return x * gg, gg.abs() * ex + x.abs() * (1.13 * eg + gelu_eval_err(g))


def gemm_out(y, err, scale=1.0, extras=(), out_dtype=None, n_scale=0):
    """(reference, bound) of the stored GEMM output y * scale (+ each of `extras`: residual, accumulated value) for an
    activation output y with error bound err: the scaled error, one u per add, and 1 ulp of out_dtype (None: an fp32
    destination, no ulp).  `scale` may be a tensor (out_scale * row_scale[m]).  n_scale: the number of fp32 products
    the scale takes (out_scale, row_scale), one u of |y * scale| each - the ulp of a half destination covers them,
    an fp32 destination (the VAE logits, an accumulated zero-conv into fp32) needs them counted."""
    t = y * scale
    ref = t + sum(extras) if extras else t
    bound = abs(scale) * err + (1 + len(extras)) * U32 * (t.abs() + sum(v.abs() for v in extras))
    if n_scale:
        bound = bound + n_scale * U32 * t.abs()
    if out_dtype is not None:
        bound = bound + ulp(ref, out_dtype)
    return ref, bound


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
