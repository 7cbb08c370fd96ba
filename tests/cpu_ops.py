"""Torch/CPU emulation of editanything_b200.ops — TEST INFRASTRUCTURE ONLY.

Lets the `-m "not gpu"` suite exercise the host-side graph logic (weight packing, skip-concat
sinks, zero-conv accumulation, GEGLU interleave, fused-skip K extension ...) of
editanything_b200.nets against the oracle without a GPU.  It is injected explicitly by the tests
(`PackedNet(..., backend=cpu_ops)`); the product never selects it.
"""
import torch
import torch.nn.functional as F

EA_GEMM_LINEAR, EA_GEMM_CONV_S1, EA_GEMM_CONV_S2, EA_GEMM_CONV_S2A = 0, 1, 2, 3
EA_ACT_NONE, EA_ACT_SILU, EA_ACT_GELU, EA_ACT_GEGLU = 0, 1, 2, 3
_count = 0


def half_dtype():
    return torch.float32


def launch_count():
    return _count


def _bump(n=1):
    global _count
    _count += n


def gemm(a, w, out=None, *, mode=0, M=None, N=None, K=None, lda=None, ldw=0, conv=None, a_extra=None,
         bias=None, rowvec=None, rows_per_batch=0, residual=None, out2=None, out_f32=None, act=0,
         out_scale=1.0, accumulate=False, ldo=None, ldr=None, ldo2=None, ld_extra=0, force_bn=0,
         force_splits=0, force_2cta=0, force_persistent=0, rowstats_out=None, ln=None, row_scale=None):
    if act == EA_ACT_GEGLU and (rowvec is not None or residual is not None or out2 is not None or out_f32 is not None
                                or accumulate or out_scale != 1.0 or row_scale is not None):
        raise RuntimeError("ea_gemm failed (-1): GEGLU applies the bias and the LayerNorm fold only")
    if (ln is not None or rowstats_out is not None) and rows_per_batch:
        raise RuntimeError("ea_gemm failed (-1): no rows_per_batch with the LayerNorm fold")
    _bump()
    Nn = w.shape[0]
    if mode == EA_GEMM_LINEAR:
        A = a.reshape(-1, a.shape[-1]).float()
        y = A @ w.float().t()
        batch_rows = rows_per_batch
        if ln is not None:      # LayerNorm fold: rstd * (x W'^T - mean * g) (+ bias below), stats from the producer
            stats, g, eps = ln
            s, m2 = stats[..., 0].float(), stats[..., 1].float()      # [K/32, M] per chunk: sum, M2 about its mean
            mu = s.sum(0) / A.shape[1]
            var = (m2.sum(0) + 32.0 * ((s / 32.0 - mu) ** 2).sum(0)) / A.shape[1]
            rstd = torch.rsqrt(var + eps)
            y = rstd[:, None] * (y - mu[:, None] * g[None, :])
    else:
        B, H, W_, Cin = conv
        x = a.float().reshape(B, -1, a.shape[-2] if a.dim() == 4 else (W_ if mode == EA_GEMM_CONV_S1 else 2 * W_), Cin).permute(0, 3, 1, 2)
        wm = w[:, :9 * Cin].float().reshape(Nn, 3, 3, Cin).permute(0, 3, 1, 2)
        if mode == EA_GEMM_CONV_S2A:
            y = F.conv2d(F.pad(x, (0, 1, 0, 1)), wm, stride=2, padding=0)
        else:
            y = F.conv2d(x, wm, stride=1 if mode == EA_GEMM_CONV_S1 else 2, padding=1)
        if a_extra is not None:
            ce = a_extra.shape[-1]
            y = y + F.conv2d(a_extra.float().permute(0, 3, 1, 2), w[:, 9 * Cin:9 * Cin + ce].float().reshape(Nn, ce, 1, 1))
        y = y.permute(0, 2, 3, 1).reshape(B * H * W_, Nn)
        batch_rows = H * W_
    if bias is not None:
        y = y + bias
    if rowvec is not None:
        nb = y.shape[0] // batch_rows if batch_rows else 1
        y = y + (rowvec.repeat_interleave(batch_rows, 0)[:y.shape[0]] if batch_rows else rowvec[:1])
    if act == EA_ACT_SILU:
        y = F.silu(y)
    elif act == EA_ACT_GELU:
        y = F.gelu(y)
    elif act == EA_ACT_GEGLU:
        y = y.reshape(y.shape[0], Nn // 128, 2, 64)
        y = (y[:, :, 0] * F.gelu(y[:, :, 1])).reshape(y.shape[0], Nn // 2)
    y = y * out_scale
    if row_scale is not None:
        y = y * row_scale.reshape(-1, 1)
    if residual is not None:
        y = y + residual.reshape(y.shape).float()
    tgt = out if out is not None else out_f32
    if tgt is None:
        tgt = torch.empty(y.shape, dtype=half_dtype())
    if accumulate:
        y = y + tgt.reshape(y.shape).float()
    tgt.copy_(y.reshape(tgt.shape))
    if out2 is not None:
        out2.copy_(y.reshape(out2.shape))
    if rowstats_out is not None:    # statistics of the stored values, each chunk's M2 about its own mean
        yc = tgt.float().reshape(y.shape[0], -1, 32)
        s = yc.sum(-1)
        m2 = ((yc - (s / 32.0)[..., None]) ** 2).sum(-1)
        rowstats_out.copy_(torch.stack([s, m2], -1).permute(1, 0, 2))
    return tgt


def gemm_grouped(calls):
    return [gemm(a, w, out, **kw) for a, w, out, kw in calls]


def attention(q, k, v, out, *, B, heads, Nq, Nkv, d, q_strides, k_strides, v_strides, o_strides, scale,
              rel_h=None, rel_w=None, rel_s=0):
    _bump()

    def view(t, N, st):
        return torch.as_strided(t, (B, N, heads, d), (st[0], st[1], d, 1), t.storage_offset()).float()

    qf = view(q, Nq, q_strides).permute(0, 2, 1, 3)
    kf = view(k, Nkv, k_strides).permute(0, 2, 1, 3)
    vf = view(v, Nkv, v_strides).permute(0, 2, 1, 3)
    s = qf @ kf.transpose(-1, -2) * scale
    if rel_h is not None:
        bias = rel_h.reshape(B, heads, Nq, rel_s, 1) + rel_w.reshape(B, heads, Nq, 1, rel_s)
        s = s + bias.reshape(B, heads, Nq, rel_s * rel_s)[..., :Nkv]
    o = (s.softmax(-1) @ vf).permute(0, 2, 1, 3).reshape(B, Nq, heads * d)
    torch.as_strided(out, (B, Nq, heads * d), (o_strides[0], o_strides[1], 1), out.storage_offset()).copy_(o)
    return out


def gn_workspace(B, device, groups=32):
    return torch.zeros(2 * B + 2 * groups * 256, device=device, dtype=torch.float32)


def groupnorm(x, gamma, beta, out, *, B, HW, C_, groups=32, eps=1e-5, silu=True, workspace=None, x2=None,
              C1=0, ldx=None, ldx2=None, ldo=None):
    _bump(2)
    xs = x.reshape(B, HW, -1).float()
    if x2 is not None:
        xs = torch.cat([xs, x2.reshape(B, HW, -1).float()], -1)
    if isinstance(gamma, (list, tuple)):       # stacked networks: images [g*B/n, (g+1)*B/n) use gamma[g] / beta[g]
        n = len(gamma)
        ipg = B // n
        y = torch.cat([F.group_norm(xs[g * ipg:(g + 1) * ipg].permute(0, 2, 1), groups, gamma[g], beta[g], eps)
                       for g in range(n)]).permute(0, 2, 1)
    else:
        y = F.group_norm(xs.permute(0, 2, 1), groups, gamma, beta, eps).permute(0, 2, 1)
    if silu:
        y = F.silu(y)
    out.copy_(y.reshape(out.shape))
    return out


def layernorm(x, gamma, beta, out, *, M, C_, eps=1e-5, ldx=None, ldo=None):
    _bump()
    out.copy_(F.layer_norm(x.float().reshape(M, C_), (C_,), gamma, beta, eps).reshape(out.shape))
    return out


def conv_direct(x, w, bias, out, *, B, Hin, Win, Cin, Cout, ksize=3, stride=1, silu=False, add=None, ldo=0):
    _bump()
    y = F.conv2d(x.float().reshape(B, Hin, Win, Cin).permute(0, 3, 1, 2), w.permute(3, 2, 0, 1), bias, stride=stride,
                 padding=ksize // 2)
    if silu:
        y = F.silu(y)
    y = y.permute(0, 2, 3, 1)
    if add is not None:
        y = y + add.float().reshape(y.shape)
    if ldo and ldo != Cout:          # output pixel stride > Cout: only the first Cout channels of every pixel are written
        out.reshape(-1, ldo)[:, :Cout].copy_(y.reshape(-1, Cout))
    else:
        out.copy_(y.reshape(out.shape))
    return out


def conv_in(x, w, bias, out, *, B, H, W, Cin, Cout, out2=None, add=None, ldo=0, ldo2=0):
    _bump()
    y = F.conv2d(x.float().reshape(B, H, W, Cin).permute(0, 3, 1, 2), w.permute(3, 2, 0, 1), bias, padding=1).permute(0, 2, 3, 1)
    if add is not None:
        y = y + add.float().reshape(y.shape)
    out.copy_(y.reshape(out.shape))
    if out2 is not None:
        out2.copy_(y.reshape(out2.shape))
    return out


def upsample2x(x, out, *, B, H, W, C_):
    _bump()
    out.copy_(F.interpolate(x.float().reshape(B, H, W, C_).permute(0, 3, 1, 2), scale_factor=2,
                            mode="nearest").permute(0, 2, 3, 1).reshape(out.shape))
    return out


def small_linear(x, w, bias, y, *, M, N, K, silu_in=False, silu_out=False):
    _bump()
    xx = F.silu(x) if silu_in else x
    r = xx @ w.float().t()
    if bias is not None:
        r = r + bias
    y.copy_(F.silu(r) if silu_out else r)
    return y


def timestep_embedding(t, out, *, B, dim):
    _bump()
    half = dim // 2
    freqs = torch.exp(-torch.log(torch.tensor(10000.0)) * torch.arange(half, dtype=torch.float32) / half)
    args = t[:, None].float() * freqs[None]
    out.copy_(torch.cat([torch.cos(args), torch.sin(args)], -1))
    return out


def step_gather(step_counter, n_rows, tables, dsts):
    _bump()
    row = max(0, min(int(step_counter.item()), n_rows - 1))
    for t, d in zip(tables, dsts):
        d.copy_(t[row].reshape(d.shape))


def out_cfg_ddim(xn, w, bias, *, latents=None, eps_out=None, coef=None, guidance=1.0, known=None, noise=None,
                 mask=None, lat_half_out=None, step_counter=None, hist=None, Nimg, H, W, C_):
    _bump()
    eps = F.conv2d(xn.float().permute(0, 3, 1, 2), w.permute(0, 3, 1, 2), bias, padding=1).permute(0, 2, 3, 1)
    if eps_out is not None:
        eps_out.copy_(eps)
    if latents is not None:
        e = eps[:Nimg] + guidance * (eps[Nimg:] - eps[:Nimg])
        sa, s1a, sap, s1ap = [float(c) for c in coef[:4]]
        x0 = (latents - s1a * e) / sa
        xp = sap * x0 + s1ap * e
        if hist is not None and float(coef[7]) != 0.0:
            c = [float(v) for v in coef]
            m1, m2, last = hist[0].clone(), hist[1].clone(), hist[2].clone()
            xc = c[8] * latents + c[9] * last + c[10] * m1 + c[11] * m2 + c[12] * x0
            xp = c[13] * xc + c[14] * x0 + c[15] * m1
            hist[1].copy_(m1)
            hist[0].copy_(x0)
            hist[2].copy_(xc)
        if known is not None:
            kn, mk = known, mask[..., None]
            if noise is not None:
                kn = float(coef[4]) * known + float(coef[5]) * noise
                mk = mk * float(coef[6])
            xp = kn * mk + xp * (1 - mk)
        if step_counter is not None:
            step_counter += 1
        latents.copy_(xp)
        if lat_half_out is not None:
            lat_half_out.copy_(torch.cat([xp, xp]))


# ------------------------------------------------------------------ SAM helpers
def sam_relpos(q, q_bs, q_ns, Rh, Rw, rel_h, rel_w, *, B, heads, S, d):
    _bump()
    qf = torch.as_strided(q, (B, S * S, heads, d), (q_bs, q_ns, d, 1), q.storage_offset()).float()
    qf = qf.permute(0, 2, 1, 3).reshape(B * heads, S, S, d)
    rel_h.copy_(torch.einsum("bhwc,hkc->bhwk", qf, Rh).reshape(rel_h.shape))
    rel_w.copy_(torch.einsum("bhwc,wkc->bhwk", qf, Rw).reshape(rel_w.shape))


def window_partition(x, out, *, B, H, W, C_, ws):
    _bump()
    nWh, nWw = (H + ws - 1) // ws, (W + ws - 1) // ws
    xp = F.pad(x.reshape(B, H, W, C_), (0, 0, 0, nWw * ws - W, 0, nWh * ws - H))
    out.copy_(xp.view(B, nWh, ws, nWw, ws, C_).permute(0, 1, 3, 2, 4, 5).reshape(out.shape))
    return out


def window_unpartition(xw, residual, out, *, B, H, W, C_, ws):
    _bump()
    nWh, nWw = (H + ws - 1) // ws, (W + ws - 1) // ws
    x = xw.reshape(B, nWh, nWw, ws, ws, C_).permute(0, 1, 3, 2, 4, 5).reshape(B, nWh * ws, nWw * ws, C_)[:, :H, :W]
    if residual is not None:
        x = x + residual.reshape(B, H, W, C_)
    out.copy_(x.reshape(out.shape))
    return out


def sam_patchify(img, out, *, B, Cin, H, W, ps):
    _bump()
    cols = F.unfold(img.float(), kernel_size=ps, stride=ps)          # [B, Cin*ps*ps, L], K order (c, kh, kw)
    out.copy_(cols.permute(0, 2, 1).reshape(out.shape))
    return out


def nhwc_to_nchw_f32(x, out, *, B, HW, C_):
    _bump()
    out.copy_(x.float().reshape(B, HW, C_).permute(0, 2, 1).reshape(out.shape))
    return out


def softmax_rows(s, p, *, rows, cols, lds=None, ldp=None):
    _bump()
    p.copy_(s.float().reshape(rows, cols).softmax(-1).reshape(p.shape))
    return p


def image_out(x, out, *, B, HW, C_, ldx, scale=0.5, shift=0.5, lo=0.0, hi=1.0):
    _bump()
    v = x.float().reshape(B, HW, ldx)[:, :, :C_] * scale + shift
    out.copy_(v.clamp(lo, hi).permute(0, 2, 1).reshape(out.shape))
    return out

