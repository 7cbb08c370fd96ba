"""Torch/CPU emulation of editanything_b200.ops for v-prediction base models - TEST INFRASTRUCTURE ONLY.

Every operator of tests/cpu_ops_unguided.py, with `out_cfg_ddim` / `out_ddim` taking `prediction` like the CUDA
wrappers: "epsilon" is the update of tests/cpu_ops_unguided.py unchanged; "v_prediction" (ea_out_cfg_vpred /
ea_out_vpred) reads the guidance-combined network output m as v, x0 = coef[0] x - coef[1] m, eps = coef[0] m +
coef[1] x, then the same DDIM / multistep update, blend, history and step counter.  eps_out stays the raw network
output.  Any other prediction raises ValueError before anything is written, as the wrappers do.  Injected explicitly
by the tests (`backend=cpu_ops_vpred`)."""
import torch
import torch.nn.functional as F

from editanything_b200.ops import check_out_buffers, check_prediction
from tests import cpu_ops, cpu_ops_unguided
from tests.cpu_ops_unguided import *  # noqa: F401,F403  (every other operator unchanged)


def _update_v(m, latents, coef, known, noise, mask, hist, step_counter):
    """The v-mode update of the kernels (include/editanything_b200.h, ea_out_cfg_vpred)."""
    sa, s1a, sap, s1ap = [float(c) for c in coef[:4]]
    x0 = sa * latents - s1a * m
    e = sa * m + s1a * latents
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
    return xp


def _conv(xn, w, bias):
    return F.conv2d(xn.float().permute(0, 3, 1, 2), w.permute(0, 3, 1, 2), bias, padding=1).permute(0, 2, 3, 1)


def out_cfg_ddim(xn, w, bias, *, latents=None, eps_out=None, coef=None, guidance=1.0, known=None, noise=None,
                 mask=None, lat_half_out=None, step_counter=None, hist=None, Nimg, H, W, C_, prediction="epsilon"):
    check_prediction("out_cfg_ddim", prediction)
    if prediction == "epsilon":
        cpu_ops_unguided.out_cfg_ddim(xn, w, bias, latents=latents, eps_out=eps_out, coef=coef, guidance=guidance,
                                      known=known, noise=noise, mask=mask, lat_half_out=lat_half_out,
                                      step_counter=step_counter, hist=hist, Nimg=Nimg, H=H, W=W, C_=C_)
        return
    check_out_buffers("out_cfg_ddim", 2, xn, w, bias, latents, eps_out, coef, known, noise, mask, lat_half_out,
                      step_counter, hist, Nimg, H, W, C_)
    cpu_ops._bump()
    out = _conv(xn, w, bias)
    if eps_out is not None:
        eps_out.copy_(out)
    if latents is None:
        return
    m = out[:Nimg] + guidance * (out[Nimg:] - out[:Nimg])          # cldm/ddim_hacked.py:192, applied to v
    xp = _update_v(m, latents, coef, known, noise, mask, hist, step_counter)
    if lat_half_out is not None:
        lat_half_out.copy_(torch.cat([xp, xp]))


def out_ddim(xn, w, bias, *, latents=None, eps_out=None, coef=None, known=None, noise=None, mask=None,
             lat_half_out=None, step_counter=None, hist=None, Nimg, H, W, C_, prediction="epsilon"):
    check_prediction("out_ddim", prediction)
    if prediction == "epsilon":
        cpu_ops_unguided.out_ddim(xn, w, bias, latents=latents, eps_out=eps_out, coef=coef, known=known, noise=noise,
                                  mask=mask, lat_half_out=lat_half_out, step_counter=step_counter, hist=hist,
                                  Nimg=Nimg, H=H, W=W, C_=C_)
        return
    check_out_buffers("out_ddim", 1, xn, w, bias, latents, eps_out, coef, known, noise, mask, lat_half_out,
                      step_counter, hist, Nimg, H, W, C_)
    cpu_ops._bump()
    out = _conv(xn, w, bias)
    if eps_out is not None:
        eps_out.copy_(out)
    if latents is None:
        return
    xp = _update_v(out, latents, coef, known, noise, mask, hist, step_counter)
    if lat_half_out is not None:
        lat_half_out.copy_(xp)
