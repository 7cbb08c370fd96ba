"""Torch/CPU emulation of editanything_b200.ops for sampling without guidance - TEST INFRASTRUCTURE ONLY.

Every operator of tests/cpu_ops.py, plus `out_ddim` (ea_out_ddim: the out conv and scheduler update of
out_cfg_ddim on N-row buffers, without guidance).  Both out-conv operators first check their buffers with
editanything_b200.ops.check_out_buffers, as the CUDA wrappers do, so a buffer sized for the other entry point fails
here on the CPU as it would before a launch.  Injected explicitly by the tests (`backend=cpu_ops_unguided`)."""
import torch.nn.functional as F

from editanything_b200.ops import check_out_buffers
from tests import cpu_ops
from tests.cpu_ops import *  # noqa: F401,F403  (every other operator unchanged)


def out_cfg_ddim(xn, w, bias, *, latents=None, eps_out=None, coef=None, guidance=1.0, known=None, noise=None,
                 mask=None, lat_half_out=None, step_counter=None, hist=None, Nimg, H, W, C_):
    check_out_buffers("out_cfg_ddim", 2, xn, w, bias, latents, eps_out, coef, known, noise, mask, lat_half_out,
                      step_counter, hist, Nimg, H, W, C_)
    cpu_ops.out_cfg_ddim(xn, w, bias, latents=latents, eps_out=eps_out, coef=coef, guidance=guidance, known=known,
                         noise=noise, mask=mask, lat_half_out=lat_half_out, step_counter=step_counter, hist=hist,
                         Nimg=Nimg, H=H, W=W, C_=C_)


def out_ddim(xn, w, bias, *, latents=None, eps_out=None, coef=None, known=None, noise=None, mask=None,
             lat_half_out=None, step_counter=None, hist=None, Nimg, H, W, C_):
    check_out_buffers("out_ddim", 1, xn, w, bias, latents, eps_out, coef, known, noise, mask, lat_half_out,
                      step_counter, hist, Nimg, H, W, C_)
    cpu_ops._bump()
    e = F.conv2d(xn.float().permute(0, 3, 1, 2), w.permute(0, 3, 1, 2), bias, padding=1).permute(0, 2, 3, 1)
    if eps_out is not None:
        eps_out.copy_(e)
    if latents is None:
        return
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
        lat_half_out.copy_(xp)
