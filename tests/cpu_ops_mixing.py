"""Torch/CPU emulation of editanything_b200.ops for the alpha-mixing pipeline - TEST INFRASTRUCTURE ONLY.

Every operator of tests/cpu_ops_vpred.py, plus `latent_mix` (ea_latent_mix): the buffers are checked with
editanything_b200.ops.check_mix_buffers as the CUDA wrapper checks them, then row *step_counter - 1 of the tables
mixes the latents in fp32 and rewrites lat_half_out.  Injected explicitly by the tests (`backend=cpu_ops_mixing`)."""
import torch

from editanything_b200.ops import check_mix_buffers
from tests import cpu_ops
from tests.cpu_ops_vpred import *  # noqa: F401,F403  (every other operator unchanged)


def latent_mix(latents, known, mask, noise, mix, *, alpha, step_counter, lat_half_out=None, copies=1, Nimg, H, W):
    check_mix_buffers(latents, known, mask, noise, mix, step_counter, lat_half_out, copies, Nimg, H, W)
    cpu_ops._bump()
    r = int(step_counter[0]) - 1
    if not 0 <= r < mix.shape[0] or float(mix[r, 3]) == 0.0:
        return
    k_init, k_noise, in_window = (float(v) for v in mix[r, :3])
    m = mask.reshape(Nimg, H, W, 1)
    x = latents.reshape(Nimg, H, W, 4)
    p = k_init * known.reshape(x.shape) + k_noise * noise.reshape(-1, Nimg, H, W, 4)[r]
    keep = p if in_window != 0.0 else x
    xn = keep * m + ((1 - alpha) * x + alpha * p) * (1 - m)
    latents.copy_(xn.reshape(latents.shape))
    if lat_half_out is not None:
        lat_half_out.copy_(torch.cat([xn] * copies).reshape(lat_half_out.shape).to(lat_half_out.dtype))
