"""-m gpu: the tile-refinement sizes on one H100.  The SD VAE encodes a 2048 x 2752 image and decodes 256 x 344
latents (N = 88064 attention tokens, past vae.FUSED_ATTN_MIN_TOKENS: the AttnBlock runs ea_attention) with graphs
on, within a fraction of the N x N logits the GEMM path would store (tests/test_gpu_highres_audit.py audits every
launch at that size); the decoder matches the fp32 oracle at 128 x 128 latents on both
AttnBlock paths; and the SD1.5 tile pass runs end to end at 2048 x 2752."""
import numpy as np
import PIL.Image
import pytest
import torch

from editanything_b200.denoise import DenoiseEngine
from editanything_b200.pipeline import StableDiffusionControlNetInpaintPipeline
from editanything_b200 import vae as vae_mod
from editanything_b200.unet_spec import SD15, make_state_dict
from editanything_b200.vae import SD_VAE, VaeDecoderEngine, VaeEngine, make_vae_state_dict
from oracle import vae_oracle as V

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
H, W = 2048, 2752                     # the long side of a 4:3 photo refined at 2048
N = (H // 8) * (W // 8)               # 88064 latent tokens
N2_HALF = N * N * 2                   # bytes of the N x N half P matrix of the GEMM path


def _vae():
    sd = dict(make_vae_state_dict(SD_VAE, 412, part="encoder"))
    sd.update(make_vae_state_dict(SD_VAE, 402))
    return VaeEngine(SD_VAE, sd, DEV)


def _peak_growth(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    out = fn()
    torch.cuda.synchronize()
    return out, torch.cuda.max_memory_allocated() - base


def _finite_not_constant(t, what):
    assert bool(torch.isfinite(t).all()), what
    assert float(t.float().std()) > 1e-3, what


def test_vae_2048x2752_graphed():
    vae = _vae()
    g = torch.Generator().manual_seed(0)
    x = torch.rand(1, 3, H, W, generator=g) * 2 - 1
    dist, grow_e = _peak_growth(lambda: vae.encode(x).latent_dist)
    _finite_not_constant(dist.mean, "encode mean")
    lat = torch.randn(1, 4, H // 8, W // 8, generator=g)
    img, grow_d = _peak_growth(lambda: vae.decode_latents(lat))
    assert img.shape == (1, 3, H, W)
    _finite_not_constant(img, "decoded image")
    print(f"peak allocation growth: encode {grow_e / 2**30:.2f} GiB, decode {grow_d / 2**30:.2f} GiB "
          f"(N^2 half = {N2_HALF / 2**30:.2f} GiB)")
    assert grow_e < N2_HALF and grow_d < N2_HALF


@pytest.mark.parametrize("fused", [False, True])
def test_decode_parity_128(fused, monkeypatch):
    """At 128 x 128 latents the AttnBlock runs the GEMM path; `fused` forces ea_attention there too."""
    if fused:
        monkeypatch.setattr(vae_mod, "FUSED_ATTN_MIN_TOKENS", 0)
    sd = make_vae_state_dict(SD_VAE, 402)
    eng = VaeDecoderEngine(SD_VAE, sd, DEV)
    lat = torch.randn(1, 4, 128, 128, generator=torch.Generator().manual_seed(5))
    out = eng.decode_latents(lat).float().cpu()
    tf32 = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with torch.no_grad():
            ref = V.decode_latents(lat.to(DEV), {k: v.to(DEV) for k, v in sd.items()}, SD_VAE).float().cpu()
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32
    err, mean = (out - ref).abs().max().item(), (out - ref).abs().mean().item()
    print(f"SD VAE decode 128x128 latents (fused={fused}) vs fp32 oracle: max-abs {err:.3e} mean-abs {mean:.3e}")
    assert out.shape == ref.shape and err < 2e-2 and mean < 2e-3


def test_tile_pass_2048x2752():
    eng = DenoiseEngine(SD15, make_state_dict(SD15, "unet", 201), [make_state_dict(SD15, "controlnet", 202)], DEV)
    pipe = StableDiffusionControlNetInpaintPipeline(eng, vae=_vae())
    g = torch.Generator().manual_seed(3)
    img = PIL.Image.fromarray(np.asarray(torch.randint(0, 256, (H, W, 3), generator=g, dtype=torch.uint8)))
    m = np.zeros((H, W), np.uint8)
    m[H // 4:3 * H // 4, W // 4:3 * W // 4] = 255
    mask = PIL.Image.fromarray(m)
    pe = torch.randn(1, 77, 768, generator=g)
    ne = torch.randn(1, 77, 768, generator=g)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    # 21 steps: with alignment_ratio 0.95 the reference blends through timesteps[i + 1], which needs a step past the
    # last blended one (0.95 n < n - 1)
    res = pipe(image=img, mask_image=mask, prompt_embeds=pe, negative_prompt_embeds=ne, num_inference_steps=21,
               generator=torch.Generator().manual_seed(4), controlnet_conditioning_image=img, height=H, width=W,
               controlnet_conditioning_scale=1.0, alignment_ratio=0.95, guidance_scale=9.0).images
    torch.cuda.synchronize()
    print(f"tile pass {W}x{H}: peak allocated {torch.cuda.max_memory_allocated() / 2**30:.2f} GiB")
    assert len(res) == 1 and res[0].size == (W, H)
    a = np.asarray(res[0]).astype(np.float64)
    assert np.isfinite(a).all() and a.std() > 1.0
