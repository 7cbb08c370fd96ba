"""CPU suite for the SD VAE's AttnBlock on both of its paths: SD_VAE (one head of d = 512) encodes and decodes
through tests/cpu_ops.py as the oracle (oracle/vae_oracle.py) does.  With the fused path (sequences longer than
vae.FUSED_ATTN_MIN_TOKENS, forced here at 8 x 8 latents) every attention block is one `attention` call with
heads = 1 and d = 512 over all images and no `softmax_rows`; with the GEMM path it is one `softmax_rows` per image
and no `attention`.  Every launch passes the launch auditor (tests/launch_audit.py)."""
import pytest
import torch

from editanything_b200 import vae as vae_mod
from editanything_b200.vae import SD_VAE, VaeDecoderEngine, VaeEncoderEngine, make_vae_state_dict
from oracle import vae_oracle as V
from tests import cpu_ops
from tests.launch_audit import Auditor

CPU = torch.device("cpu")
REL_FRO = 1e-4


class Trace:
    """Forwards every operator to `backend` and records (name, keyword arguments)."""

    def __init__(self, backend):
        self.backend, self.calls = backend, []

    def __getattr__(self, name):
        fn = getattr(self.backend, name)
        if name == "half_dtype" or not callable(fn):
            return fn

        def call(*args, **kw):
            self.calls.append((name, kw))
            return fn(*args, **kw)
        return call


def _n_attn_blocks(blocks):
    return sum(kind == "attn" for kind, *_ in blocks)


def _check_trace(tr, eng, B, n_tokens, fused):
    n_blocks = _n_attn_blocks(eng.blocks)
    assert n_blocks >= 1
    attn = [kw for name, kw in tr.calls if name == "attention"]
    n_softmax = sum(name == "softmax_rows" for name, _ in tr.calls)
    if not fused:
        assert not attn and n_softmax == B * n_blocks
        return
    assert len(attn) == n_blocks
    for kw in attn:
        assert (kw["B"], kw["heads"], kw["d"], kw["Nq"], kw["Nkv"]) == (B, 1, 512, n_tokens, n_tokens), kw
    assert n_softmax == 0


def _rel(a, b):
    return ((a - b).norm() / b.norm()).item()


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("h,w", [(8, 8), (8, 12)])
def test_sd_vae_decode(h, w, fused, monkeypatch):
    if fused:
        monkeypatch.setattr(vae_mod, "FUSED_ATTN_MIN_TOKENS", 0)
    sd = make_vae_state_dict(SD_VAE, 402)
    aud = Auditor(cpu_ops, f"sd_vae_decoder_{h}x{w}")
    tr = Trace(aud)
    eng = VaeDecoderEngine(SD_VAE, sd, CPU, backend=tr)
    lat = torch.randn(2, SD_VAE.z_channels, h, w, generator=torch.Generator().manual_seed(h * w))
    img = eng.decode_latents(lat, use_graph=False)
    with torch.no_grad():
        ref = V.decode_latents(lat, sd, SD_VAE)
    assert img.shape == ref.shape == (2, 3, 8 * h, 8 * w)
    rel = _rel(img, ref)
    print(f"sd_vae decode {h}x{w}: rel-fro {rel:.3e} max-abs {(img - ref).abs().max().item():.3e}")
    assert rel < REL_FRO
    _check_trace(tr, eng, 2, h * w, fused)
    assert aud.calls > 50


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("h,w", [(8, 8), (8, 12)])
def test_sd_vae_encode(h, w, fused, monkeypatch):
    if fused:
        monkeypatch.setattr(vae_mod, "FUSED_ATTN_MIN_TOKENS", 0)
    sd = make_vae_state_dict(SD_VAE, 412, part="encoder")
    aud = Auditor(cpu_ops, f"sd_vae_encoder_{h}x{w}")
    tr = Trace(aud)
    eng = VaeEncoderEngine(SD_VAE, sd, CPU, backend=tr)
    x = torch.rand(2, 3, 8 * h, 8 * w, generator=torch.Generator().manual_seed(h + w)) * 2 - 1
    dist = eng.encode(x, use_graph=False).latent_dist
    mom = torch.cat([dist.mean, dist.logvar], 1)
    with torch.no_grad():
        ref = V.encode_moments(x, sd, SD_VAE)
    ref = torch.cat([ref[:, :SD_VAE.z_channels], ref[:, SD_VAE.z_channels:].clamp(-30.0, 20.0)], 1)
    assert mom.shape == ref.shape == (2, 2 * SD_VAE.z_channels, h, w)
    rel = _rel(mom, ref)
    print(f"sd_vae encode {h}x{w}: rel-fro {rel:.3e} max-abs {(mom - ref).abs().max().item():.3e}")
    assert rel < REL_FRO
    _check_trace(tr, eng, 2, h * w, fused)
    assert aud.calls > 50
