"""-m gpu: every launch of the 2048 x 2752 tile-refinement pass audited by tests/launch_audit.py on one H100: the SD VAE
decoder at 256 x 344 latents and encoder at 2048 x 2752 (the 256-channel full-resolution upsample output is 2.9 GB,
past 2^31 bytes; the full-resolution GroupNorms reduce 45 M values per statistic), and two UniPC steps of the SD1.5
tile pass in lockstep with one ControlNet, its hint stack at 2048 x 2752 (88064-token self-attention at level 1, the
inpaint blend live).  Each launch runs eagerly through the auditor; the same decode and steps replayed from their
CUDA graphs must equal the eager results bit for bit, so that the audited launches are the ones the pipeline runs.

The module prints, per case, the number of audited launches, the wall time, the device's peak allocation and the
auditor's own largest growth during one call, and the worst error / bound per (op, call site)."""
import time

import pytest
import torch

from editanything_b200 import ops
from editanything_b200.denoise import DenoiseEngine
from editanything_b200.unet_spec import SD15, make_state_dict
from editanything_b200.vae import SD_VAE, VaeDecoderEngine, VaeEncoderEngine, make_vae_state_dict
from tests.launch_audit import Auditor, set_unipc
from tests.test_step_trace_cpu import _set_env

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
H, W = 2048, 2752
h, w = H // 8, W // 8                 # 256 x 344 latents, 88064 tokens
WORST = {}          # (op, call site) -> worst error / bound over every case
WORST_UNIT = {}     # GroupNorm (op, call site) -> the same without the derived statistics term
RUNS = {}           # case -> (audited launches, seconds, peak GiB, the auditor's own peak GiB)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if RUNS:
        print(f"\n{torch.cuda.get_device_name(DEV)}: audited launches, wall time, peak device memory and the "
              f"auditor's own largest growth in one call, per case:")
        for k, (n, s, m, own) in RUNS.items():
            print(f"  {k:28s} {n:5d} launches  {s:7.1f} s  {m:6.2f} GiB  auditor {own:6.2f} GiB")
    if WORST:
        print("worst error / bound per (op, call site):")
        for (op, site), v in sorted(WORST.items()):
            unit = f"  (without the derived statistics term: {WORST_UNIT[(op, site)]:.3f})" if (op, site) in WORST_UNIT \
                else ""
            print(f"  {op:20s} {site:18s} {v:.3f}{unit}")


def _audited(case, body):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(DEV)
    aud = Auditor(ops, case)
    t0 = time.perf_counter()
    out = body(aud)
    torch.cuda.synchronize()
    peak = max(aud.peak_bytes, torch.cuda.max_memory_allocated(DEV))
    RUNS[case] = (aud.calls, time.perf_counter() - t0, peak / 2 ** 30, aud.own_peak_bytes / 2 ** 30)
    for k, v in aud.worst.items():
        WORST[k] = max(WORST.get(k, 0.0), v)
    for k, v in aud.worst_unit.items():
        WORST_UNIT[k] = max(WORST_UNIT.get(k, 0.0), v)
    assert aud.calls > 0 and aud.unaudited == 0
    assert peak < 80 * 10 ** 9
    return aud, out


def _sites(aud):
    return {op for op, _ in aud.counts}


def test_sd_vae_decoder_256x344():
    """Every launch of the decode; then the same decode eagerly and from its CUDA graph (the auditor passing the
    launches through unchecked) equals the audited eager image bit for bit, and the graph captured exactly the
    audited operator calls and the eager decode's kernel launches (a warm-up and a capture pass)."""
    lat = torch.randn(1, 4, h, w, generator=torch.Generator().manual_seed(8)).to(DEV)

    def body(aud):
        eng = VaeDecoderEngine(SD_VAE, make_vae_state_dict(SD_VAE, 7), DEV, backend=aud)
        img = eng.decode_latents(lat, use_graph=False)
        return eng, img
    aud, (eng, eager) = _audited("sd_vae_decoder_256x344", body)
    assert {"conv_direct", "gemm", "groupnorm", "attention", "upsample2x", "image_out"} <= _sites(aud)
    aud.enabled = False
    n0 = ops.launch_count()
    again = eng.decode_latents(lat, use_graph=False)
    launches = ops.launch_count() - n0                  # kernel launches of one decode (GroupNorm: one or two)
    n0 = ops.launch_count()
    graphed = eng.decode_latents(lat, use_graph=True)
    assert ops.launch_count() - n0 == 2 * launches      # the warm-up and the captured pass
    assert aud.unaudited == 3 * aud.calls, (aud.unaudited, aud.calls)
    assert eager.shape == (1, 3, H, W) and torch.equal(again, eager) and torch.equal(graphed, eager)
    print(f"decoder: {aud.calls} operator calls audited = {launches} kernel launches; the graph captures the same")


def test_sd_vae_encoder_2048x2752():
    x = (torch.rand(1, 3, H, W, generator=torch.Generator().manual_seed(9)) * 2 - 1).to(DEV)

    def body(aud):
        eng = VaeEncoderEngine(SD_VAE, make_vae_state_dict(SD_VAE, 7, part="encoder"), DEV, backend=aud)
        return eng, eng.encode(x, use_graph=False).latent_dist.mean
    aud, (eng, eager) = _audited("sd_vae_encoder_2048x2752", body)
    assert {"conv_in", "gemm", "groupnorm", "attention", "conv_direct", "nhwc_to_nchw_f32"} <= _sites(aud)
    aud.enabled = False
    graphed = eng.encode(x, use_graph=True).latent_dist.mean
    assert aud.unaudited == 2 * aud.calls, (aud.unaudited, aud.calls)
    assert torch.equal(graphed, eager)


def test_sd15_tile_step_256x344(monkeypatch):
    """The tile pass's denoising engine: SD1.5 + one ControlNet in lockstep, one image with CFG (guidance 9), the
    hint stack on a 2048 x 2752 hint, the inpaint blend live (known / mask / noise) and two UniPC steps so that the
    multistep history is read.  Then the same two steps, replayed from the captured step graph, equal the same two
    steps run eagerly (both unaudited), which equal the audited ones, bit for bit."""
    _set_env(monkeypatch, "tiny_cn1")
    g = torch.Generator().manual_seed(11)
    ctx = torch.randn(2, 77, 768, generator=g)
    hint = torch.rand(1, 3, H, W, generator=g)
    lat0 = torch.randn(1, 4, h, w, generator=g)
    known = torch.randn(1, 4, h, w, generator=g)
    noise = torch.randn(1, 4, h, w, generator=g)
    mask = torch.zeros(1, 1, h, w)
    mask[..., h // 4:3 * h // 4, w // 4:3 * w // 4] = 1.0

    def run(eng, use_graph):
        eng.begin(lat0, guidance=9.0, known_nchw=known, mask_n1hw=mask, noise_nchw=noise, use_graph=use_graph)
        set_unipc(eng, 20)
        for _ in range(2):
            eng.step()
        return eng.latents()

    def body(aud):
        eng = DenoiseEngine(SD15, make_state_dict(SD15, "unet", 201), [make_state_dict(SD15, "controlnet", 202)], DEV,
                            backend=aud)
        assert [R.n for R in eng.runner.groups] == [2]
        eng.prepare(ctx, [torch.cat([hint, hint])], [1.0], cfg_duplicated=True)
        return eng, run(eng, False)
    aud, (eng, audited) = _audited("sd15_tile_step_256x344", body)
    assert {"conv_direct", "gemm", "groupnorm", "attention", "step_gather", "out_cfg_ddim"} <= _sites(aud)
    assert sum(n for (op, _), n in aud.counts.items() if op == "out_cfg_ddim") == 2
    aud.enabled = False
    eager = run(eng, False)
    graphed = run(eng, True)
    assert torch.equal(eager, audited), "the audited eager steps differ from the same steps unaudited"
    assert torch.equal(graphed, eager), float((graphed - eager).abs().max())
