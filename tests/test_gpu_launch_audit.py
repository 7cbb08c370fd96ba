"""-m gpu: every launch of the denoising step, the SAM encoder and the VAE, audited on its production arguments by
tests/launch_audit.py: each call checked against float64 on its own inputs with the per-element bound of its kernel's
suite, its stores confined to the operands the C ABI declares, and a fenced re-run (NaN everywhere outside the declared
read extents, NaN margins around every storage) bit-identical to the production run.

The full-size cases (SD1.5 512^2 and SD2.1 768^2 steps, SAM ViT-H, the SD VAE) reach what the tiny configurations
cannot: 64^2 / 96^2 attention, the planner's production tile choices, the uncached GroupNorm path, the VAE's N = 4096
fp32 logits GEMM, the 64 -> 70 padded SAM windows.  All runs are eager (no CUDA graph): graph replay against eager is checked bit for bit in test_gpu_nocfg /
test_gpu_vpred.  The module prints, per case, the number of audited launches, the wall time and the peak device
memory, and the worst error / bound per (op, call site) over all cases."""
import time

import pytest
import torch

from editanything_b200 import ops
from editanything_b200.denoise import DenoiseEngine
from editanything_b200.sam import SamEncoderEngine
from editanything_b200.denoise import ddim_schedule
from editanything_b200.sam_spec import SAM_TINY, SAM_VIT_H, make_sam_state_dict
from editanything_b200.unet_spec import SD15, SD21, TINY, TINY21, make_state_dict
from editanything_b200.vae import SD_VAE, VAE_TINY, VaeDecoderEngine, VaeEncoderEngine, make_vae_state_dict
from oracle.inputs import make_inputs
from oracle.make_golden_sam import make_image as sam_image
from oracle.make_golden_vae import make_image as vae_image
from tests.launch_audit import Auditor, denoise_engine, run_trace_case, set_unipc
from tests.test_step_trace_cpu import CASES, _set_env

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
WORST = {}          # (op, call site) -> worst error / bound over every case
WORST_UNIT = {}     # GroupNorm (op, call site) -> the same without the derived statistics term
RUNS = {}           # case -> (audited launches, seconds, peak GiB, the auditor's own peak GiB)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if RUNS:
        print("\naudited launches, wall time, peak device memory and the auditor's own largest growth in one call, "
              "per case:")
        for k, (n, s, m, own) in RUNS.items():
            print(f"  {k:32s} {n:5d} launches  {s:7.1f} s  {m:6.2f} GiB  auditor {own:6.2f} GiB")
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
    body(aud)
    torch.cuda.synchronize()
    peak = max(aud.peak_bytes, torch.cuda.max_memory_allocated(DEV))      # the auditor resets the peak per call
    RUNS[case] = (aud.calls, time.perf_counter() - t0, peak / 2 ** 30, aud.own_peak_bytes / 2 ** 30)
    for k, v in aud.worst.items():
        WORST[k] = max(WORST.get(k, 0.0), v)
    for k, v in aud.worst_unit.items():
        WORST_UNIT[k] = max(WORST_UNIT.get(k, 0.0), v)
    assert aud.calls > 0
    return aud


# ---- DenoiseEngine at reduced width ---------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(CASES))
def test_denoise_step_trace_cases(name, monkeypatch):
    """prepare (hint stack, context K/V, embeddings), three UniPC steps (the multistep history live) and one eps() of
    every step-trace case; with three or four ControlNets the encoder runs as two groups of grouped launches."""
    _set_env(monkeypatch, name)

    def body(aud):
        eng, *inputs = denoise_engine(name, aud, DEV)
        run_trace_case(eng, *inputs, unipc_steps=3)
    _audited(name, body)


def _engine(aud, cfg, n_cn):
    usd = make_state_dict(cfg, "unet", 61)
    csds = [make_state_dict(cfg, "controlnet", 62 + i) for i in range(n_cn)]
    return DenoiseEngine(cfg, usd, csds, DEV, backend=aud)


@pytest.mark.parametrize("N", [1, 3])
def test_denoise_unguided(N, monkeypatch):
    """Sampling without guidance: the networks on the N images alone (odd image counts reach the partial last image
    block of the 8x8 convolutions), the update through ea_out_ddim."""
    _set_env(monkeypatch, "tiny_cn1")

    def body(aud):
        eng = _engine(aud, TINY, 1)
        x, ctx, hints = make_inputs(TINY, N, 8, 7, 5, n_controlnets=1)
        eng.prepare(ctx, hints, [0.8], guided=False)
        eng.begin(x[:, :4], guidance=1.0, use_graph=False)
        set_unipc(eng, 20)
        for _ in range(3):
            eng.step()
        eng.eps(x, 500)
    _audited(f"unguided_N{N}", body)


def test_denoise_vpred(monkeypatch):
    _set_env(monkeypatch, "tiny_cn1")

    def body(aud):
        eng = _engine(aud, TINY21, 1)
        x, ctx, hints = make_inputs(TINY21, 2, 8, 7, 5, n_controlnets=1)
        eng.prepare(ctx, hints, [0.9])
        eng.begin(x[:1, :4], guidance=7.5, use_graph=False)
        set_unipc(eng, 20, prediction_type="v_prediction")
        for _ in range(3):
            eng.step()
    _audited("vpred_tiny21_cn1", body)


# ---- SAM and VAE ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [1, 3])
def test_sam_tiny_encode(B):
    def body(aud):
        eng = SamEncoderEngine(SAM_TINY, make_sam_state_dict(SAM_TINY, 5), DEV, backend=aud)
        eng._encode_eager(sam_image(SAM_TINY, B, 7).to(DEV))
    _audited(f"sam_tiny_B{B}", body)


def test_vae_tiny_decode_and_encode():
    """B = 3 at sides that are not powers of two: 4x6 latents, a 24x24 image."""
    def dec(aud):
        eng = VaeDecoderEngine(VAE_TINY, make_vae_state_dict(VAE_TINY, 7), DEV, backend=aud)
        eng.decode_latents(torch.randn(3, 4, 4, 6, generator=torch.Generator().manual_seed(8)), use_graph=False)

    def enc(aud):
        eng = VaeEncoderEngine(VAE_TINY, make_vae_state_dict(VAE_TINY, 7, part="encoder"), DEV, backend=aud)
        eng.encode(vae_image(3, 24, 9), use_graph=False)
    _audited("vae_tiny_decoder_B3", dec)
    _audited("vae_tiny_encoder_B3", enc)


# ---- full size ------------------------------------------------------------------------------------------------
def _one_step(eng, x, guided=True):
    n = x.shape[0] // 2 if guided else x.shape[0]
    eng.begin(x[:n, :4], guidance=7.5, use_graph=False)
    ts, a, ap = ddim_schedule(50)
    eng.step(int(ts[2]), float(a[2]), float(ap[2]))


def test_sd15_512_one_image_cfg_two_controlnets_lockstep(monkeypatch):
    """prepare and one step of SD1.5 at 512^2: one image + CFG, the UNet encoder and 2 ControlNets in lockstep."""
    _set_env(monkeypatch, "tiny_cn2")

    def body(aud):
        eng = _engine(aud, SD15, 2)
        x, ctx, hints = make_inputs(SD15, 2, 64, 77, 5, n_controlnets=2)
        eng.prepare(ctx, hints, [0.5, 1.0])
        _one_step(eng, x)
    _audited("sd15_512_cfg_cn2_lockstep", body)


def test_sd21_768_four_images_cfg_one_controlnet(monkeypatch):
    """prepare and one step of SD2.1 at 768^2: four images + CFG (eight network rows), one ControlNet in lockstep."""
    _set_env(monkeypatch, "tiny_cn1")

    def body(aud):
        eng = _engine(aud, SD21, 1)
        x, ctx, hints = make_inputs(SD21, 8, 96, 77, 5, n_controlnets=1)
        eng.prepare(ctx, hints, [1.0])
        _one_step(eng, x)
    _audited("sd21_768_n4_cfg_cn1", body)


def test_sam_vit_h_patch_embed_blocks_0_7_and_neck():
    """ViT-H at B = 1 through the engine's own encode: the patch embedding, block 0 (windowed: the 64 grid padded to
    70 for ws 14), block 7 (global attention) and the neck are audited; the other 30 blocks run unchecked."""
    def body(aud):
        eng = SamEncoderEngine(SAM_VIT_H, make_sam_state_dict(SAM_VIT_H, 5), DEV, backend=aud)
        block = eng._block

        def audited_block(i, x, B):
            aud.enabled = i in (0, 7)
            try:
                return block(i, x, B)
            finally:
                aud.enabled = True
        eng._block = audited_block
        eng._encode_eager(sam_image(SAM_VIT_H, 1, 7).to(DEV))
        assert 0 not in SAM_VIT_H.global_attn_indexes and SAM_VIT_H.window_size == 14
        assert 7 in SAM_VIT_H.global_attn_indexes
    _audited("sam_vit_h_B1_pe_b0_b7_neck", body)


def test_sd_vae_decoder_64_and_encoder_512():
    """The SD VAE decoder at 64x64 latents (512^2 levels: the uncached GroupNorm path; the AttnBlock's
    4096 x 4096 fp32 logits with lda = ldw = 2c) and the encoder at 512^2, B = 1."""
    def dec(aud):
        eng = VaeDecoderEngine(SD_VAE, make_vae_state_dict(SD_VAE, 7), DEV, backend=aud)
        eng.decode_latents(torch.randn(1, 4, 64, 64, generator=torch.Generator().manual_seed(8)), use_graph=False)

    def enc(aud):
        eng = VaeEncoderEngine(SD_VAE, make_vae_state_dict(SD_VAE, 7, part="encoder"), DEV, backend=aud)
        eng.encode(vae_image(1, 512, 9), use_graph=False)
    _audited("sd_vae_decoder_64", dec)
    _audited("sd_vae_encoder_512", enc)
