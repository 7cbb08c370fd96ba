"""ea_gemm_plan (no GPU needed): invariants of the launch planner over the GEMM shapes of the
BASELINE.json configs (SD1.5 512x512 / 1024x1024, SD2.1 768x768 N=4, SAM ViT-H, the VAE): tile widths the
planner may pick (32 / 64 / 128: the kernel's register budget), one CTA per SM, stage rings that fit the 216 KB
ring of the kernel's shared memory, split-K grids that are fully resident (the spinning fix-up waits for sibling
CTAs), GEGLU tiles of exactly 128 columns."""
import ctypes as C
import itertools

from editanything_b200 import _lib

WS = 48 * 1024 * 1024 + 65536
N_SM = 132
RING = 216 * 1024      # GEMM_SMEM_RING of ea_gemm.cu


def _plan(mt, N, kb, act=0, ws=WS):
    lib = _lib.load()
    out = (C.c_int * 5)()
    assert lib.ea_gemm_plan(mt, N, kb, act, ws, N_SM, out) == 0
    bn, stages, splits, kbps, occ_two = list(out)
    return bn, stages, splits, kbps, occ_two % 10, occ_two // 10


def _shapes():
    ms = [128, 512, 2048, 8192, 32768, 4608 * 4, 262144, 25 * 196, 4096]      # rows: 8x8 ... 512x512, SAM windows/global
    ns = [8, 256, 320, 640, 960, 1280, 1920, 2560, 3840, 5120, 10240]
    kbs = [1, 5, 10, 20, 40, 45, 80, 90, 135, 180, 270, 360, 540]
    return itertools.product(ms, ns, kbs)


def test_plans_are_launchable():
    for M, N, kb in _shapes():
        mt = (M + 127) // 128
        bn, stages, splits, kbps, occ, two = _plan(mt, N, kb)
        assert bn in (32, 64, 128), (M, N, kb, bn)
        assert bn == 32 or N > bn - 32, "a narrower tile would cover N"
        assert 2 <= stages <= 8 and occ == 1 and two == 0
        stage_bytes = 128 * 128 + bn * 128
        assert stages * stage_bytes <= RING, (M, N, kb, bn, stages)
        assert stages <= max(kb, 2), "no more stages than K-blocks"
        assert splits >= 1 and kbps * splits >= kb and kbps * (splits - 1) < kb, (kb, splits, kbps)
        if splits > 1:
            tiles = mt * ((N + bn - 1) // bn)
            assert tiles * splits <= occ * N_SM, ("split CTAs must all be resident", M, N, kb, bn, splits, occ)
            assert tiles * splits * 128 * bn * 4 <= WS - 65536, "partial tiles must fit the workspace"
            assert kbps >= 4, "a split owns at least 4 K-blocks"


def test_geglu_tiles_are_128_wide():
    for M, N, kb in [(8192, 2560, 5), (2048, 5120, 10), (512, 10240, 20), (128, 10240, 20), (4608 * 4, 2560, 5)]:
        bn, *_ = _plan((M + 127) // 128, N, kb, act=_lib.EA_ACT_GEGLU)
        assert bn == 128


def test_no_workspace_means_no_split():
    for mt, N, kb in [(1, 1280, 180), (4, 1280, 360), (1, 1280, 540)]:
        assert _plan(mt, N, kb, ws=0)[2] == 1
        assert _plan(mt, N, kb)[2] > 1        # the weight-streaming 8x8 / 16x16 layers do split with one


def test_bad_arguments_are_rejected():
    lib = _lib.load()
    out = (C.c_int * 5)()
    assert lib.ea_gemm_plan(0, 320, 5, 0, WS, N_SM, out) != 0
    assert lib.ea_gemm_plan(4, 320, 0, 0, WS, N_SM, out) != 0
    assert lib.ea_gemm_plan(4, 320, 5, 0, WS, N_SM, None) != 0
