"""-m gpu: the persistent GEMM variant (ea_gemm_args.force_persistent = 1 | 2: one CTA per SM walks the tile list)
against the one-tile-per-CTA kernel on the same inputs.  Both compute every output element with the same K order in
fp32, so the results
must agree to the last bit; grids are chosen to give every CTA several tiles (the ring's barrier
phase wrap-around) and a ragged last wave."""
import pytest
import torch

from editanything_b200 import _lib as L
from editanything_b200 import ops

pytestmark = pytest.mark.gpu


def _pair(fn):
    a = fn(0)
    b = fn(1)
    torch.cuda.synchronize()
    return a, b


@pytest.mark.parametrize("variant", [1, 2])
@pytest.mark.parametrize("M,N,K,res,act", [
    (8192, 2560, 320, False, "geglu"),      # 1280 tiles: ~9 per CTA
    (8192, 960, 320, False, "none"),        # qkv at 64x64
    (8192, 320, 1280, True, "none"),        # ff2 with residual
    (19000, 640, 192, True, "gelu"),        # ragged M, ragged last wave
    (300, 2048, 64, False, "none"),         # one K-block per tile
    (8192, 320, 320, True, "none"),         # one wave, 96/160-wide tiles: odd number of 32-column chunks
    (2048, 64, 640, False, "none"),         # tile narrower than one 64-column group: the 2nd warp-group idles
])
def test_linear_matches_one_tile_kernel(M, N, K, res, act, variant):
    dev = torch.device("cuda:0")
    dt = ops.half_dtype()
    g = torch.Generator(device=dev).manual_seed(M + N + K)
    x = torch.randn(M, K, device=dev, generator=g).to(dt)
    w = (torch.randn(N, K, device=dev, generator=g) / K ** 0.5).to(dt)
    b = torch.randn(N, device=dev, generator=g)
    n_out = N // 2 if act == "geglu" else N
    r = torch.randn(M, n_out, device=dev, generator=g).to(dt) if res else None
    code = {"none": L.EA_ACT_NONE, "gelu": L.EA_ACT_GELU, "geglu": L.EA_ACT_GEGLU}[act]

    def run(persist):
        out = torch.full((M, n_out), 7.0, device=dev, dtype=dt)
        ops.gemm(x, w, out, bias=b, residual=r, act=code, force_persistent=variant if persist else -1, force_2cta=-1,
                 force_splits=1)
        return out
    ref, got = _pair(run)
    assert torch.equal(ref, got), float((ref.float() - got.float()).abs().max())


@pytest.mark.parametrize("variant", [1, 2])
@pytest.mark.parametrize("B,H,W,cin,cout,mode,extra", [
    (2, 64, 64, 320, 320, "s1", 0),
    (8, 96, 96, 320, 320, "s1", 0),        # SD2.1 768x768 N=4: 576 M-tiles
    (1, 512, 512, 128, 128, "s1", 0),      # VAE top level: 2048 M-tiles
    (2, 64, 64, 640, 320, "s1", 320),      # fused 1x1 skip as extra K columns
    (2, 32, 32, 320, 320, "s2", 0),
    (1, 128, 128, 128, 128, "s2a", 0),
])
def test_conv_matches_one_tile_kernel(B, H, W, cin, cout, mode, extra, variant):
    dev = torch.device("cuda:0")
    dt = ops.half_dtype()
    g = torch.Generator(device=dev).manual_seed(B * H + cin)
    s = 1 if mode == "s1" else 2
    x = torch.randn(B, H * s, W * s, cin, device=dev, generator=g).to(dt)
    w = (torch.randn(cout, 9 * cin + extra, device=dev, generator=g) / (9 * cin) ** 0.5).to(dt)
    b = torch.randn(cout, device=dev, generator=g)
    rv = torch.randn(B, cout, device=dev, generator=g)
    xe = torch.randn(B, H, W, extra, device=dev, generator=g).to(dt) if extra else None
    m = {"s1": L.EA_GEMM_CONV_S1, "s2": L.EA_GEMM_CONV_S2, "s2a": L.EA_GEMM_CONV_S2A}[mode]

    def run(persist):
        out = torch.full((B * H * W, cout), 7.0, device=dev, dtype=dt)
        ops.gemm(x, w, out, mode=m, conv=(B, H, W, cin), bias=b, rowvec=rv, a_extra=xe,
                 ld_extra=extra, force_persistent=variant if persist else -1, force_2cta=-1, force_splits=1)
        return out
    ref, got = _pair(run)
    assert torch.equal(ref, got), float((ref.float() - got.float()).abs().max())
