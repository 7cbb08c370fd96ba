"""-m gpu: ea_attention with heads wider than 192 (the VAE AttnBlock's one head of d = 512) against the float64
definition (tests/attn_ref.py): head dims on both sides of the 192 boundary, heads and batches, ragged query and
key counts against the 64-row query tile and the 32-key K / V tile, the adversarial softmax inputs of
attn_ref.make_inputs, q / k / v as slices of one [B N, 3 d] buffer (how the VAE feeds them), padded output rows with
canaries, the shape check past d = 512, determinism, and the VAE's sequence lengths up to 88064 tokens.
Gate, per element: |out - o| <= the attn_ref.attention_bound of the kernel's arithmetic, counted over the wide
kernel's 32-key tiles; and overall rel_fro < 1e-3."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from editanything_b200 import _lib as L
from editanything_b200 import ops
from tests import attn_ref

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
CANARY = 7.0
EA_ERR_SHAPE = -2
WIDE_TILE = 32            # keys per K / V tile of the d > 192 kernel


def _bound(q, k, v, scale, dtype):
    """attention_bound with the tile count of the kernel that runs d: attn_ref counts 64-key sub-tiles above d = 80,
    the d > 192 kernel takes 32 keys per tile.  Every extra tile adds one ex2 rescale (EX2_REL, a logit shift times
    sum_k P_k |v_k| + |o|) and one more rounding of O and l (2 u sum_k P_k |v_k| + u |o|); sum_k P_k |v_k| and |o|
    are at most max_k |v_k| per column."""
    o, bound = attn_ref.attention_bound(q, k, v, scale, dtype=dtype)
    d, Nkv = q.shape[3], k.shape[1]
    if d > 192:
        extra = -(-Nkv // WIDE_TILE) - -(-Nkv // attn_ref.sub_tile(d))
        vmax = v.double().abs().amax(dim=1, keepdim=True)                   # [B, 1, heads, d]
        bound = bound + extra * (2 * attn_ref.EX2_REL + 3 * attn_ref.U) * vmax
    return o, bound


def _launch(q, k, v, obuf, B, heads, Nq, Nkv, d, qs, ks, vs, os_, scale):
    ops.attention(q, k, v, obuf, B=B, heads=heads, Nq=Nq, Nkv=Nkv, d=d, q_strides=qs, k_strides=ks, v_strides=vs,
                  o_strides=os_, scale=scale)
    torch.cuda.synchronize()


def _run(B, heads, Nq, Nkv, d, *, gen="randn", scale=None, fused=False, pad=8, o_pad=8, gap=0, seed=0):
    """One ea_attention call on attn_ref.make_inputs(gen); q / k / v rows padded by `pad` elements (or slices of one
    [B, N, 3 heads d] buffer), output rows padded by `o_pad` columns and batch elements `gap` rows apart past Nq, all
    padding holding CANARY.  Returns (out [B, Nq, heads, d], q, k, v [B, n, heads, d], scale, output buffer)."""
    dt = ops.half_dtype()
    scale = d ** -0.5 if scale is None else scale
    x = attn_ref.make_inputs(gen, B, heads, Nq, Nkv, d, scale, seed=seed, device=DEV, dtype=dt)
    C_ = heads * d
    if fused:
        assert Nq == Nkv
        buf = torch.cat([x[n].reshape(B, Nq, C_) for n in "qkv"], -1).contiguous()
        q, k, v = buf[..., :C_], buf[..., C_:2 * C_], buf[..., 2 * C_:]
        qs = ks = vs = (Nq * 3 * C_, 3 * C_)
    else:
        def padded(t, n):
            p = torch.full((B, n, C_ + pad), math.nan, device=DEV, dtype=dt)
            p[..., :C_] = t.reshape(B, n, C_)
            return p[..., :C_]
        q, k, v = padded(x["q"], Nq), padded(x["k"], Nkv), padded(x["v"], Nkv)
        qs, ks, vs = (Nq * (C_ + pad), C_ + pad), (Nkv * (C_ + pad), C_ + pad), (Nkv * (C_ + pad), C_ + pad)
    o_ns = C_ + o_pad
    obuf = torch.full((B, Nq + gap, o_ns), CANARY, device=DEV, dtype=dt)
    _launch(q, k, v, obuf, B, heads, Nq, Nkv, d, qs, ks, vs, ((Nq + gap) * o_ns, o_ns), scale)
    shp = lambda t, n: t.reshape(B, n, heads, d)  # noqa: E731
    return shp(obuf[:, :Nq, :C_], Nq), x["q"], x["k"], x["v"], scale, obuf


def _check(name, out, q, k, v, scale, obuf=None, rows=None):
    """Canaries intact; every element within its bound; rel_fro < 1e-3.  rows: check only these query rows."""
    heads, d = q.shape[2], q.shape[3]
    C_, Nq = heads * d, q.shape[1]
    if obuf is not None:
        if obuf.shape[-1] > C_:
            assert bool((obuf[..., C_:] == CANARY).all()), f"{name}: wrote past heads * d"
        if obuf.shape[1] > Nq:
            assert bool((obuf[:, Nq:] == CANARY).all()), f"{name}: wrote into the rows past Nq"
    if rows is not None:
        out, q = out[:, rows], q[:, rows]
    assert bool(torch.isfinite(out).all()), name
    ref, bound = _bound(q, k, v, scale, out.dtype)
    got = out.double()
    err = (got - ref).abs()
    ratio = err / bound
    i = int(torch.argmax(ratio.reshape(-1)))
    worst = float(ratio.reshape(-1)[i])
    rel_fro = float(torch.linalg.vector_norm(got - ref) / torch.linalg.vector_norm(ref))
    print(f"ATTN_ERR {name} worst_ratio={worst:.3f} max_abs={float(err.max()):.3e} rel_fro={rel_fro:.3e}")
    if not worst <= 1.0:
        b, r, h, c = (int(x) for x in np.unravel_index(i, tuple(ref.shape)))
        n_bad = int((~(err <= bound)).sum())
        raise AssertionError(f"{name}: {n_bad} of {ref.numel()} elements out of bound; worst at (b={b}, q={r}, "
                             f"head={h}, c={c}): got {float(got[b, r, h, c])!r}, ref {float(ref[b, r, h, c])!r}, "
                             f"bound {float(bound[b, r, h, c]):.3e}, ratio {worst:.3g}")
    assert rel_fro < 1e-3, (name, rel_fro)


# d = 192 is the last width of the narrow kernels, 200 the first of the wide one (a partial 64-column Q / K box and a
# partial 16-column V box), 256 warp-group 1's columns wholly past d, 504 / 512 the widest
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("heads", [1, 2])
@pytest.mark.parametrize("d", [192, 200, 256, 504, 512])
def test_head_dims(d, heads, B):
    out, q, k, v, scale, obuf = _run(B, heads, 129, 300, d, gen="distinct", seed=d + heads + B)
    _check(f"d{d} heads{heads} B{B}", out, q, k, v, scale, obuf)


# ragged against the 64-row query tile and the 32-key tile; 4100 keys = 128 full tiles and 4 keys
@pytest.mark.parametrize("n", [1, 31, 33, 63, 65, 129, 4100])
@pytest.mark.parametrize("d", [200, 512])
def test_ragged_keys(n, d):
    out, q, k, v, scale, obuf = _run(2, 1, 70, n, d, gen="flat-offset", seed=n)
    _check(f"keys{n} d{d}", out, q, k, v, scale, obuf)


@pytest.mark.parametrize("n", [1, 31, 33, 63, 65, 129, 4100])
@pytest.mark.parametrize("d", [200, 512])
def test_ragged_queries(n, d):
    out, q, k, v, scale, obuf = _run(2, 1, n, 97, d, gen="distinct", gap=5, seed=n + 1)
    _check(f"queries{n} d{d}", out, q, k, v, scale, obuf)


# a dominant logit (peaked), constant rows (ties), a max that rises on every tile or sits in the first one, and
# large-magnitude logits (scale 3: logits of spread ~70)
@pytest.mark.parametrize("gen,scale", [("peaked", None), ("ties", None), ("rising", None), ("early", None),
                                       ("flat-offset", None), ("randn", 3.0), ("peaked", 3.0)])
@pytest.mark.parametrize("d", [256, 512])
def test_adversarial_softmax(gen, scale, d):
    out, q, k, v, s, obuf = _run(2, 1, 130, 400, d, gen=gen, scale=scale, seed=11)
    _check(f"{gen} d{d} scale{scale}", out, q, k, v, s, obuf)


def test_vae_layout_and_canaries():
    """q / k / v as column slices of one [B N, 3 * 512] buffer, output rows of stride 512 + 64 with batch elements
    16 rows apart past Nq: the padding columns and rows keep their canaries."""
    out, q, k, v, scale, obuf = _run(3, 1, 1000, 1000, 512, gen="flat-offset", fused=True, o_pad=64, gap=16, seed=5)
    _check("vae layout", out, q, k, v, scale, obuf)


def test_shape_limit():
    """d = 520 (and the rel-pos bias above d = 192) is EA_ERR_SHAPE, before any launch."""
    dt = ops.half_dtype()
    x = torch.zeros(2, 64, 520, device=DEV, dtype=dt)
    o = torch.full((2, 64, 520), CANARY, device=DEV, dtype=dt)
    a = L.AttnArgs()
    a.q = a.k = a.v = x.data_ptr()
    a.out = o.data_ptr()
    a.B, a.heads, a.Nq, a.Nkv, a.d = 2, 1, 64, 64, 520
    a.q_bs = a.k_bs = a.v_bs = a.o_bs = 64 * 520
    a.q_ns = a.k_ns = a.v_ns = a.o_ns = 520
    a.scale = 0.05
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    assert L.lib().ea_attention(C.byref(a), stream) == EA_ERR_SHAPE
    a.d = 512
    rel = torch.zeros(2, 64, 8, device=DEV)
    a.rel_h = a.rel_w = rel.data_ptr()
    a.rel_s = 8
    assert L.lib().ea_attention(C.byref(a), stream) == EA_ERR_SHAPE
    torch.cuda.synchronize()
    assert bool((o == CANARY).all())


def test_deterministic():
    a = _run(2, 1, 4100, 4100, 512, fused=True, seed=9)[5].clone()
    b = _run(2, 1, 4100, 4100, 512, fused=True, seed=9)[5]
    assert torch.equal(a, b)


# the SD VAE's mid-block attention: 64 x 64 latents (512 px), 128 x 128 (1024 px) in full; 256 x 344 (2048 x 2752 px)
# on its first, middle and last 64-row query tiles against all keys
@pytest.mark.parametrize("N", [4096, 16384])
def test_vae_sizes(N):
    out, q, k, v, scale, obuf = _run(1, 1, N, N, 512, fused=True, o_pad=0, seed=N)
    _check(f"vae N{N}", out, q, k, v, scale, obuf)


def test_vae_2048x2752_sampled_rows():
    N = 256 * 344
    out, q, k, v, scale, obuf = _run(1, 1, N, N, 512, fused=True, o_pad=0, seed=3)
    mid = (N // 64 // 2) * 64
    rows = torch.cat([torch.arange(0, 64), torch.arange(mid, mid + 64), torch.arange(N - 64, N)]).to(DEV)
    _check("vae N88064 sampled", out, q, k, v, scale, obuf, rows=rows)
