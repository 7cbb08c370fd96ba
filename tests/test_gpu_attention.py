"""-m gpu: ea_attention against the float64 definition (tests/attn_ref.py) over every P V accumulator width and its
boundaries, with and without the rel-pos bias, the shapes the denoising step and SAM run, ragged edges, strided
q / k / v and a padded output row.  Gate: the one of tests/test_gpu_ops.py, max_abs < 2.5e-3 max(1, |ref|max) and
rel_fro < 1e-3.  Each case prints its error (pytest -s)."""
import pytest
import torch

from editanything_b200 import ops
from tests import attn_ref

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
CANARY = 7.0


def _run(B, heads, Nq, Nkv, d, *, bias=False, fused=False, pad=8, o_pad=8, seed=0):
    """One ea_attention call on seeded inputs; q / k / v rows padded by `pad` elements (or slices of one fused
    [B, N, 3 C] buffer), output rows by `o_pad`.  Returns (out [B, Nq, heads, d], reference, output buffer)."""
    dt = ops.half_dtype()
    g = torch.Generator(device=DEV).manual_seed(seed)
    C = heads * d
    if fused:
        assert Nq == Nkv
        buf = torch.randn(B, Nq, 3 * C, device=DEV, generator=g).to(dt)
        q, k, v = buf[..., :C], buf[..., C:2 * C], buf[..., 2 * C:]
        qs = ks = vs = (Nq * 3 * C, 3 * C)
    else:
        q = torch.randn(B, Nq, C + pad, device=DEV, generator=g).to(dt)[..., :C]
        k = torch.randn(B, Nkv, C + pad, device=DEV, generator=g).to(dt)[..., :C]
        v = torch.randn(B, Nkv, C + pad, device=DEV, generator=g).to(dt)[..., :C]
        qs, ks, vs = (Nq * (C + pad), C + pad), (Nkv * (C + pad), C + pad), (Nkv * (C + pad), C + pad)
    rel = {}
    if bias:
        S = 1
        while S * S < Nkv:
            S += 1
        rel = dict(rel_h=torch.randn(B * heads, Nq, S, device=DEV, generator=g),
                   rel_w=torch.randn(B * heads, Nq, S, device=DEV, generator=g), rel_s=S)
    o_ns = C + o_pad
    obuf = torch.full((B, Nq, o_ns), CANARY, device=DEV, dtype=dt)
    scale = d ** -0.5
    ops.attention(q, k, v, obuf, B=B, heads=heads, Nq=Nq, Nkv=Nkv, d=d, q_strides=qs, k_strides=ks, v_strides=vs,
                  o_strides=(Nq * o_ns, o_ns), scale=scale, **rel)
    torch.cuda.synchronize()
    shp = lambda t, n: t.reshape(B, n, heads, d)  # noqa: E731
    ref = attn_ref.attention(shp(q, Nq), shp(k, Nkv), shp(v, Nkv), scale, rel.get("rel_h"), rel.get("rel_w"),
                             rel.get("rel_s", 0))
    return shp(obuf[..., :C], Nq), ref, obuf


def _check(name, out, ref, obuf=None):
    C = ref.shape[2] * ref.shape[3]
    if obuf is not None and obuf.shape[-1] > C:
        assert bool((obuf[..., C:] == CANARY).all()), f"{name}: wrote past heads * d"
    err = (out.double() - ref).abs()
    max_abs = float(err.max())
    ref_max = float(ref.abs().max())
    rel_fro = float(torch.linalg.vector_norm(out.double() - ref) / torch.linalg.vector_norm(ref))
    print(f"ATTN_ERR {name} max_abs={max_abs:.3e} rel_fro={rel_fro:.3e} ref_max={ref_max:.3f}")
    assert torch.isfinite(out).all(), name
    assert max_abs < 2.5e-3 * max(1.0, ref_max), (name, max_abs, ref_max)
    assert rel_fro < 1e-3, (name, rel_fro)


# P V widths 48 / 64 / 80 / 160 / 192 and both sides of each boundary; Nq, Nkv ragged (3 key tiles)
@pytest.mark.parametrize("bias", [False, True])
@pytest.mark.parametrize("d", [8, 40, 48, 56, 64, 72, 80, 88, 136, 160, 168, 192])
def test_head_dims(d, bias):
    out, ref, obuf = _run(1, 2, 200, 300, d, bias=bias, seed=d)
    _check(f"d{d} bias={bias}", out, ref, obuf)


@pytest.mark.parametrize("case", [
    # name: B, heads, Nq, Nkv, d, bias, fused
    ("self64 fused B6", 6, 8, 4096, 4096, 40, False, True),
    ("cross64 77 keys", 2, 8, 4096, 77, 40, False, False),
    ("self32 d80", 2, 8, 1024, 1024, 80, False, True),
    ("self16 d160", 2, 8, 256, 256, 160, False, True),
    ("mid d160", 2, 8, 64, 64, 160, False, True),
    ("sam window", 25, 16, 196, 196, 80, True, False),
    ("sam global", 1, 16, 4096, 4096, 80, True, False),
], ids=lambda c: c[0])
def test_step_and_sam_shapes(case):
    name, B, heads, Nq, Nkv, d, bias, fused = case
    out, ref, obuf = _run(B, heads, Nq, Nkv, d, bias=bias, fused=fused, o_pad=0, seed=B + Nq)
    _check(name, out, ref, obuf)


@pytest.mark.parametrize("Nq,Nkv", [(100, 130), (300, 77), (130, 1), (40, 500), (1, 129), (63, 256)])
@pytest.mark.parametrize("d", [40, 160])
def test_ragged_edges(Nq, Nkv, d):
    out, ref, obuf = _run(2, 3, Nq, Nkv, d, pad=24, o_pad=40, seed=Nq * 7 + Nkv)
    _check(f"ragged Nq={Nq} Nkv={Nkv} d={d}", out, ref, obuf)


def test_canary_rows_and_columns():
    """Output rows of stride > heads * d: the padding columns and rows past Nq keep their contents."""
    B, heads, Nq, Nkv, d = 2, 2, 70, 150, 40
    out, ref, obuf = _run(B, heads, Nq, Nkv, d, o_pad=16, seed=3)
    _check("canary", out, ref, obuf)
    assert bool((obuf[..., heads * d:] == CANARY).all())


def test_deterministic():
    a = _run(2, 8, 1024, 1024, 40, fused=True, seed=9)[2].clone()
    b = _run(2, 8, 1024, 1024, 40, fused=True, seed=9)[2]
    assert torch.equal(a, b)
