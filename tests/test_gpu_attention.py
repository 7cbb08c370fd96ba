"""-m gpu: ea_attention against the float64 definition (tests/attn_ref.py) over every P V accumulator width and its
boundaries, with and without the rel-pos bias, the shapes the denoising step and SAM run, ragged edges, strided
q / k / v, batch gaps and padded output rows, on inputs that stress the softmax (attn_ref.make_inputs).
Gate, per element: |out - o| <= attn_ref.attention_bound (the kernel's rounding budget); and overall
rel_fro < 1e-3, which for zero-mean V under a flat softmax is tighter than any worst-case bound.  Each case prints
its worst error / bound (pytest -s), and the module prints the worst per generator."""
import math
import time

import numpy as np
import pytest
import torch

from editanything_b200 import ops
from tests import attn_ref

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
CANARY = 7.0
WORST = {}             # generator -> worst |err| / bound seen in this run


@pytest.fixture(scope="module", autouse=True)
def _report():
    t0 = time.perf_counter()
    yield
    if WORST:
        print(f"\nworst error / bound per generator ({time.perf_counter() - t0:.0f} s):")
        for g in sorted(WORST):
            print(f"  {g:12s} {WORST[g]:.3f}")


def _run(B, heads, Nq, Nkv, d, *, bias=False, fused=False, pad=8, o_pad=8, seed=0):
    """One ea_attention call on seeded inputs; q / k / v rows padded by `pad` elements (or slices of one fused
    [B, N, 3 C] buffer), output rows by `o_pad`.  Returns (out [B, Nq, heads, d], reference, bound, output buffer)."""
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
        S = attn_ref.rel_size(Nkv)
        rel = dict(rel_h=torch.randn(B * heads, Nq, S, device=DEV, generator=g),
                   rel_w=torch.randn(B * heads, Nq, S, device=DEV, generator=g), rel_s=S)
    o_ns = C + o_pad
    obuf = torch.full((B, Nq, o_ns), CANARY, device=DEV, dtype=dt)
    scale = d ** -0.5
    ops.attention(q, k, v, obuf, B=B, heads=heads, Nq=Nq, Nkv=Nkv, d=d, q_strides=qs, k_strides=ks, v_strides=vs,
                  o_strides=(Nq * o_ns, o_ns), scale=scale, **rel)
    torch.cuda.synchronize()
    shp = lambda t, n: t.reshape(B, n, heads, d)  # noqa: E731
    ref, bound = attn_ref.attention_bound(shp(q, Nq), shp(k, Nkv), shp(v, Nkv), scale, rel.get("rel_h"),
                                          rel.get("rel_w"), rel.get("rel_s", 0), dtype=dt)
    return shp(obuf[..., :C], Nq), ref, bound, obuf


def _check(name, gen, out, ref, bound, obuf=None, Nq=None):
    """Canary columns (and rows past Nq of a batch gap) intact, every element within its bound, rel_fro < 1e-3."""
    C = ref.shape[2] * ref.shape[3]
    if obuf is not None:
        if obuf.shape[-1] > C:
            assert bool((obuf[..., C:] == CANARY).all()), f"{name}: wrote past heads * d"
        if Nq is not None and obuf.shape[1] > Nq:
            assert bool((obuf[:, Nq:] == CANARY).all()), f"{name}: wrote into the gap between batch elements"
    assert bool(torch.isfinite(out).all()), name
    got = out.double()
    err = (got - ref).abs()
    ratio = err / bound
    i = int(torch.argmax(ratio.reshape(-1)))
    worst = float(ratio.reshape(-1)[i])
    rel_fro = float(torch.linalg.vector_norm(got - ref) / torch.linalg.vector_norm(ref))
    WORST[gen] = max(WORST.get(gen, 0.0), worst)
    print(f"ATTN_ERR {name} worst_ratio={worst:.3f} max_abs={float(err.max()):.3e} rel_fro={rel_fro:.3e}")
    if not worst <= 1.0:
        b, q, h, c = (int(x) for x in np.unravel_index(i, tuple(ref.shape)))
        n_bad = int((~(err <= bound)).sum())
        raise AssertionError(f"{name}: {n_bad} of {ref.numel()} elements out of bound; worst at (b={b}, q={q}, "
                             f"head={h}, c={c}): got {float(got[b, q, h, c])!r}, ref {float(ref[b, q, h, c])!r}, "
                             f"bound {float(bound[b, q, h, c]):.3e}, ratio {worst:.3g}")
    assert rel_fro < 1e-3, (name, rel_fro)


# P V widths 48 / 64 / 80 / 160 / 192 and both sides of each boundary; Nq, Nkv ragged (3 key tiles)
@pytest.mark.parametrize("bias", [False, True])
@pytest.mark.parametrize("d", [8, 40, 48, 56, 64, 72, 80, 88, 136, 160, 168, 192])
def test_head_dims(d, bias):
    out, ref, bound, obuf = _run(1, 2, 200, 300, d, bias=bias, seed=d)
    _check(f"d{d} bias={bias}", "randn", out, ref, bound, obuf)


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
    out, ref, bound, obuf = _run(B, heads, Nq, Nkv, d, bias=bias, fused=fused, o_pad=0, seed=B + Nq)
    _check(name, "randn", out, ref, bound, obuf)


@pytest.mark.parametrize("Nq,Nkv", [(100, 130), (300, 77), (130, 1), (40, 500), (1, 129), (63, 256)])
@pytest.mark.parametrize("d", [40, 160])
def test_ragged_edges(Nq, Nkv, d):
    out, ref, bound, obuf = _run(2, 3, Nq, Nkv, d, pad=24, o_pad=40, seed=Nq * 7 + Nkv)
    _check(f"ragged Nq={Nq} Nkv={Nkv} d={d}", "randn", out, ref, bound, obuf)


def test_canary_rows_and_columns():
    """Output rows of stride > heads * d: the padding columns and rows past Nq keep their contents."""
    B, heads, Nq, Nkv, d = 2, 2, 70, 150, 40
    out, ref, bound, obuf = _run(B, heads, Nq, Nkv, d, o_pad=16, seed=3)
    _check("canary", "randn", out, ref, bound, obuf)
    assert bool((obuf[..., heads * d:] == CANARY).all())


def test_deterministic():
    a = _run(2, 8, 1024, 1024, 40, fused=True, seed=9)[3].clone()
    b = _run(2, 8, 1024, 1024, 40, fused=True, seed=9)[3]
    assert torch.equal(a, b)


# ---- generated inputs over attn_ref.CASES ------------------------------------------------------------------------
def _buffer(parts, B, rows, cols):
    """[B, rows, cols] NaN-filled buffer with each [B, n, C] part at its column offset: a read of a padding column
    or a gap row turns the output into NaN."""
    buf = torch.full((B, rows, cols), math.nan, device=DEV, dtype=parts[0][0].dtype)
    for x, col in parts:
        buf[:, :x.shape[1], col:col + x.shape[2]] = x
    return buf


@pytest.mark.parametrize("name", list(attn_ref.CASES))
def test_generated_case(name):
    gen, B, heads, Nq, Nkv, d, scale, rel_s, layout = attn_ref.CASES[name]
    scale = d ** -0.5 if scale is None else scale
    dt = ops.half_dtype()
    inp = attn_ref.make_inputs(gen, B, heads, Nq, Nkv, d, scale, rel_s, seed=len(name), device=DEV, dtype=dt)
    C = heads * d
    q, k, v = (inp[n].reshape(B, -1, C) for n in ("q", "k", "v"))
    gap = 5 if layout == "gap" else 0
    if layout == "fused":
        buf = _buffer([(q, 0), (k, C), (v, 2 * C)], B, Nq, 3 * C)
        qp, kp, vp = buf, buf[..., C:], buf[..., 2 * C:]
        qs = ks = vs = (Nq * 3 * C, 3 * C)
    elif layout == "kv":
        qp = _buffer([(q, 0)], B, Nq, C + 8)
        kp = _buffer([(k, 0), (v, C)], B, Nkv, 2 * C)
        vp = kp[..., C:]
        qs, ks = (Nq * (C + 8), C + 8), (Nkv * 2 * C, 2 * C)
        vs = ks
    else:
        qp = _buffer([(q, 0)], B, Nq + gap, C + 8)
        kp = _buffer([(k, 0)], B, Nkv + gap, C + 8)
        vp = _buffer([(v, 0)], B, Nkv + gap, C + 8)
        qs, ks, vs = (((n + gap) * (C + 8), C + 8) for n in (Nq, Nkv, Nkv))
    o_rows, o_ns = Nq + gap, C + 8
    obuf = torch.full((B, o_rows, o_ns), CANARY, device=DEV, dtype=dt)
    rel = dict(rel_h=inp["rel_h"], rel_w=inp["rel_w"], rel_s=rel_s) if rel_s else {}
    ops.attention(qp, kp, vp, obuf, B=B, heads=heads, Nq=Nq, Nkv=Nkv, d=d, q_strides=qs, k_strides=ks,
                  v_strides=vs, o_strides=(o_rows * o_ns, o_ns), scale=scale, **rel)
    torch.cuda.synchronize()
    ref, bound = attn_ref.attention_bound(inp["q"], inp["k"], inp["v"], scale, inp["rel_h"], inp["rel_w"], rel_s,
                                          dtype=dt)
    out = obuf[:, :Nq, :C].reshape(B, Nq, heads, d)
    _check(name, gen, out, ref, bound, obuf, Nq)
