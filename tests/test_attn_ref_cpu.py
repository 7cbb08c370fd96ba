"""The float64 attention reference of tests/test_gpu_attention.py, checked on the CPU against an explicit per-row loop;
the output of attention_bound against it, and the input generators and case table the GPU test runs."""
import math

import torch

from tests import attn_ref


def _loop(q, k, v, scale, rel_h, rel_w, rel_s):
    B, Nq, heads, d = q.shape
    Nkv = k.shape[1]
    out = torch.zeros(B, Nq, heads, d, dtype=torch.float64)
    for b in range(B):
        for h in range(heads):
            for i in range(Nq):
                logits = []
                for j in range(Nkv):
                    x = float((q[b, i, h] * k[b, j, h]).sum()) * scale
                    if rel_h is not None:
                        x += float(rel_h[b * heads + h, i, j // rel_s]) + float(rel_w[b * heads + h, i, j % rel_s])
                    logits.append(x)
                m = max(logits)
                w = [math.exp(x - m) for x in logits]
                tot = sum(w)
                for j in range(Nkv):
                    out[b, i, h] += w[j] / tot * v[b, j, h]
    return out


def test_attention_reference_matches_loop():
    g = torch.Generator().manual_seed(5)
    B, heads, Nq, Nkv, d, S = 2, 3, 5, 9, 4, 3
    q, k, v = (torch.randn(B, n, heads, d, generator=g, dtype=torch.float64) for n in (Nq, Nkv, Nkv))
    rel_h = torch.randn(B * heads, Nq, S, generator=g, dtype=torch.float64)
    rel_w = torch.randn(B * heads, Nq, S, generator=g, dtype=torch.float64)
    for rh, rw in ((None, None), (rel_h, rel_w)):
        got = attn_ref.attention(q, k, v, 0.7, rh, rw, S)
        assert torch.allclose(got, _loop(q, k, v, 0.7, rh, rw, S), rtol=1e-12, atol=1e-12)


def test_attention_bound_output_matches_reference():
    """attention_bound's o is attention()'s, also when its query-row chunks split a (batch, head); its bound is
    positive and at least the output rounding everywhere."""
    g = torch.Generator().manual_seed(6)
    B, heads, Nq, Nkv, d, S = 2, 3, 37, 23, 16, 5
    q, k, v = (torch.randn(B, n, heads, d, generator=g).half() for n in (Nq, Nkv, Nkv))
    rel_h = torch.randn(B * heads, Nq, S, generator=g)
    rel_w = torch.randn(B * heads, Nq, S, generator=g)
    for rh, rw in ((None, None), (rel_h, rel_w)):
        want = attn_ref.attention(q, k, v, 0.3, rh, rw, S)
        for chunk in (1 << 25, 5 * Nkv):
            o, bound = attn_ref.attention_bound(q, k, v, 0.3, rh, rw, S, chunk=chunk)
            assert torch.allclose(o, want, rtol=1e-12, atol=1e-12)
            assert bool((bound >= attn_ref.R.ulp(o, torch.float16)).all())


def test_inputs_are_seeded_and_shaped():
    for gen in attn_ref.GENERATORS:
        a = attn_ref.make_inputs(gen, 2, 3, 5, 9, 16, 0.25, rel_s=3, seed=1)
        b = attn_ref.make_inputs(gen, 2, 3, 5, 9, 16, 0.25, rel_s=3, seed=1)
        assert a["q"].shape == (2, 5, 3, 16) and a["k"].shape == a["v"].shape == (2, 9, 3, 16), gen
        assert a["rel_h"].shape == a["rel_w"].shape == (6, 5, 3), gen
        for key in a:
            assert torch.equal(a[key], b[key]), (gen, key)


def test_cases_cover_every_generator_and_keep_b_and_heads_above_one():
    gens = {c[0] for c in attn_ref.CASES.values()}
    assert gens == set(attn_ref.GENERATORS) - {"randn"}
    for name, (gen, B, heads, Nq, Nkv, d, scale, rel_s, layout) in attn_ref.CASES.items():
        assert B >= 2 and heads >= 2, name
        assert not rel_s or rel_s * rel_s >= Nkv, name
