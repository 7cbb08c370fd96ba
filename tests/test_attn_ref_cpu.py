"""The float64 attention reference of tests/test_gpu_attention.py, checked on the CPU against an explicit per-row loop."""
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
