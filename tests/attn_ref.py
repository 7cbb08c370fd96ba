"""Float64 reference of ea_attention written from its definition (include/editanything_b200.h):
out = softmax(Q K^T * scale + bias) V with bias[q, kk] = rel_h[q, kk // rel_s] + rel_w[q, kk % rel_s]."""
import torch


def attention(q, k, v, scale, rel_h=None, rel_w=None, rel_s=0):
    """q: [B, Nq, heads, d], k / v: [B, Nkv, heads, d]; rel_h / rel_w: [B * heads, Nq, rel_s] or None.
    Returns [B, Nq, heads, d] in float64, one batch element at a time (bounded memory at 4096 x 4096 logits)."""
    B, Nq, heads, d = q.shape
    Nkv = k.shape[1]
    out = torch.empty(B, Nq, heads, d, dtype=torch.float64, device=q.device)
    for b in range(B):
        s = torch.einsum("qhc,khc->hqk", q[b].double(), k[b].double()) * scale
        if rel_h is not None:
            kk = torch.arange(Nkv, device=q.device)
            rh = rel_h[b * heads:(b + 1) * heads].double()
            rw = rel_w[b * heads:(b + 1) * heads].double()
            s = s + rh[:, :, kk // rel_s] + rw[:, :, kk % rel_s]
        out[b] = torch.einsum("hqk,khc->qhc", torch.softmax(s, dim=-1), v[b].double())
    return out
