"""Float64 reference of ea_attention written from its definition (include/editanything_b200.h):
out = softmax(Q K^T * scale + bias) V with bias[q, kk] = rel_h[q, kk // rel_s] + rel_w[q, kk % rel_s].

Also the per-element error bound of the kernel's arithmetic (attention_bound), the input generators that stress the
softmax, and the table of cases tests/test_gpu_attention.py runs on the GPU and tests/test_attn_bound_cpu.py runs
through a CPU model of the kernel."""
import math

import torch

from tests import fp64_refs as R

U = R.U32
LOG2E = 1.4426950408889634
# ex2.approx.ftz.f32: "maximum relative error for .f32 type is 2 ulp across the full range of inputs" (PTX ISA,
# section "Floating Point Instructions: ex2"); 2 ulp of the result is at most 2^-22 of it.
EX2_REL = 2.0 ** -22


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


def sub_tile(d):
    """Keys per S sub-tile of the kernel: 128 while the P V accumulator is at most 80 wide, 64 above."""
    return 128 if d <= 80 else 64


def storage_rounding(dtype):
    """(u_P, s_P) of the 16-bit type P is stored in for P V: unit roundoff and subnormal spacing."""
    if dtype == torch.float16:
        return 2.0 ** -11, 2.0 ** -24
    return 2.0 ** -8, 2.0 ** -133


def attention_bound(q, k, v, scale, rel_h=None, rel_w=None, rel_s=0, dtype=torch.float16, chunk=1 << 25):
    """(o, bound), both [B, Nq, heads, d] float64 on the inputs' device: the exact output and a bound on
    |ea_attention - o| per element, for 16-bit q / k / v (exact in float64) and fp32 rel_h / rel_w.

    The kernel (editanything_b200/csrc/ea_attn.cu) forms x_k = fma(s_k, scale log2e, -m) in the log2 domain with the
    running max m, p_k = ex2(x_k) in fp32, accumulates l = sum p in fp32 from the unrounded p, rounds p to `dtype`
    for O += P V (fp32 accumulation), rescales O and l by ex2(m_old - m_new) when the max rises, and stores O / l.
    With P the exact softmax weights, o = P V and u = 2^-24, the bound is the sum of:
      * output rounding: ulp(o) of `dtype`;
      * P quantisation: sum_k max(u_P P_k, (s_P / 2) P_max) |v_k|.  u_P / s_P are the unit roundoff / subnormal
        spacing of `dtype`.  p is rounded relative to the running max, which never exceeds the final one, and
        ulp(x c) / c <= eps x, so P relative to the final max bounds it.  Not mean-subtracted: l does not see it;
      * logit and exponent error: sum_k P_k ln2 delta_k (|v_k| + |o|), where delta_k is the log2-domain error of x_k:
          - (d + 8) u scale log2e sum_c |q_c k_c| for the fp32 Q K^T;
          - 4 u (|s_k scale log2e| + |bias_k log2e| + the row's max |logit| log2e) for the rounded scale log2e, the
            bias add, the FMA and the running max;
          - with the bias, 3 u log2e (|rel_h| + |rel_w|) for their products with log2e and their sum;
          - (n_sub + 1) EX2_REL / ln2: the ex2 of p and of every rescale factor a tile goes through (O and l are
            rescaled by the same factor, so its error acts as a shift of that tile's logits);
      * accumulation of O and l and the final divide: (Nkv + 2 n_sub + 8) u sum_k P_k |v_k| +
        (Nkv + n_sub + 8) u |o|, n_sub = ceil(Nkv / sub_tile(d)).
    Computed per (batch, head) in chunks of query rows (`chunk` logits at a time), so that 16384-token
    self-attention fits in memory."""
    B, Nq, heads, d = q.shape
    Nkv = k.shape[1]
    n_sub = -(-Nkv // sub_tile(d))
    u_p, s_p = storage_rounding(dtype)
    dev = q.device
    o = torch.empty(B, Nq, heads, d, dtype=torch.float64, device=dev)
    bound = torch.empty_like(o)
    rows = max(1, chunk // Nkv)
    kk = torch.arange(Nkv, device=dev)
    ex2_term = (n_sub + 1) * EX2_REL
    for b in range(B):
        for h in range(heads):
            K = k[b, :, h].double()
            V = v[b, :, h].double()
            Ka, Va = K.abs(), V.abs()
            for r0 in range(0, Nq, rows):
                Q = q[b, r0:r0 + rows, h].double()
                s = (Q @ K.T) * scale
                lnd = (d + 8) * U * scale * (Q.abs() @ Ka.T) + 4 * U * s.abs() + ex2_term
                if rel_h is not None:
                    rh = rel_h[b * heads + h, r0:r0 + rows].double()[:, kk // rel_s]
                    rw = rel_w[b * heads + h, r0:r0 + rows].double()[:, kk % rel_s]
                    s = s + rh + rw
                    lnd = lnd + 7 * U * (rh.abs() + rw.abs())      # 4 u |bias| + 3 u (|rel_h| + |rel_w|)
                lnd = lnd + 4 * U * s.abs().amax(dim=1, keepdim=True)
                P = torch.softmax(s, dim=1)
                del s
                ob = P @ V
                pv = P @ Va
                oa = ob.abs()
                w = P * lnd
                err = w @ Va + w.sum(dim=1, keepdim=True) * oa
                del w, lnd
                err += torch.maximum(u_p * P, (s_p / 2) * P.amax(dim=1, keepdim=True)) @ Va
                err += (Nkv + 2 * n_sub + 8) * U * pv + (Nkv + n_sub + 8) * U * oa
                err += R.ulp(ob, dtype)
                o[b, r0:r0 + rows, h] = ob
                bound[b, r0:r0 + rows, h] = err
    return o, bound


# ---- input generators -----------------------------------------------------------------------------------------
GENERATORS = ("randn", "flat-offset", "peaked", "rising", "early", "ties", "bias", "distinct")


def rel_size(Nkv):
    """Smallest rel_s with rel_s^2 >= Nkv."""
    S = math.isqrt(Nkv)
    return S if S * S >= Nkv else S + 1


def make_inputs(gen, B, heads, Nq, Nkv, d, scale, rel_s=0, *, seed=0, device="cpu", dtype=torch.float16):
    """Seeded q [B, Nq, heads, d], k / v [B, Nkv, heads, d] in `dtype` and, with rel_s > 0, fp32 rel_h / rel_w
    [B * heads, Nq, rel_s].  z = scale sqrt(d) is the logit spread of N(0, 1) q and k.
      randn        q, k, v ~ N(0, 1)
      flat-offset  v = 1 + N(0, 1): |o| ~ 1, so a wrong normaliser shows
      peaked       logits of spread 12: one dominant key per row, most P fp16-subnormal or zero
      rising       logits rise by 24 from the first key to the last along a direction shared by q and k: the max
                   rises on every tile and O is rescaled each time
      early        the reverse: the max is in the first tile and late tiles underflow
      ties         every k row equal: a uniform softmax over all keys, v = 1 + N(0, 1)
      bias         rel_h a ramp in kh with a random sign per row, rel_w random, both of magnitude 3 max(1, z)
      distinct     v = N(0, 1) + 10 b + h, so a read from another (batch, head) shows"""
    g = torch.Generator(device=device).manual_seed(seed)

    def rn(*shape):
        return torch.randn(*shape, generator=g, device=device)

    q, k, v = rn(B, Nq, heads, d), rn(B, Nkv, heads, d), rn(B, Nkv, heads, d)
    z = scale * math.sqrt(d)
    if gen == "flat-offset":
        v = v + 1.0
    elif gen == "peaked":
        q = q * (12.0 / z)
    elif gen in ("rising", "early"):
        dirn = torch.full((d,), d ** -0.5, device=device)
        ramp = torch.linspace(0.0, 1.0, Nkv, device=device)
        if gen == "early":
            ramp = 1.0 - ramp
        alpha = math.sqrt(d)
        beta = 24.0 * ramp / (scale * alpha)                              # q.k_j scale = 24 ramp_j
        q = alpha * dirn + 0.05 * q
        k = beta[None, :, None, None] * dirn + 0.05 * k
    elif gen == "ties":
        k = k[:, :1].expand(B, Nkv, heads, d).clone()
        v = v + 1.0
    elif gen == "distinct":
        v = v + (10.0 * torch.arange(B, device=device)[:, None, None, None]
                 + torch.arange(heads, device=device)[None, None, :, None])
    rel_h = rel_w = None
    if rel_s:
        if gen == "bias":
            a = 3.0 * max(1.0, z)
            sign = torch.where(rn(B * heads, Nq, 1) < 0, -1.0, 1.0)
            rel_h = a * sign * torch.linspace(-1.0, 1.0, rel_s, device=device) + 0.1 * rn(B * heads, Nq, rel_s)
            rel_w = a * rn(B * heads, Nq, rel_s)
        else:
            rel_h, rel_w = rn(B * heads, Nq, rel_s), rn(B * heads, Nq, rel_s)
    return dict(q=q.to(dtype), k=k.to(dtype), v=v.to(dtype), rel_h=rel_h, rel_w=rel_w)


# ---- cases ------------------------------------------------------------------------------------------------------
# name -> (gen, B, heads, Nq, Nkv, d, scale (None: d^-0.5), rel_s (0: no bias), layout)
#   layout "pad":   q / k / v / out rows padded by 8 elements
#   layout "gap":   also gaps of rows between batch elements of q, k, v and out (canary rows in out's gaps)
#   layout "kv":    cross-attention: K and V interleaved in one [B * Nkv, 2 heads d] buffer (nets.py)
#   layout "fused": self-attention: q | k | v of one [B, N, 3 heads d] buffer (nets.py)
CASES = {}


def _case(name, gen, B, heads, Nq, Nkv, d, scale=None, rel_s=0, layout="pad"):
    assert name not in CASES, name
    CASES[name] = (gen, B, heads, Nq, Nkv, d, scale, rel_s, layout)


WIDTHS = (40, 64, 80, 160, 192)       # P V accumulator widths 48 / 64 / 80 / 160 / 192
# every generator at every width, with and without the bias: Nq mod 128 = 65 (warp-group 1 split), Nkv mod 128 =
# 65 and mod 64 = 1, three key tiles (pipelined up to d = 80 without the bias, one-stage ring at d = 192)
for _d in WIDTHS:
    for _g in GENERATORS[1:]:
        if _g != "bias":
            _case(f"{_g} d{_d}", _g, 2, 2, 193, 321, _d)
        _case(f"{_g} d{_d} bias", _g, 2, 2, 193, 321, _d, rel_s=18)
# ragged key counts: Nkv mod 128 in {1, 64, 65, 127} (single tiles at 1 / 64 / 65 / 127), mod 64 in {1, 63}
for _d in (64, 160):
    for _n in (1, 64, 65, 127, 129, 192, 255, 385):
        _case(f"keys{_n} d{_d}", "flat-offset", 2, 2, 100, _n, _d)
        _case(f"keys{_n} d{_d} bias", "flat-offset", 2, 2, 100, _n, _d, rel_s=rel_size(_n))
# ragged query counts: Nq mod 128 in {1, 8, 64, 65}: warp-group 1 wholly past Nq, or the lo / hi rows of a quad split
for _d in (40, 160):
    for _n in (1, 8, 64, 65, 129, 136, 192, 193):
        _case(f"queries{_n} d{_d}", "distinct", 2, 2, _n, 300, _d)
# softmax scales
for _s in (1.0, 0.05, 3.0):
    for _g in ("flat-offset", "peaked", "rising", "early"):
        for _d in (64, 160):
            _case(f"{_g} d{_d} scale{_s}", _g, 2, 2, 130, 400, _d, scale=_s)
    _case(f"bias d80 scale{_s}", "bias", 2, 2, 130, 400, 80, scale=_s, rel_s=20)
# a key count at which the rescale defect of the CPU model shows at two tiles
_case("rising d64 keys129", "rising", 2, 2, 64, 129, 64)
_case("flat-offset d64 keys129 scale0.05", "flat-offset", 2, 2, 65, 129, 64, scale=0.05)
# batch strides with gaps
for _d in (40, 160):
    _case(f"gap d{_d}", "distinct", 3, 2, 150, 200, _d, layout="gap")
    _case(f"gap d{_d} bias", "bias", 3, 2, 150, 196, _d, rel_s=14, layout="gap")
# the denoising step's layouts: cross-attention on 77 context tokens at the UNets' head dims
_case("cross sd15 d40", "flat-offset", 2, 8, 4096, 77, 40, layout="kv")
_case("cross sd15 d80", "peaked", 2, 8, 1024, 77, 80, layout="kv")
_case("cross sd15 d160", "distinct", 2, 8, 256, 77, 160, layout="kv")
_case("cross sd21 d64", "flat-offset", 2, 5, 2304, 77, 64, layout="kv")
# the largest self-attentions: SD1.5 1024 x 1024 (128 x 128 latents, 16384 tokens) and SD2.1 768 x 768 (9216)
_case("self sd15-1024 16384", "flat-offset", 2, 8, 16384, 16384, 40, layout="fused")
_case("self sd21-768 9216", "flat-offset", 2, 5, 9216, 9216, 64, layout="fused")
# SAM ViT-H: 14 x 14 windows (25 per image) and 64 x 64 global attention, d = 80, 16 heads; two images
_case("sam window", "bias", 50, 16, 196, 196, 80, rel_s=14)
_case("sam global", "bias", 2, 16, 4096, 4096, 80, rel_s=64)
_case("sam global peaked", "peaked", 2, 16, 4096, 4096, 80, rel_s=64)
