"""GPU bring-up probe: every C-ABI operator against a plain torch fp32 reference.

Each case runs in its own subprocess (a faulting kernel kills only its own CUDA context) under a
timeout; results are appended to gpurun_out/probe_ops.jsonl.
Usage: python tools/gpu_probe_ops.py [case ...]      (no args = all cases)
"""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, "gpurun_out")


def _err(a, b):
    a = a.float()
    b = b.float()
    d = (a - b).abs()
    return {"max_abs": d.max().item(), "ref_max": b.abs().max().item(),
            "rel_fro": (d.norm() / (b.norm() + 1e-12)).item()}


def case_gemm_linear(force_bn=0, M=300, N=320, K=320, **kw):
    import torch
    from editanything_b200 import ops, _lib as L
    dt = ops.half_dtype()
    torch.manual_seed(0)
    a = torch.randn(M, K, device="cuda").to(dt)
    w = (torch.randn(N, K, device="cuda") / K ** 0.5).to(dt)
    bias = torch.randn(N, device="cuda")
    res = torch.randn(M, N, device="cuda").to(dt)
    out = torch.full((M, N), 7.0, device="cuda", dtype=dt)
    ops.gemm(a, w, out, bias=bias, residual=res, force_bn=force_bn, **kw)
    torch.cuda.synchronize()
    ref = a.float() @ w.float().t() + bias + res.float()
    return _err(out, ref)


def case_gemm_plain():
    # smallest possible: one tile, K=64, no epilogue extras
    import torch
    from editanything_b200 import ops
    dt = ops.half_dtype()
    torch.manual_seed(1)
    a = torch.randn(128, 64, device="cuda").to(dt)
    w = torch.randn(128, 64, device="cuda").to(dt) / 8
    out = ops.gemm(a, w, force_bn=128)
    torch.cuda.synchronize()
    return _err(out, a.float() @ w.float().t())


def case_gemm_bn64():
    return case_gemm_linear(force_bn=64)


def case_gemm_bn128():
    return case_gemm_linear(force_bn=128)


def case_gemm_bn256():
    return case_gemm_linear(force_bn=256, M=512, N=512, K=1024)


def case_gemm_big():
    return case_gemm_linear(M=8192, N=1280, K=2560)


def case_gemm_ktail():
    return case_gemm_linear(M=154, N=320, K=776)  # K not a multiple of 64, M ragged


def case_gemm_splitk():
    """Small-M, long-K problems: the planner splits K; also forced split counts (3, 7) and a
    repeat launch (the in-kernel counters must have been re-armed)."""
    import torch
    from editanything_b200 import ops
    dt = ops.half_dtype()
    torch.manual_seed(11)
    res, worst = {}, 0.0
    for (M, N, K, fs) in [(128, 1280, 11520, 0), (128, 1280, 5120, 3), (512, 1280, 2560, 0), (100, 320, 1288, 7),
                          (128, 1280, 11520, 0)]:
        a = torch.randn(M, K, device="cuda").to(dt)
        w = (torch.randn(N, K, device="cuda") / K ** 0.5).to(dt)
        bias = torch.randn(N, device="cuda")
        resid = torch.randn(M, N, device="cuda").to(dt)
        out = torch.full((M, N), 7.0, device="cuda", dtype=dt)
        ops.gemm(a, w, out, bias=bias, residual=resid, force_splits=fs)
        torch.cuda.synchronize()
        e = _err(out, a.float() @ w.float().t() + bias + resid.float())
        res[f"{M}x{N}x{K}/s{fs}#{len(res)}"] = e
        worst = max(worst, e["max_abs"] / max(1.0, e["ref_max"]))
    ws = ops.gemm_workspace(torch.device("cuda", torch.cuda.current_device()))
    res["counters_rearmed"] = int(ws[:65536].view(torch.int32).abs().sum().item())
    res["max_abs"] = worst if res["counters_rearmed"] == 0 else 1e9
    res["ref_max"] = 1.0
    return res


def case_concurrent_variants():
    """The no-inter-CTA-wait variants used when several streams run concurrently: two-pass GroupNorm
    and split-K whose last-arriving CTA reduces the tile (ops.set_lane(lane, True))."""
    from editanything_b200 import ops
    ops.set_lane(1, True)
    try:
        a = case_groupnorm()
        b = case_gemm_splitk()
        c = case_conv_8_skip_splitk()
        d = case_gemm_splitk_geglu()
    finally:
        ops.set_lane(0, False)
    w = max(a["max_abs"], b["max_abs"], c["max_abs"] / max(1.0, c["ref_max"]), d["max_abs"])
    return {"max_abs": w, "ref_max": 1.0, "gn": a["max_abs"], "splitk": b["max_abs"], "conv": c["max_abs"], "geglu": d["max_abs"]}


def case_gemm_splitk_geglu():
    import torch
    from editanything_b200 import ops, _lib as L
    dt = ops.half_dtype()
    torch.manual_seed(12)
    M, C_, F = 128, 1280, 1280  # proj: C -> 2F, small M => planner may split K; also forced
    a = torch.randn(M, C_, device="cuda").to(dt)
    w = (torch.randn(2 * F, C_, device="cuda") / C_ ** 0.5).to(dt)
    b = torch.randn(2 * F, device="cuda")
    idx = torch.cat([torch.cat([torch.arange(j * 64, j * 64 + 64), F + torch.arange(j * 64, j * 64 + 64)])
                     for j in range(F // 64)]).cuda()
    y = a.float() @ w.float().t() + b
    ref = y[:, :F] * torch.nn.functional.gelu(y[:, F:])
    worst = 0.0
    for fs in (0, 4):
        out = ops.gemm(a, w[idx].contiguous(), bias=b[idx].contiguous(), act=L.EA_ACT_GEGLU, force_splits=fs)
        torch.cuda.synchronize()
        e = _err(out, ref)
        worst = max(worst, e["max_abs"] / max(1.0, e["ref_max"]))
    return {"max_abs": worst, "ref_max": 1.0}


def case_gemm_geglu():
    import torch
    from editanything_b200 import ops, _lib as L
    dt = ops.half_dtype()
    torch.manual_seed(2)
    M, C_, F = 256, 320, 1280  # proj: C -> 2F
    a = torch.randn(M, C_, device="cuda").to(dt)
    w = (torch.randn(2 * F, C_, device="cuda") / C_ ** 0.5).to(dt)
    b = torch.randn(2 * F, device="cuda")
    # interleave per 64: block j = [value rows j*64..+64 | gate rows F + j*64..+64]
    idx = torch.cat([torch.cat([torch.arange(j * 64, j * 64 + 64), F + torch.arange(j * 64, j * 64 + 64)])
                     for j in range(F // 64)]).cuda()
    out = ops.gemm(a, w[idx].contiguous(), bias=b[idx].contiguous(), act=L.EA_ACT_GEGLU)
    torch.cuda.synchronize()
    y = a.float() @ w.float().t() + b
    ref = y[:, :F] * torch.nn.functional.gelu(y[:, F:])
    return _err(out, ref)


def case_gemm_accum_scale_dual():
    import torch
    from editanything_b200 import ops
    dt = ops.half_dtype()
    torch.manual_seed(3)
    M, N, K = 256, 320, 320
    a = torch.randn(M, K, device="cuda").to(dt)
    w = (torch.randn(N, K, device="cuda") / K ** 0.5).to(dt)
    bias = torch.randn(N, device="cuda")
    buf = torch.randn(M, 2 * N, device="cuda").to(dt)  # concat buffer; accumulate into right half
    before = buf.clone()
    ops.gemm(a, w, buf[:, N:], bias=bias, out_scale=0.5, accumulate=True, ldo=2 * N)
    torch.cuda.synchronize()
    ref = before.float()
    ref[:, N:] += 0.5 * (a.float() @ w.float().t() + bias)
    e1 = _err(buf, ref)
    o1 = torch.empty(M, N, device="cuda", dtype=dt)
    o2 = torch.zeros(M, 2 * N, device="cuda", dtype=dt)
    rv = torch.randn(2, N, device="cuda")
    ops.gemm(a, w, o1, rowvec=rv, rows_per_batch=128, out2=o2[:, N:], ldo2=2 * N)
    torch.cuda.synchronize()
    r2 = a.float() @ w.float().t() + rv.repeat_interleave(128, 0)
    e2 = _err(o1, r2)
    e3 = _err(o2[:, N:], r2)
    return {"accum": e1, "rowvec": e2, "dual": e3, "max_abs": max(e1["max_abs"], e2["max_abs"], e3["max_abs"]),
            "ref_max": e1["ref_max"]}


def _conv_case(B, H, W, Cin, Cout, stride=1, extra=0, seed=4):
    import torch
    import torch.nn.functional as F
    from editanything_b200 import ops, _lib as L
    dt = ops.half_dtype()
    torch.manual_seed(seed)
    Hin, Win = H * stride, W * stride
    x = torch.randn(B, Cin, Hin, Win, device="cuda").to(dt)
    w = (torch.randn(Cout, Cin, 3, 3, device="cuda") / (9 * Cin) ** 0.5).to(dt)
    bias = torch.randn(Cout, device="cuda")
    rv = torch.randn(B, Cout, device="cuda")
    x_nhwc = x.permute(0, 2, 3, 1).contiguous()
    wp = w.permute(0, 2, 3, 1).reshape(Cout, 9 * Cin)
    ref = F.conv2d(x.float(), w.float(), bias, stride=stride, padding=1) + rv[:, :, None, None]
    xe = None
    if extra:
        xr = torch.randn(B, extra, H, W, device="cuda").to(dt)
        ws = (torch.randn(Cout, extra, 1, 1, device="cuda") / extra ** 0.5).to(dt)
        ref = ref + F.conv2d(xr.float(), ws.float())
        xe = xr.permute(0, 2, 3, 1).contiguous()
        wp = torch.cat([wp, ws.reshape(Cout, extra)], 1)
    wp = wp.contiguous()
    out = torch.empty(B * H * W, Cout, device="cuda", dtype=dt)
    ops.gemm(x_nhwc, wp, out, mode=L.EA_GEMM_CONV_S1 if stride == 1 else L.EA_GEMM_CONV_S2,
             conv=(B, H, W, Cin), a_extra=xe, bias=bias, rowvec=rv)
    torch.cuda.synchronize()
    ref = ref.permute(0, 2, 3, 1).reshape(B * H * W, Cout)
    return _err(out, ref)


def case_conv_64():
    return _conv_case(2, 64, 64, 320, 320)


def case_conv_32():
    return _conv_case(2, 32, 32, 640, 640)


def case_conv_8():
    return _conv_case(2, 8, 8, 1280, 1280)


def case_conv_8_skip_splitk():
    return _conv_case(2, 8, 8, 1280, 1280, extra=2560)


def case_conv_8_b1():
    return _conv_case(1, 8, 8, 128, 64)


def case_conv_16_skip():
    return _conv_case(2, 16, 16, 1280, 1280, extra=1920)


def case_conv_s2():
    return _conv_case(2, 32, 32, 320, 320, stride=2)


def case_conv_s2_small():
    return _conv_case(2, 8, 8, 1280, 1280, stride=2)


def case_conv_96():
    return _conv_case(1, 96, 96, 64, 64)


def _attn_case(B, heads, Nq, Nkv, d, seed=5, fused=False, rel_s=0):
    import torch
    from editanything_b200 import ops
    dt = ops.half_dtype()
    torch.manual_seed(seed)
    C_ = heads * d
    if fused:
        qkv = torch.randn(B, Nq, 3 * C_, device="cuda").to(dt)
        q, k, v = qkv[..., :C_], qkv[..., C_:2 * C_], qkv[..., 2 * C_:]
        qs = ks = vs = (Nq * 3 * C_, 3 * C_)
    else:
        q = torch.randn(B, Nq, C_, device="cuda").to(dt)
        k = torch.randn(B, Nkv, C_, device="cuda").to(dt)
        v = torch.randn(B, Nkv, C_, device="cuda").to(dt)
        qs, ks, vs = (Nq * C_, C_), (Nkv * C_, C_), (Nkv * C_, C_)
    out = torch.zeros(B, Nq, C_, device="cuda", dtype=dt)
    scale = d ** -0.5
    rel_h = rel_w = None
    if rel_s:
        rel_h = torch.randn(B * heads, Nq, rel_s, device="cuda")
        rel_w = torch.randn(B * heads, Nq, rel_s, device="cuda")
    ops.attention(q, k, v, out, B=B, heads=heads, Nq=Nq, Nkv=Nkv, d=d, q_strides=qs, k_strides=ks,
                  v_strides=vs, o_strides=(Nq * C_, C_), scale=scale, rel_h=rel_h, rel_w=rel_w, rel_s=rel_s)
    torch.cuda.synchronize()
    qf = q.float().reshape(B, Nq, heads, d).permute(0, 2, 1, 3)
    kf = k.float().reshape(B, Nkv, heads, d).permute(0, 2, 1, 3)
    vf = v.float().reshape(B, Nkv, heads, d).permute(0, 2, 1, 3)
    s = qf @ kf.transpose(-1, -2) * scale
    if rel_s:
        bias = rel_h.reshape(B, heads, Nq, rel_s, 1) + rel_w.reshape(B, heads, Nq, 1, rel_s)
        s = s + bias.reshape(B, heads, Nq, rel_s * rel_s)[..., :Nkv]
    ref = (s.softmax(-1) @ vf).permute(0, 2, 1, 3).reshape(B, Nq, C_)
    return _err(out, ref)


def case_attn_d64():
    return _attn_case(1, 2, 128, 128, 64)


def case_attn_d40_self():
    return _attn_case(2, 8, 4096, 4096, 40, fused=True)


def case_attn_db_long():
    """Double-buffered-logits kernel (d <= 64, >= 384 keys): ragged key count (last 96-key tile partial),
    d = 40 and d = 64, more than one CTA wave."""
    r1 = _attn_case(2, 8, 4096, 4000, 40)
    r2 = _attn_case(1, 10, 2304, 2304, 64)
    r3 = _attn_case(2, 8, 2300, 400, 40)
    w = max(r["max_abs"] for r in (r1, r2, r3))
    return {"max_abs": w, "ref_max": max(r["ref_max"] for r in (r1, r2, r3)), "rel_fro": max(r["rel_fro"] for r in (r1, r2, r3))}


def case_attn_d80_self():
    return _attn_case(2, 8, 1024, 1024, 80)


def case_attn_d160_self():
    return _attn_case(2, 8, 256, 256, 160)


def case_attn_cross77():
    return _attn_case(2, 8, 1024, 77, 80)


def case_attn_cross77_d40():
    return _attn_case(2, 8, 4096, 77, 40)


def case_attn_sam_window():
    return _attn_case(3, 16, 196, 196, 80, rel_s=14)


def case_attn_sam_global():
    return _attn_case(1, 4, 4096, 4096, 80, rel_s=64)


def case_groupnorm():
    import torch
    import torch.nn.functional as F
    from editanything_b200 import ops
    dt = ops.half_dtype()
    torch.manual_seed(6)
    res = {}
    worst = 0.0
    for (B, H, C1, C2) in [(2, 64, 320, 0), (2, 16, 1280, 640), (2, 32, 640, 320), (2, 8, 1280, 1280)]:
        C_ = C1 + C2
        x1 = (torch.randn(B, H, H, C1, device="cuda") * 2 + 0.5).to(dt)
        x2 = (torch.randn(B, H, H, C2, device="cuda") - 1).to(dt) if C2 else None
        g = torch.randn(C_, device="cuda")
        b = torch.randn(C_, device="cuda")
        out = torch.empty(B, H, H, C_, device="cuda", dtype=dt)
        ops.groupnorm(x1, g, b, out, B=B, HW=H * H, C_=C_, eps=1e-5, silu=True, x2=x2, C1=C1)
        torch.cuda.synchronize()
        xc = torch.cat([x1, x2], -1) if C2 else x1
        ref = F.silu(F.group_norm(xc.float().permute(0, 3, 1, 2), 32, g, b, 1e-5)).permute(0, 2, 3, 1)
        e = _err(out, ref)
        res[f"{B}x{H}x{C1}+{C2}"] = e
        worst = max(worst, e["max_abs"] / max(1.0, e["ref_max"]))
    res["max_abs"] = worst       # relative to each case's output magnitude (fp16 ulp scales with it)
    res["ref_max"] = 1.0
    return res


def case_layernorm():
    import torch
    import torch.nn.functional as F
    from editanything_b200 import ops
    dt = ops.half_dtype()
    torch.manual_seed(7)
    worst = 0.0
    for (M, C_) in [(8192, 320), (512, 1280), (100, 640), (77, 256)]:
        x = (torch.randn(M, C_, device="cuda") * 3 + 1).to(dt)
        g = torch.randn(C_, device="cuda")
        b = torch.randn(C_, device="cuda")
        out = torch.empty_like(x)
        ops.layernorm(x, g, b, out, M=M, C_=C_, eps=1e-5)
        torch.cuda.synchronize()
        e = _err(out, F.layer_norm(x.float(), (C_,), g, b, 1e-5))
        worst = max(worst, e["max_abs"] / max(1.0, e["ref_max"]))
    return {"max_abs": worst, "ref_max": 1.0}


def case_small_ops():
    import torch
    import torch.nn.functional as F
    from editanything_b200 import ops
    dt = ops.half_dtype()
    torch.manual_seed(8)
    r = {}
    # conv_direct
    x = torch.randn(2, 3, 32, 32, device="cuda").to(dt)
    w = torch.randn(16, 3, 3, 3, device="cuda") * 0.2
    b = torch.randn(16, device="cuda")
    out = torch.empty(2, 32, 32, 16, device="cuda", dtype=dt)
    ops.conv_direct(x.permute(0, 2, 3, 1).contiguous(), w.permute(2, 3, 1, 0).contiguous(), b, out,
                    B=2, Hin=32, Win=32, Cin=3, Cout=16, silu=True)
    ref = F.silu(F.conv2d(x.float(), w, b, padding=1)).permute(0, 2, 3, 1)
    r["conv_direct_s1"] = _err(out, ref)
    x = torch.randn(2, 32, 32, 32, device="cuda").to(dt)
    w = torch.randn(96, 32, 3, 3, device="cuda") * 0.1
    out = torch.empty(2, 16, 16, 96, device="cuda", dtype=dt)
    add = torch.randn(2, 16, 16, 96, device="cuda").to(dt)
    ops.conv_direct(x.permute(0, 2, 3, 1).contiguous(), w.permute(2, 3, 1, 0).contiguous(), None, out,
                    B=2, Hin=32, Win=32, Cin=32, Cout=96, stride=2, add=add)
    ref = F.conv2d(x.float(), w, None, stride=2, padding=1).permute(0, 2, 3, 1) + add.float()
    r["conv_direct_s2"] = _err(out, ref)
    # upsample
    x = torch.randn(2, 8, 8, 64, device="cuda").to(dt)
    out = torch.empty(2, 16, 16, 64, device="cuda", dtype=dt)
    ops.upsample2x(x, out, B=2, H=8, W=8, C_=64)
    ref = F.interpolate(x.float().permute(0, 3, 1, 2), scale_factor=2, mode="nearest").permute(0, 2, 3, 1)
    r["upsample"] = _err(out, ref)
    # small linear + timestep embedding
    t = torch.tensor([981.0, 981.0], device="cuda")
    emb = torch.empty(2, 320, device="cuda")
    ops.timestep_embedding(t, emb, B=2, dim=320)
    half = 160
    freqs = torch.exp(-torch.log(torch.tensor(10000.0)) * torch.arange(half, device="cuda") / half)
    args = t[:, None] * freqs[None]
    r["temb"] = _err(emb, torch.cat([torch.cos(args), torch.sin(args)], -1))
    W1 = (torch.randn(1280, 320, device="cuda") / 18).to(dt)
    b1 = torch.randn(1280, device="cuda")
    y = torch.empty(2, 1280, device="cuda")
    ops.small_linear(emb, W1, b1, y, M=2, N=1280, K=320, silu_out=True)
    r["small_linear"] = _err(y, F.silu(emb @ W1.float().t() + b1))
    y2 = torch.empty(2, 320, device="cuda")
    W2 = (torch.randn(320, 1280, device="cuda") / 36).to(dt)
    ops.small_linear(y, W2, None, y2, M=2, N=320, K=1280, silu_in=True)
    r["small_linear_siluin"] = _err(y2, F.silu(y) @ W2.float().t())
    torch.cuda.synchronize()
    r["max_abs"] = max(v["max_abs"] / max(1.0, v["ref_max"]) for v in r.values())   # relative to magnitude
    r["ref_max"] = 1.0
    return r


def case_conv_in():
    import torch
    import torch.nn.functional as F
    from editanything_b200 import ops
    dt = ops.half_dtype()
    torch.manual_seed(13)
    x = torch.randn(2, 4, 64, 64, device="cuda").to(dt)
    w = torch.randn(320, 4, 3, 3, device="cuda") * 0.2
    b = torch.randn(320, device="cuda")
    add = torch.randn(2, 64, 64, 320, device="cuda").to(dt)
    out = torch.empty(2, 64, 64, 320, device="cuda", dtype=dt)
    cat = torch.zeros(2, 64, 64, 640, device="cuda", dtype=dt)
    ops.conv_in(x.permute(0, 2, 3, 1).contiguous(), w.permute(2, 3, 1, 0).contiguous(), b, out, B=2, H=64, W=64, Cin=4,
                Cout=320, out2=cat[..., 320:], ldo2=640, add=add)
    torch.cuda.synchronize()
    ref = F.conv2d(x.float(), w, b, padding=1).permute(0, 2, 3, 1) + add.float()
    e1, e2 = _err(out, ref), _err(cat[..., 320:], ref)
    return {"max_abs": max(e1["max_abs"], e2["max_abs"]) / max(1.0, e1["ref_max"]), "ref_max": 1.0,
            "left_untouched": float(cat[..., :320].abs().max().item())}


def case_out_cfg_ddim():
    import torch
    import torch.nn.functional as F
    from editanything_b200 import ops
    dt = ops.half_dtype()
    torch.manual_seed(9)
    Nimg, H, C_ = 2, 16, 320
    xn = torch.randn(2 * Nimg, H, H, C_, device="cuda").to(dt)
    w = torch.randn(4, C_, 3, 3, device="cuda") / (9 * C_) ** 0.5
    b = torch.randn(4, device="cuda")
    lat = torch.randn(Nimg, H, H, 4, device="cuda")
    lat0 = lat.clone()
    eps_out = torch.empty(2 * Nimg, H, H, 4, device="cuda")
    coef = torch.tensor([0.3, 0.95, 0.4, 0.91], device="cuda")
    known = torch.randn(Nimg, H, H, 4, device="cuda")
    mask = (torch.rand(Nimg, H, H, device="cuda") > 0.5).float()
    lh = torch.empty(2 * Nimg, H, H, 4, device="cuda", dtype=dt)
    ops.out_cfg_ddim(xn, w.permute(0, 2, 3, 1).contiguous(), b, latents=lat, eps_out=eps_out, coef=coef,
                     guidance=9.0, known=known, mask=mask, lat_half_out=lh, Nimg=Nimg, H=H, W=H, C_=C_)
    torch.cuda.synchronize()
    eps = F.conv2d(xn.float().permute(0, 3, 1, 2), w, b, padding=1).permute(0, 2, 3, 1)
    e = eps[:Nimg] + 9.0 * (eps[Nimg:] - eps[:Nimg])
    x0 = (lat0 - 0.95 * e) / 0.3
    xp = 0.4 * x0 + 0.91 * e
    xp = known * mask[..., None] + xp * (1 - mask[..., None])
    r = {"eps": _err(eps_out, eps), "lat": _err(lat, xp), "lat_half": _err(lh, torch.cat([xp, xp]))}
    r["max_abs"] = max(r["eps"]["max_abs"], r["lat"]["max_abs"] / 10)
    r["ref_max"] = 1.0
    return r


def _ln_fold_case(M, C, N, geglu, persistent, seed=21):
    """LayerNorm folded into the GEMMs around it: producer (x = a w0^T + b0 + res, row statistics) ->
    consumer (LN(x) w1^T + b1, optionally GEGLU) against torch fp32 on the same half inputs."""
    import torch
    import torch.nn.functional as F
    from editanything_b200 import ops, _lib as L
    dt = ops.half_dtype()
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = torch.randn(M, C, device="cuda", generator=g).to(dt)
    w0 = (torch.randn(C, C, device="cuda", generator=g) / C ** 0.5).to(dt)
    b0 = torch.randn(C, device="cuda", generator=g)
    res = (torch.randn(M, C, device="cuda", generator=g) * 2 + 0.7).to(dt)     # non-zero row means
    gam = 1 + 0.2 * torch.randn(C, device="cuda", generator=g)
    bet = 0.3 * torch.randn(C, device="cuda", generator=g)
    w1 = torch.randn(N, C, device="cuda", generator=g) / C ** 0.5
    b1 = torch.randn(N, device="cuda", generator=g)
    # pack like nets.PackedNet._pack_attn
    wg = (w1.double() * gam.double()[None, :]).float().to(dt)
    gvec = wg.double().sum(1).float()
    cvec = (w1.double() @ bet.double()).float() + b1
    fp = persistent
    x = torch.full((M, C), 7.0, device="cuda", dtype=dt)
    st = torch.full((C // 32, M, 2), float("nan"), device="cuda")
    ops.gemm(a, w0, x, bias=b0, residual=res, rowstats_out=st, force_persistent=fp)
    out = ops.gemm(x, wg, bias=cvec, ln=(st, gvec, 1e-5), act=L.EA_ACT_GEGLU if geglu else L.EA_ACT_NONE,
                   force_persistent=fp)
    torch.cuda.synchronize()
    xr = x.float()                                     # what the consumer really read
    x_ref = a.float() @ w0.float().t() + b0 + res.float()
    y = F.layer_norm(xr, (C,), gam, bet, 1e-5) @ w1.t() + b1
    if geglu:
        y = y.reshape(M, N // 128, 2, 64)
        y = (y[:, :, 0] * F.gelu(y[:, :, 1])).reshape(M, N // 2)
    st_ref = torch.stack([x_ref.reshape(M, C // 32, 32).sum(-1), (x_ref ** 2).reshape(M, C // 32, 32).sum(-1)], -1).permute(1, 0, 2)
    r = {"x": _err(x, x_ref), "stats": _err(st, st_ref), "out": _err(out, y)}
    # the consumer multiplies fp16(W*gamma) while the reference rounds nothing: allow that extra rounding
    r["max_abs"] = max(r["x"]["max_abs"], r["out"]["max_abs"] / 2, r["stats"]["max_abs"] / 50)
    r["ref_max"] = max(1.0, y.abs().max().item() / 2)
    r["rel_fro"] = max(r["out"]["rel_fro"], r["stats"]["rel_fro"]) / 2
    return r


def case_ln_fold_linear():
    return _ln_fold_case(2048, 640, 1920, False, -1)


def case_ln_fold_linear_ragged():
    return _ln_fold_case(300, 320, 960, False, -1, seed=22)


def case_ln_fold_geglu():
    return _ln_fold_case(2048, 640, 5120, True, -1, seed=23)


def case_ln_fold_linear_persistent():
    return _ln_fold_case(2048, 640, 1920, False, 2, seed=24)


def case_ln_fold_geglu_persistent():
    return _ln_fold_case(8192, 320, 2560, True, 2, seed=25)


def case_ln_fold_geglu_persistent4():
    return _ln_fold_case(2048, 1280, 10240, True, 1, seed=26)


def case_step_gather_and_renoised_blend():
    """ea_step_gather (row *ctr of every table -> fixed buffers) and the re-noised, per-step gated inpaint blend
    + step counter of ea_out_cfg_ddim (utils/stable_diffusion_controlnet_inpaint.py:1647-1656)."""
    import torch
    import torch.nn.functional as F
    from editanything_b200 import ops
    dt = ops.half_dtype()
    torch.manual_seed(10)
    Nimg, H, C_ = 2, 16, 320
    tab_c = torch.rand(5, 8, device="cuda") * 0.5 + 0.3
    tab_c[:, 6] = torch.tensor([1.0, 1.0, 0.0, 1.0, 0.0])
    tab_e = torch.randn(5, 2, 1000, device="cuda")
    tab_f = torch.randn(5, 3, 37, device="cuda")
    coef, e_buf, f_buf = torch.zeros(8, device="cuda"), torch.zeros(2, 1000, device="cuda"), torch.zeros(3, 37, device="cuda")
    ctr = torch.zeros(1, device="cuda", dtype=torch.int32)
    xn = torch.randn(2 * Nimg, H, H, C_, device="cuda").to(dt)
    w = torch.randn(4, C_, 3, 3, device="cuda") / (9 * C_) ** 0.5
    b = torch.randn(4, device="cuda")
    lat = torch.randn(Nimg, H, H, 4, device="cuda")
    ref = lat.clone()
    known, noise = torch.randn(Nimg, H, H, 4, device="cuda"), torch.randn(Nimg, H, H, 4, device="cuda")
    mask = (torch.rand(Nimg, H, H, device="cuda") > 0.5).float()
    eps = F.conv2d(xn.float().permute(0, 3, 1, 2), w, b, padding=1).permute(0, 2, 3, 1)
    e = eps[:Nimg] + 7.0 * (eps[Nimg:] - eps[:Nimg])
    worst = 0.0
    for i in range(7):                    # two steps past the table: the row index clamps to the last row
        ops.step_gather(ctr, 5, [tab_c, tab_e, tab_f], [coef, e_buf, f_buf])
        ops.out_cfg_ddim(xn, w.permute(0, 2, 3, 1).contiguous(), b, latents=lat, coef=coef, guidance=7.0, known=known,
                         noise=noise, mask=mask, step_counter=ctr, Nimg=Nimg, H=H, W=H, C_=C_)
        torch.cuda.synchronize()
        r_ = min(i, 4)
        c = tab_c[r_]
        x0 = (ref - c[1] * e) / c[0]
        xp = c[2] * x0 + c[3] * e
        mk = mask[..., None] * c[6]
        ref = (c[4] * known + c[5] * noise) * mk + xp * (1 - mk)
        ref = ref.clamp(-50, 50)
        lat.clamp_(-50, 50)
        assert int(ctr.item()) == i + 1
        assert torch.equal(coef, tab_c[r_]) and torch.equal(e_buf, tab_e[r_]) and torch.equal(f_buf, tab_f[r_])
        worst = max(worst, ((lat - ref).abs().max() / ref.abs().max().clamp_min(1)).item())
        lat.copy_(ref)
    return {"max_abs": worst / 10, "ref_max": 1.0}


def _grouped_case(kind, seed=31, **force):
    """ea_gemm_grouped (3 networks, one launch) against three separate ea_gemm launches with the same plan:
    every output element is computed with the same K order, so the results must be bit-identical."""
    import torch
    from editanything_b200 import ops, _lib as L
    dt = ops.half_dtype()
    g = torch.Generator(device="cuda").manual_seed(seed)
    n = 3
    calls_a, calls_b = [], []
    outs_a, outs_b = [], []
    if kind == "linear":
        M, N, K = 2048, 640, 640
        for i in range(n):
            a = torch.randn(M, K, device="cuda", generator=g).to(dt)
            w = (torch.randn(N, K, device="cuda", generator=g) / K ** 0.5).to(dt)
            b = torch.randn(N, device="cuda", generator=g)
            r = torch.randn(M, N, device="cuda", generator=g).to(dt)
            o2 = torch.zeros(M, N, device="cuda", dtype=dt) if i == 0 else None
            kw = dict(bias=b, residual=r, **force)
            oa, ob = torch.full((M, N), 7.0, device="cuda", dtype=dt), torch.full((M, N), 7.0, device="cuda", dtype=dt)
            calls_a.append((a, w, oa, dict(kw, out2=o2) if o2 is not None else kw))
            calls_b.append((a, w, ob, kw))
            outs_a.append(oa); outs_b.append(ob)
    elif kind == "geglu":
        M, N, K = 2048, 5120, 640
        for i in range(n):
            a = torch.randn(M, K, device="cuda", generator=g).to(dt)
            w = (torch.randn(N, K, device="cuda", generator=g) / K ** 0.5).to(dt)
            b = torch.randn(N, device="cuda", generator=g)
            kw = dict(bias=b, act=L.EA_ACT_GEGLU, **force)
            oa, ob = torch.full((M, N // 2), 7.0, device="cuda", dtype=dt), torch.full((M, N // 2), 7.0, device="cuda", dtype=dt)
            calls_a.append((a, w, oa, kw)); calls_b.append((a, w, ob, kw))
            outs_a.append(oa); outs_b.append(ob)
    else:   # conv: 3x3 stride 1 with the time-embedding row vector; "conv8" = the split-K 8x8 level
        B, H, C, Cout = (2, 8, 1280, 1280) if kind == "conv8" else (2, 32, 640, 640)
        for i in range(n):
            x = torch.randn(B, H, H, C, device="cuda", generator=g).to(dt)
            w = (torch.randn(Cout, 9 * C, device="cuda", generator=g) / (9 * C) ** 0.5).to(dt)
            rv = torch.randn(B, Cout, device="cuda", generator=g)
            kw = dict(mode=L.EA_GEMM_CONV_S1, conv=(B, H, H, C), rowvec=rv, **force)
            oa = torch.full((B * H * H, Cout), 7.0, device="cuda", dtype=dt)
            ob = torch.full((B * H * H, Cout), 7.0, device="cuda", dtype=dt)
            calls_a.append((x, w, oa, kw)); calls_b.append((x, w, ob, kw))
            outs_a.append(oa); outs_b.append(ob)
    ops.gemm_grouped(calls_a)
    for a, w, o, kw in calls_b:
        ops.gemm(a, w, o, **kw)
    torch.cuda.synchronize()
    worst = max((x.float() - y.float()).abs().max().item() for x, y in zip(outs_a, outs_b))
    o2_ok = kind != "linear" or torch.equal(calls_a[0][3]["out2"], outs_a[0])
    if kind == "conv8":
        # K is split over the SMs that are left: three networks in one launch get a different split count than
        # one network alone, i.e. another fp32 summation order - compare with one output rounding of slack
        return {"max_abs": worst, "ref_max": max(o.float().abs().max().item() for o in outs_b)}
    ref = calls_b[1][0].float() @ calls_b[1][1].float().t() + calls_b[1][3]["bias"] + calls_b[1][3]["residual"].float() \
        if kind == "linear" else None
    r = _err(outs_b[1], ref) if ref is not None else {"max_abs": 0.0, "ref_max": 1.0}
    # same plan, same K order: grouped == separate to the last bit (x 1000 so that one differing ulp fails)
    return {"max_abs": worst * 1000 + r["max_abs"] + (0.0 if o2_ok else 1e3), "ref_max": r["ref_max"]}


def case_grouped_linear():
    return _grouped_case("linear", force_persistent=-1)


def case_grouped_linear_persistent():
    return _grouped_case("linear", seed=32, force_persistent=2)


def case_grouped_geglu_persistent():
    return _grouped_case("geglu", seed=34, force_persistent=2)


def case_grouped_geglu():
    return _grouped_case("geglu", seed=35, force_persistent=-1)


def case_grouped_conv():
    return _grouped_case("conv32", seed=36)


def case_grouped_conv_splitk():
    return _grouped_case("conv8", seed=37)


def case_groupnorm_stacked_nets():
    """ea_groupnorm with one (gamma, beta) per stacked network (ea_gn_args.n_nets)."""
    import torch
    import torch.nn.functional as F
    from editanything_b200 import ops
    dt = ops.half_dtype()
    torch.manual_seed(12)
    n, B, H, C_ = 3, 2, 16, 320
    x = (torch.randn(n * B, H, H, C_, device="cuda") * 1.5 + 0.3).to(dt)
    gam = [1 + 0.2 * torch.randn(C_, device="cuda") for _ in range(n)]
    bet = [0.2 * torch.randn(C_, device="cuda") for _ in range(n)]
    out = torch.empty_like(x)
    ws = ops.gn_workspace(n * B, "cuda")
    ops.groupnorm(x, gam, bet, out, B=n * B, HW=H * H, C_=C_, eps=1e-5, silu=True, workspace=ws)
    torch.cuda.synchronize()
    xs = x.float().permute(0, 3, 1, 2)
    ref = torch.cat([F.silu(F.group_norm(xs[g * B:(g + 1) * B], 32, gam[g], bet[g], 1e-5)) for g in range(n)]).permute(0, 2, 3, 1)
    return _err(out, ref)


def case_sam_helpers():
    import torch
    from editanything_b200 import ops
    dt = ops.half_dtype()
    torch.manual_seed(10)
    B, H, C_, ws = 2, 64, 64, 14
    x = torch.randn(B, H, H, C_, device="cuda").to(dt)
    nW = (H + ws - 1) // ws
    xw = torch.empty(B * nW * nW, ws, ws, C_, device="cuda", dtype=dt)
    ops.window_partition(x, xw, B=B, H=H, W=H, C_=C_, ws=ws)
    Hp = nW * ws
    xp = torch.nn.functional.pad(x, (0, 0, 0, Hp - H, 0, Hp - H))
    ref = xp.view(B, nW, ws, nW, ws, C_).permute(0, 1, 3, 2, 4, 5).reshape(-1, ws, ws, C_)
    r = {"partition": _err(xw, ref)}
    res = torch.randn(B, H, H, C_, device="cuda").to(dt)
    out = torch.empty(B, H, H, C_, device="cuda", dtype=dt)
    ops.window_unpartition(xw, res, out, B=B, H=H, W=H, C_=C_, ws=ws)
    r["unpartition"] = _err(out, x.float() + res.float())
    heads, S, d = 4, 14, 80
    q = torch.randn(3, S * S, heads * d, device="cuda").to(dt)
    Rh = torch.randn(S, S, d, device="cuda")
    Rw = torch.randn(S, S, d, device="cuda")
    rel_h = torch.empty(3 * heads, S * S, S, device="cuda")
    rel_w = torch.empty(3 * heads, S * S, S, device="cuda")
    ops.sam_relpos(q, S * S * heads * d, heads * d, Rh, Rw, rel_h, rel_w, B=3, heads=heads, S=S, d=d)
    torch.cuda.synchronize()
    qf = q.float().reshape(3, S, S, heads, d).permute(0, 3, 1, 2, 4).reshape(3 * heads, S, S, d)
    r["rel_h"] = _err(rel_h.reshape(3 * heads, S, S, S), torch.einsum("bhwc,hkc->bhwk", qf, Rh))
    r["rel_w"] = _err(rel_w.reshape(3 * heads, S, S, S), torch.einsum("bhwc,wkc->bhwk", qf, Rw))
    r["max_abs"] = max(v["max_abs"] / max(1.0, v["ref_max"]) for v in r.values())   # relative to magnitude
    r["ref_max"] = 1.0
    return r


CASES = {k[5:]: v for k, v in list(globals().items()) if k.startswith("case_") and callable(v)
         and k not in ("case_gemm_linear",)}


def main():
    os.makedirs(OUT, exist_ok=True)
    if len(sys.argv) >= 3 and sys.argv[1] == "--one":
        name = sys.argv[2]
        t0 = time.time()
        r = CASES[name]()
        r["case"] = name
        r["secs"] = round(time.time() - t0, 2)
        print("RESULT " + json.dumps(r))
        return
    names = sys.argv[1:] or list(CASES)
    log = open(os.path.join(OUT, "probe_ops.jsonl"), "a")
    for name in names:
        try:
            p = subprocess.run([sys.executable, os.path.abspath(__file__), "--one", name], capture_output=True,
                               text=True, timeout=240)
            line = [l for l in p.stdout.splitlines() if l.startswith("RESULT ")]
            if line:
                rec = json.loads(line[-1][7:])
            else:
                rec = {"case": name, "error": (p.stderr or p.stdout)[-1500:], "rc": p.returncode}
        except subprocess.TimeoutExpired:
            rec = {"case": name, "error": "timeout"}
        ok = "error" not in rec and rec.get("max_abs", 1e9) < 0.05 * max(1.0, rec.get("ref_max", 1.0))
        rec["ok"] = bool(ok)
        log.write(json.dumps(rec) + "\n")
        log.flush()
        short = {k: rec[k] for k in ("case", "ok", "max_abs", "ref_max", "rel_fro", "secs", "error") if k in rec}
        print(json.dumps(short)[:600], flush=True)


if __name__ == "__main__":
    main()
