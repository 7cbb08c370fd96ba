"""Micro-benchmarks of the C-ABI operators at the shapes of BASELINE.json configs[1]
(CUDA events on the launching stream, L2 flushed between iterations by cycling > L2 of operands).
Usage: python tools/bench_ops.py [attn] [gemm] [norm]"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from editanything_b200 import _lib as L  # noqa: E402
from editanything_b200 import ops  # noqa: E402


def timeit(fn, iters=20, warm=3):
    """Average device time of fn() in microseconds.  The calls are captured into ONE CUDA graph and
    the graph is replayed (the Python + ctypes + cuTensorMapEncode cost of a launch is ~25 us and
    would otherwise hide every kernel faster than that)."""
    iters = int(os.environ.get("EA_BENCH_ITERS", iters))
    warm = int(os.environ.get("EA_BENCH_WARM", warm))
    for _ in range(max(warm, 1)):
        fn()
    torch.cuda.synchronize()
    if os.environ.get("EA_BENCH_GRAPH", "1") == "0" or iters == 1:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / iters * 1e3
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
    torch.cuda.current_stream().wait_stream(s)
    with torch.cuda.graph(g):
        for _ in range(iters):
            fn()
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    g.replay()
    g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / (2 * iters) * 1e3  # us


def bench_attn():
    dt = ops.half_dtype()
    out = []
    # (name, B, heads, Nq, Nkv, d, fused_qkv).  fused_qkv: q, k and v are column slices of one [B, N, 3 C] projection
    # output, the layout of the step's self-attention (nets.py); B = 6 is the lockstep UNet encoder + 2 ControlNets.
    for name, B, h, Nq, Nkv, d, fused in [("self64 d40", 2, 8, 4096, 4096, 40, False),
                                          ("self64 d40 fused B6", 6, 8, 4096, 4096, 40, True),
                                          ("self64 d40 fused B2", 2, 8, 4096, 4096, 40, True),
                                          ("cross64 d40", 2, 8, 4096, 77, 40, False),
                                          ("cross64 d40 B6", 6, 8, 4096, 77, 40, False),
                                          ("self32 d80", 2, 8, 1024, 1024, 80, False), ("cross32 d80", 2, 8, 1024, 77, 80, False),
                                          ("self16 d160", 2, 8, 256, 256, 160, False), ("cross16 d160", 2, 8, 256, 77, 160, False),
                                          ("self8 d160", 2, 8, 64, 64, 160, False),
                                          ("sam_global d80", 1, 16, 4096, 4096, 80, False),
                                          ("sam_window d80", 25, 16, 196, 196, 80, False),
                                          ("self128 d40 (1024px)", 2, 8, 16384, 16384, 40, False)]:
        C_ = h * d
        if fused:
            qkv = torch.randn(B, Nq, 3 * C_, device="cuda").to(dt)
            q, k, v = qkv[..., :C_], qkv[..., C_:2 * C_], qkv[..., 2 * C_:]
            qs = ks = vs = (Nq * 3 * C_, 3 * C_)
        else:
            q = torch.randn(B, Nq, C_, device="cuda").to(dt)
            k = torch.randn(B, Nkv, C_, device="cuda").to(dt)
            v = torch.randn(B, Nkv, C_, device="cuda").to(dt)
            qs, ks, vs = (Nq * C_, C_), (Nkv * C_, C_), (Nkv * C_, C_)
        o = torch.empty(B, Nq, C_, device="cuda", dtype=dt)
        rel = {}
        if name.startswith("sam"):
            S = int(Nq ** 0.5)
            rel = dict(rel_h=torch.randn(B * h, Nq, S, device="cuda"), rel_w=torch.randn(B * h, Nq, S, device="cuda"), rel_s=S)

        def fn():
            ops.attention(q, k, v, o, B=B, heads=h, Nq=Nq, Nkv=Nkv, d=d, q_strides=qs, k_strides=ks, v_strides=vs,
                          o_strides=(Nq * C_, C_), scale=d ** -0.5, **rel)
        us = timeit(fn, iters=5 if Nq > 8000 else 20)
        fl = 4.0 * B * h * Nq * Nkv * d
        out.append({"op": "attn", "case": name, "us": round(us, 1), "tflops": round(fl / us / 1e6, 1)})
        print(json.dumps(out[-1]), flush=True)
    return out


def bench_gemm():
    dt = ops.half_dtype()
    out = []
    # conv3x3: (name, B, H, Cin, Cout)
    for name, B, H, Cin, Cout in [("conv64 320->320", 2, 64, 320, 320), ("conv64 640->320", 2, 64, 640, 320),
                                  ("conv64 960->320", 2, 64, 960, 320),
                                  ("conv32 640->640", 2, 32, 640, 640), ("conv32 1280->640", 2, 32, 1280, 640),
                                  ("conv16 1280->1280", 2, 16, 1280, 1280), ("conv16 2560->1280", 2, 16, 2560, 1280),
                                  ("conv8 1280->1280", 2, 8, 1280, 1280), ("conv8 2560->1280", 2, 8, 2560, 1280)]:
        n_w = max(1, int(300e6 // (Cout * 9 * Cin * 2)) + 1)   # cycle > L2 worth of weights: HBM-cold like the real step
        ws = [(torch.randn(Cout, 9 * Cin, device="cuda") / (9 * Cin) ** 0.5).to(dt) for _ in range(n_w)]
        x = torch.randn(B, H, H, Cin, device="cuda").to(dt)
        y = torch.empty(B, H, H, Cout, device="cuda", dtype=dt)
        bias = torch.randn(Cout, device="cuda")
        it = [0]

        def fn():
            ops.gemm(x, ws[it[0] % n_w], y, mode=L.EA_GEMM_CONV_S1, conv=(B, H, H, Cin), bias=bias)
            it[0] += 1
        us = timeit(fn)
        fl = 2.0 * B * H * H * Cout * 9 * Cin
        wb = Cout * 9 * Cin * 2
        out.append({"op": "conv3x3", "case": name, "us": round(us, 1), "tflops": round(fl / us / 1e6, 1),
                    "w_gbs": round(wb / us / 1e3, 1)})
        print(json.dumps(out[-1]), flush=True)
    # linear: (name, M, N, K, act)
    for name, M, N, K, act in [("qkv64", 8192, 960, 320, 0), ("ff1_64 geglu", 8192, 2560, 320, 3), ("ff2_64", 8192, 320, 1280, 0),
                               ("qkv32", 2048, 1920, 640, 0), ("ff1_32 geglu", 2048, 5120, 640, 3), ("ff2_32", 2048, 640, 2560, 0),
                               ("qkv16", 512, 3840, 1280, 0), ("ff1_16 geglu", 512, 10240, 1280, 3), ("ff2_16", 512, 1280, 5120, 0),
                               ("ff1_8 geglu", 128, 10240, 1280, 3), ("ff2_8", 128, 1280, 5120, 0),
                               ("sam_qkv", 4900, 3840, 1280, 0), ("sam_fc1", 4096, 5120, 1280, 2), ("sam_fc2", 4096, 1280, 5120, 0)]:
        n_w = max(1, int(300e6 // (N * K * 2)) + 1)
        ws = [(torch.randn(N, K, device="cuda") / K ** 0.5).to(dt) for _ in range(n_w)]
        x = torch.randn(M, K, device="cuda").to(dt)
        y = torch.empty(M, N // 2 if act == 3 else N, device="cuda", dtype=dt)
        bias = torch.randn(N, device="cuda")
        it = [0]

        def fn():
            ops.gemm(x, ws[it[0] % n_w], y, bias=bias, act=act)
            it[0] += 1
        us = timeit(fn)
        out.append({"op": "linear", "case": name, "us": round(us, 1), "tflops": round(2.0 * M * N * K / us / 1e6, 1),
                    "w_gbs": round(N * K * 2 / us / 1e3, 1)})
        print(json.dumps(out[-1]), flush=True)
    return out


def bench_norm():
    dt = ops.half_dtype()
    out = []
    for name, B, H, C_ in [("gn64 320", 2, 64, 320), ("gn64 960", 2, 64, 960), ("gn32 640", 2, 32, 640),
                           ("gn16 1280", 2, 16, 1280), ("gn8 2560", 2, 8, 2560)]:
        x = torch.randn(B, H, H, C_, device="cuda").to(dt)
        y = torch.empty_like(x)
        g, b = torch.randn(C_, device="cuda"), torch.randn(C_, device="cuda")
        ws = ops.gn_workspace(B, "cuda")
        us = timeit(lambda: ops.groupnorm(x, g, b, y, B=B, HW=H * H, C_=C_, workspace=ws))
        out.append({"op": "groupnorm", "case": name, "us": round(us, 1), "gbs": round(2 * x.numel() * 2 / us / 1e3, 1)})
        print(json.dumps(out[-1]), flush=True)
    for name, M, C_ in [("ln 8192x320", 8192, 320), ("ln 2048x640", 2048, 640), ("ln 512x1280", 512, 1280)]:
        x = torch.randn(M, C_, device="cuda").to(dt)
        y = torch.empty_like(x)
        g, b = torch.randn(C_, device="cuda"), torch.randn(C_, device="cuda")
        us = timeit(lambda: ops.layernorm(x, g, b, y, M=M, C_=C_))
        out.append({"op": "layernorm", "case": name, "us": round(us, 1), "gbs": round(2 * x.numel() * 2 / us / 1e3, 1)})
        print(json.dumps(out[-1]), flush=True)
    return out


if __name__ == "__main__":
    which = sys.argv[1:] or ["attn", "gemm", "norm"]
    res = []
    if "attn" in which:
        res += bench_attn()
    if "gemm" in which:
        res += bench_gemm()
    if "norm" in which:
        res += bench_norm()
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    tag = os.environ.get("EA_BENCH_TAG", "ops")
    json.dump(res, open(os.path.join(ROOT, "gpurun_out", f"bench_{tag}.json"), "w"), indent=1)
