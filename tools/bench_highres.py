"""High-resolution tile refinement on one GPU: the SD VAE's mid-block attention, VAE encode + decode, and the tile
pass's denoising step, with the peak allocation of each.

  * attention: the fused ea_attention launch (one head of d = 512 over q / k / v slices of one [N, 3 * 512] buffer)
    against the GEMM -> softmax_rows -> GEMM sequence the AttnBlock ran before (fp32 N x N logits, half P), re-enacted
    here through ops.gemm / ops.softmax_rows, alternating, at 64^2, 128^2 and 192 x 256 latents;
  * VAE encode + decode (graphs on; the AttnBlock takes the path vae.py selects for the size) and the captured
    denoising step of the tile pass (SD1.5 full size, one ControlNet, 1 image + CFG, synthetic weights) at 1024^2,
    1536 x 2048 and 2048 x 2752, `--reps` calls per timed window.
The GEMM sequence is not run where its N x N buffers alone would not fit on an 80 GB card.

    python tools/bench_highres.py [--reps 10] [--rounds 5] [--out DIR]

Prints one JSON line with the card name and power limit beside the numbers."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from editanything_b200 import ops  # noqa: E402
from editanything_b200.denoise import DenoiseEngine, ddim_schedule  # noqa: E402
from editanything_b200.unet_spec import SD15, make_state_dict  # noqa: E402
from editanything_b200.vae import SD_VAE, VaeEngine, make_vae_state_dict  # noqa: E402

C = 512
ATTN_LATENTS = [(64, 64), (128, 128), (192, 256)]
IMAGE_SIZES = [(1024, 1024), (1536, 2048), (2048, 2752)]     # (height, width)


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def _time(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def _stats(v):
    return {"median": round(statistics.median(v), 3), "min": round(min(v), 3), "max": round(max(v), 3)}


def _peak(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return round(torch.cuda.max_memory_allocated() / 2**30, 2)


def bench_attention(reps, rounds):
    dev = torch.device("cuda:0")
    hdt = ops.half_dtype()
    out = {}
    g = torch.Generator(device=dev).manual_seed(0)
    wv = (torch.randn(C, C, device=dev, generator=g) * C ** -0.5).to(hdt)
    bv = torch.randn(C, device=dev, generator=g) * 0.1
    for h, w in ATTN_LATENTS:
        n = h * w
        qkv = torch.randn(n, 3 * C, device=dev, generator=g).to(hdt)
        hn = qkv[:, 2 * C:].contiguous()       # the GroupNorm output the parent projected V from
        ao = torch.empty(n, C, device=dev, dtype=hdt)
        st = (n * 3 * C, 3 * C)

        def fused():
            ops.attention(qkv, qkv[:, C:], qkv[:, 2 * C:], ao, B=1, heads=1, Nq=n, Nkv=n, d=C, q_strides=st,
                          k_strides=st, v_strides=st, o_strides=(n * C, C), scale=C ** -0.5)

        ways = {"fused": fused}
        if 6 * n * n < 60 * 2**30:
            s = torch.empty(n, n, device=dev, dtype=torch.float32)
            pr = torch.empty(n, n, device=dev, dtype=hdt)
            vt = torch.empty(C, n, device=dev, dtype=hdt)
            ao2 = torch.empty(n, C, device=dev, dtype=hdt)

            def gemm_softmax_gemm():
                ops.gemm(qkv[:, :C], qkv[:, C:2 * C], out_f32=s, K=C, lda=3 * C, ldw=3 * C, out_scale=C ** -0.5)
                ops.softmax_rows(s, pr, rows=n, cols=n)
                ops.gemm(wv, hn, vt)
                ops.gemm(pr, vt, ao2, bias=bv)

            ways["gemm_softmax_gemm"] = gemm_softmax_gemm
        for fn in ways.values():
            fn()
        torch.cuda.synchronize()
        times = {k: [] for k in ways}
        for _ in range(rounds):
            for k, fn in ways.items():
                times[k].append(_time(fn, reps))
        res = {k: _stats(v) for k, v in times.items()}
        if "gemm_softmax_gemm" not in ways:
            res["gemm_softmax_gemm"] = "not run: its N x N buffers do not fit"
        else:
            res["fused_over_gemm_softmax_gemm"] = round(res["fused"]["median"] /
                                                        res["gemm_softmax_gemm"]["median"], 3)
        out[f"{h}x{w}"] = res
        del qkv, hn, ao
        ways.clear()
        torch.cuda.empty_cache()
    return out


def bench_sizes(reps, rounds):
    dev = torch.device("cuda:0")
    vsd = dict(make_vae_state_dict(SD_VAE, 412, part="encoder", device=dev))
    vsd.update(make_vae_state_dict(SD_VAE, 402, device=dev))
    vae = VaeEngine(SD_VAE, vsd, dev)
    eng = DenoiseEngine(SD15, make_state_dict(SD15, "unet", 201), [make_state_dict(SD15, "controlnet", 202)], dev)
    ts, a, ap_ = ddim_schedule(30)
    out = {}
    g = torch.Generator().manual_seed(0)
    for hh, ww in IMAGE_SIZES:
        x = (torch.rand(1, 3, hh, ww, generator=g) * 2 - 1).to(dev)
        lat = torch.randn(1, 4, hh // 8, ww // 8, generator=g).to(dev)
        res = {"latents": f"{hh // 8}x{ww // 8}"}
        res["vae_encode_peak_gib"] = _peak(lambda: vae.encode(x))
        res["vae_decode_peak_gib"] = _peak(lambda: vae.decode_latents(lat))
        enc, dec = [], []
        for _ in range(rounds):
            enc.append(_time(lambda: vae.encode(x), reps))
            dec.append(_time(lambda: vae.decode_latents(lat), reps))
        res["vae_encode_ms"], res["vae_decode_ms"] = _stats(enc), _stats(dec)
        ctx = torch.randn(2, 77, 768, generator=g)
        hints = [torch.rand(2, 3, hh, ww, generator=g)]
        eng.prepare(ctx, hints, [1.0])
        eng.set_schedule(ts, a, ap_)
        eng.begin(lat.cpu(), guidance=9.0, use_graph=True)

        def step():
            eng.step()
        res["step_peak_gib"] = _peak(lambda: [step() for _ in range(3)])   # capture + warm-up
        steps = []
        for _ in range(rounds):
            eng.step_ctr.zero_()
            steps.append(_time(step, reps))
        res["step_ms"] = _stats(steps)
        out[f"{hh}x{ww}"] = res
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("needs a GPU: nothing is measured without one")
    res = {"card": _card(), "reps": args.reps, "rounds": args.rounds,
           "attention_ms": bench_attention(args.reps, args.rounds),
           "sizes": bench_sizes(args.reps, args.rounds)}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_highres.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
