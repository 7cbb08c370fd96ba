"""Time the captured denoising step of the alpha-mixing inpaint pipeline against the plain inpaint pipeline's step
(SD1.5, synthetic weights, classifier-free guidance, a 20-step DDIM schedule): at 512x512 with the SAM and inpaint
ControlNets for N = 1 and N = 4 images, and at the 1024x1024 tile pass (one tile ControlNet, N = 1).  The two steps
share the packed weights and differ by one launch, ea_latent_mix after the update.  Each variant keeps its own
captured step; they are timed in alternation (CUDA events over `--steps` graph replays, median and min-max of
`--rounds`).  The kernel alone is timed too: CUDA events over 10 replays of a graph of 100 launches on the same
buffers, against the bytes it moves (latents read and written, known, noise row, mask, both half copies), for its
share of HBM bandwidth.

    python tools/bench_mixing.py [--steps 19] [--rounds 7] [--out DIR]

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

HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def _stats(v):
    return {"median": round(statistics.median(v), 4), "min": round(min(v), 4), "max": round(max(v), 4)}


def _start(eng, lat, known, mask, mixing, S):
    """One request: the plain inpaint schedule (blend window 0.95) or the mixing one (mix after every step but the
    last, alpha 0.5), then the capture and two warm-up replays."""
    ts, a, ap = ddim_schedule(S)
    n = len(ts)
    k = [(0.9, 0.3)] * n
    if mixing:
        eng.set_schedule(ts, a, ap, mix=([x[0] for x in k], [x[1] for x in k],
                                         [1.0 if i < 0.95 * n else 0.0 for i in range(n)], [1.0] * (n - 1) + [0.0]))
        z = torch.randn((n - 1,) + tuple(lat.shape), device=eng.dev)
        eng.begin(lat, 7.5, known_nchw=known, mask_n1hw=mask, mix_alpha=0.5, mix_noise=z)
    else:
        on = [1.0 if i < 0.95 * n else 0.0 for i in range(n)]
        eng.set_schedule(ts, a, ap, blend=([x[0] for x in k], [x[1] for x in k], on))
        eng.begin(lat, 7.5, known_nchw=known, mask_n1hw=mask, noise_nchw=torch.randn_like(lat))
    for _ in range(3):
        eng.step()
    return n


def bench_steps(args, dev):
    base = DenoiseEngine(SD15, make_state_dict(SD15, "unet", 101),
                         [make_state_dict(SD15, "controlnet", s) for s in (102, 103)], dev)
    g = torch.Generator().manual_seed(11)
    cases = {}
    for name, n, size, n_cn in (("512_N1", 1, 512, 2), ("512_N4", 4, 512, 2), ("tile_1024_N1", 1, 1024, 1)):
        ctx = torch.randn(2 * n, 77, SD15.context_dim, generator=g)
        hints = [torch.rand(n, 3, size, size, generator=g) * (255 if i == 0 else 1) for i in range(n_cn)]
        h = size // 8
        lat, known = torch.randn(n, 4, h, h, generator=g), torch.randn(n, 4, h, h, generator=g)
        mask = torch.zeros(n, 1, h, h)
        mask[..., h // 4:3 * h // 4, h // 4:3 * h // 4] = 1.0
        for mixing in (False, True):
            eng = DenoiseEngine(SD15, None, None, dev, unet_packed=base.unet, controlnets_packed=base.cns[:n_cn])
            eng.prepare(ctx, [torch.cat([x, x]) for x in hints], [1.0] * n_cn, cfg_duplicated=True)
            cases[(name, mixing)] = (eng, lat, known, mask)
    times = {k: [] for k in cases}
    steps = {}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for r in range(args.rounds + 1):               # round 0: capture and warm-up, not recorded
        for key, (eng, lat, known, mask) in cases.items():
            steps[key] = _start(eng, lat, known, mask, key[1], args.steps + 1)
            eng.step_ctr.zero_()
            torch.cuda.synchronize()
            e0.record()
            for _ in range(args.steps):
                eng.step()
            e1.record()
            torch.cuda.synchronize()
            if r:
                times[key].append(e0.elapsed_time(e1) / args.steps)
    out = {}
    for name in dict.fromkeys(k[0] for k in cases):
        p, m = (cases[(name, x)][0] for x in (False, True))
        tp, tm = statistics.median(times[(name, False)]), statistics.median(times[(name, True)])
        out[name] = {"plain_inpaint": dict(_stats(times[(name, False)]), launches=p.launches_per_step),
                     "mixing": dict(_stats(times[(name, True)]), launches=m.launches_per_step),
                     "mixing_minus_plain_ms": round(tm - tp, 4)}
    kernel = {}
    for name in dict.fromkeys(k[0] for k in cases):
        eng = cases[(name, True)][0]
        n_px = eng.lat.numel() // 4
        kw = dict(alpha=0.5, step_counter=eng.step_ctr, lat_half_out=eng.x_half, copies=2, Nimg=eng.lat.shape[0],
                  H=eng.lat.shape[1], W=eng.lat.shape[2])
        eng.step_ctr.fill_(1)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(20):
                ops.latent_mix(eng.lat, eng.known, eng.mask, eng.mix_noise, eng.mix_tab, **kw)
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()        # 100 launches in one graph: the kernel, not the host's launch rate
        with torch.cuda.graph(graph):
            for _ in range(100):
                ops.latent_mix(eng.lat, eng.known, eng.mask, eng.mix_noise, eng.mix_tab, **kw)
        graph.replay()
        torch.cuda.synchronize()
        e0.record()
        for _ in range(10):
            graph.replay()
        e1.record()
        torch.cuda.synchronize()
        us = e0.elapsed_time(e1)             # ms for 1000 launches = us per launch
        nbytes = n_px * (16 * 4 + 4 + 2 * 8)     # latents r+w, known, noise row (fp32 x4); mask; 2 half copies
        kernel[name] = {"us_per_launch": round(us, 3), "bytes": nbytes,
                        "share_of_hbm_peak": round(nbytes / (us * 1e-6) / HBM_BYTES_PER_S, 3)}
    return out, kernel


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=19)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("needs a GPU: nothing is measured without one")
    dev = torch.device("cuda:0")
    steps, kernel = bench_steps(args, dev)
    res = {"card": _card(), "config": "sd15, captured step with CFG, DDIM; 512: SAM + inpaint ControlNets, "
                                      "tile_1024: one ControlNet", "steps": args.steps, "rounds": args.rounds,
           "ms_per_step": steps, "ea_latent_mix": kernel}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_mixing.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
