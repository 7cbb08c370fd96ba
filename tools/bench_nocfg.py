"""Time the captured denoising step with and without classifier-free guidance (SD1.5 512x512, 2 ControlNets, the
flagship shapes of bench.py, synthetic weights) at N = 1 and N = 4 images.  Guided steps run the networks on 2N rows,
unguided ones on N.  The four variants share one set of packed weights, each keeps its own captured step, and they
are timed in alternation (CUDA events over `--steps` graph replays, median of `--rounds`).

    python tools/bench_nocfg.py [--steps 20] [--rounds 5] [--out DIR]

Prints one JSON line with the card name and power limit beside the numbers."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from editanything_b200.denoise import DenoiseEngine, ddim_schedule  # noqa: E402
from editanything_b200.unet_spec import SD15, make_state_dict  # noqa: E402


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("needs a GPU: nothing is measured without one")
    dev = torch.device("cuda:0")
    base = DenoiseEngine(SD15, make_state_dict(SD15, "unet", 101),
                         [make_state_dict(SD15, "controlnet", s) for s in (102, 103)], dev)
    ts, a, ap_ = ddim_schedule(50)
    g = torch.Generator().manual_seed(11)
    variants = {}
    for n in (1, 4):
        ctx = torch.randn(2 * n, 77, SD15.context_dim, generator=g)
        hints = [torch.randint(0, 256, (2 * n, 3, 512, 512), generator=g).float(), torch.rand(2 * n, 3, 512, 512, generator=g)]
        lat = torch.randn(n, 4, 64, 64, generator=g)
        for guided in (True, False):
            eng = base if not variants else DenoiseEngine(SD15, None, None, dev, unet_packed=base.unet,
                                                         controlnets_packed=base.cns)
            c, h = (ctx, hints) if guided else (ctx[n:], [x[n:] for x in hints])
            eng.prepare(c, h, [0.5, 1.0], guided=guided)
            eng.set_schedule(ts, a, ap_)
            eng.begin(lat, guidance=7.5, use_graph=True)
            for _ in range(3):
                eng.step()                     # capture + warm-up
            variants[(n, guided)] = eng
    torch.cuda.synchronize()
    times = {k: [] for k in variants}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(args.rounds):
        for k, eng in variants.items():
            eng.step_ctr.zero_()
            e0.record()
            for _ in range(args.steps):
                eng.step()
            e1.record()
            torch.cuda.synchronize()
            times[k].append(e0.elapsed_time(e1) / args.steps)
    res = {"card": _card(), "config": "sd15_512 2 ControlNets, captured step", "steps": args.steps,
           "rounds": args.rounds, "ms_per_step": {}}
    for (n, guided), v in times.items():
        res["ms_per_step"][f"N{n}_{'guided' if guided else 'unguided'}"] = {
            "median": round(statistics.median(v), 3), "min": round(min(v), 3), "max": round(max(v), 3),
            "network_rows": 2 * n if guided else n}
    for n in (1, 4):
        m = res["ms_per_step"]
        res[f"N{n}_unguided_over_guided"] = round(m[f"N{n}_unguided"]["median"] / m[f"N{n}_guided"]["median"], 3)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_nocfg.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
