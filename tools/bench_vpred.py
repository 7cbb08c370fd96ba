"""Time the captured denoising step of an epsilon-prediction and a v-prediction model (SD2.1 768x768: 96x96 latents,
N = 4 images + classifier-free guidance, one ControlNet, synthetic weights).  The two variants share one set of packed
weights and differ only in the step's last kernel (ea_out_cfg_ddim against ea_out_cfg_vpred); each keeps its own
captured step, and they are timed in alternation (CUDA events over `--steps` graph replays, median of `--rounds`).

    python tools/bench_vpred.py [--steps 20] [--rounds 5] [--out DIR]

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
from editanything_b200.unet_spec import SD21, make_state_dict  # noqa: E402


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
    n = 4
    base = DenoiseEngine(SD21, make_state_dict(SD21, "unet", 101), [make_state_dict(SD21, "controlnet", 102)], dev)
    ts, a, ap_ = ddim_schedule(50)
    g = torch.Generator().manual_seed(11)
    ctx = torch.randn(2 * n, 77, SD21.context_dim, generator=g)
    hints = [torch.randint(0, 256, (2 * n, 3, 768, 768), generator=g).float()]
    lat = torch.randn(n, 4, 96, 96, generator=g)
    variants = {}
    for pt in ("epsilon", "v_prediction"):
        eng = base if not variants else DenoiseEngine(SD21, None, None, dev, unet_packed=base.unet,
                                                     controlnets_packed=base.cns)
        eng.prepare(ctx, hints, [1.0])
        eng.set_schedule(ts, a, ap_, prediction_type=pt)
        eng.begin(lat, guidance=7.5, use_graph=True)
        for _ in range(3):
            eng.step()                     # capture + warm-up
        variants[pt] = eng
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
    res = {"card": _card(), "config": "sd21_768 N=4 + CFG, 1 ControlNet, captured step", "steps": args.steps,
           "rounds": args.rounds, "ms_per_step": {}}
    for k, v in times.items():
        res["ms_per_step"][k] = {"median": round(statistics.median(v), 3), "min": round(min(v), 3),
                                 "max": round(max(v), 3)}
    m = res["ms_per_step"]
    res["v_over_epsilon"] = round(m["v_prediction"]["median"] / m["epsilon"]["median"], 4)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_vpred.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
