"""Time every distinct ea_gemm launch of one bench denoising step (SD1.5, 64x64 latents, CFG batch 2, two ControlNets)
with one row tile per CTA (force_2cta = -1), two row tiles per CTA (+1) and the planner's choice (0).

The launches are recorded from the engine exactly as bench.py's roofline probe records them.  Each distinct launch is
re-issued REPS times inside one CUDA graph and the replays are timed with CUDA events, so host overhead is excluded.
Prints one line per shape (count per step, microseconds per launch, achieved TFLOP/s, algorithmic bytes) and the
per-step totals, with the card name and power limit read in the same run.  Usage (on an H100):

    python tools/gemm_rowpair_ab.py [--reps 20] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

VARIANTS = (-1, 1, 0)


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def _rows(a, kw):
    conv = kw.get("conv")
    return conv[0] * conv[1] * conv[2] if conv else (kw.get("M") or a.shape[0])


def _bytes(a, w, kw):
    """Operands the algorithm needs: A + W + output (+ residual), fp16."""
    conv = kw.get("conv")
    m = _rows(a, kw)
    k_in = conv[3] if conv else w.shape[1]
    n_out = w.shape[0] // 2 if kw.get("act") == 3 else w.shape[0]
    return 2 * (m * k_in + w.numel() + m * n_out * (2 if kw.get("residual") is not None else 1))


def _key(rec):
    calls = rec[1] if rec[0] == "grouped" else [rec[:4]]
    a, w, _, kw = calls[0]
    return (len(calls), kw.get("mode", 0), _rows(a, kw), w.shape[0], w.shape[1], kw.get("act", 0),
            kw.get("residual") is not None, kw.get("ln") is not None, kw.get("rowstats_out") is not None)


def _issue(ops, rec, f2):
    if rec[0] == "grouped":
        ops.gemm_grouped([(a, w, o, dict(kw, force_2cta=f2)) for a, w, o, kw in rec[1]])
    else:
        a, w, out, kw, _ = rec
        ops.gemm(a, w, out, **dict(kw, force_2cta=f2))


def _time_us(ops, rec, f2, reps):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _issue(ops, rec, f2)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(reps):
            _issue(ops, rec, f2)
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    best = float("inf")
    for _ in range(5):
        e0.record()
        g.replay()
        e1.record()
        torch.cuda.synchronize()
        best = min(best, e0.elapsed_time(e1) * 1e3 / reps)
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None, help="directory for gemm_rowpair_ab.json")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    import bench
    from editanything_b200 import ops
    from editanything_b200.denoise import DenoiseEngine, ddim_schedule
    from editanything_b200.unet_spec import SD15, make_state_dict

    card = _card()
    dev = torch.device("cuda:0")
    usd = make_state_dict(SD15, "unet", 101, device=dev)
    csds = [make_state_dict(SD15, "controlnet", c, device=dev) for c in (102, 103)]
    eng = DenoiseEngine(SD15, usd, csds, dev)
    del usd, csds
    x, ctx, hints = bench.make_inputs(SD15, 2, 64, 77, 11)
    ts, a, ap_ = ddim_schedule(bench.DDIM_STEPS)
    eng.prepare(ctx, hints, [0.5, 1.0], cfg_duplicated=True)
    eng.set_schedule(ts, a, ap_)
    probe = bench.GemmProbe(ops)
    eng.ops = eng.runner.ops = eng.unet.ops = probe
    for c in eng.cns:
        c.ops = probe
    eng.begin(x[:1], guidance=9.0, use_graph=False)
    eng.step(int(ts[0]), float(a[0]), float(ap_[0]))
    probe.records.clear()
    eng.step(int(ts[1]), float(a[1]), float(ap_[1]))
    torch.cuda.synchronize()

    shapes = {}
    for rec in probe.records:
        k = _key(rec)
        if k not in shapes:
            calls = rec[1] if rec[0] == "grouped" else [rec[:4]]
            shapes[k] = {"rec": rec, "count": 0, "flop": rec[4],
                         "bytes": sum(_bytes(a_, w_, kw_) for a_, w_, _, kw_ in calls)}
        shapes[k]["count"] += 1

    print(f"card: {card}; {len(probe.records)} GEMM launches per step, {len(shapes)} distinct")
    print(f"{'groups mode M N K act res ln st':>44} {'n':>3} " +
          " ".join(f"{'us(' + str(v) + ')':>9} {'TF/s':>6}" for v in VARIANTS) + f" {'MB':>7}")
    rows, tot = [], {v: 0.0 for v in VARIANTS}
    for k, sh in shapes.items():
        us = {v: _time_us(ops, sh["rec"], v, args.reps) for v in VARIANTS}
        for v in VARIANTS:
            tot[v] += sh["count"] * us[v]
        rows.append({"key": list(k), "count": sh["count"], "flop": sh["flop"], "alg_bytes": sh["bytes"],
                     "us": {str(v): us[v] for v in VARIANTS}})
        print(f"{str(k):>44} {sh['count']:>3} " +
              " ".join(f"{us[v]:9.1f} {sh['flop'] / us[v] * 1e-6:6.0f}" for v in VARIANTS) +
              f" {sh['bytes'] / 1e6:7.1f}")
    best = sum(r["count"] * min(r["us"][str(v)] for v in (-1, 1)) for r in rows)
    print("per step (ms): " + ", ".join(f"force_2cta={v}: {tot[v] / 1e3:.3f}" for v in VARIANTS) +
          f", best of -1/+1 per shape: {best / 1e3:.3f}")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "gemm_rowpair_ab.json"), "w") as f:
            json.dump({"card": card, "reps": args.reps, "shapes": rows,
                       "step_ms": {str(v): tot[v] / 1e3 for v in VARIANTS}, "best_ms": best / 1e3}, f, indent=1)


if __name__ == "__main__":
    main()
