"""Time the captured denoising step of text-to-image generation (all-region generation: SD1.5 512x512, the SAM
ControlNet alone, synthetic weights) at N = 1 and N = 4 images with guess mode off and on, beside the inpaint
pipeline's step (SAM + inpaint ControlNets) at N = 1, all with classifier-free guidance.  In guess mode the ControlNet
still runs on all 2N rows; only its zero-convs skip the unconditional half.  The variants share one set of packed
weights, each keeps its own captured step, and they are timed in alternation (CUDA events over `--steps` graph
replays, median and min-max of `--rounds`).  Then `EditAnythingLoraModel.process(enable_all_generate=True)` end to end
at 512x512, 20 steps, 2 images, `--rounds` calls each: without the tile pass, and with it at the demo's defaults
(refine_image_resolution 1024, refine_alignment_ratio 0.95: one 1024x1024 tile-ControlNet pass per image, VAE
encode and decode included).  SAM is a stand-in mask generator (bench.py times the ViT-H encode), and the text
encoder a stand-in embedding.

    python tools/bench_txt2img.py [--steps 20] [--rounds 5] [--out DIR]

Prints one JSON line with the card name and power limit beside the numbers."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time
from types import SimpleNamespace

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from editanything_b200.denoise import DenoiseEngine, ddim_schedule  # noqa: E402
from editanything_b200.unet_spec import SD15, make_state_dict  # noqa: E402


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def _stats(v):
    return {"median": round(statistics.median(v), 3), "min": round(min(v), 3), "max": round(max(v), 3)}


class _Sam:
    """A stand-in automatic mask generator: three fixed rectangles."""

    def generate(self, image):
        h, w = image.shape[:2]
        out = []
        for i, (y0, x0, dy, dx) in enumerate([(0, 0, h // 2, w // 2), (h // 4, w // 4, h // 2, w // 2)]):
            m = np.zeros((h, w), dtype=bool)
            m[y0:y0 + dy, x0:x0 + dx] = True
            out.append({"segmentation": m, "area": int(m.sum()) + i})
        return out


class _Tok:
    model_max_length = 77

    def __call__(self, text, padding=None, max_length=None, truncation=True, return_tensors="pt"):
        ids = [1] + [3 + sum(map(ord, w)) % 400 for w in text.split()][:75] + [2]
        return SimpleNamespace(input_ids=torch.tensor([ids + [0] * ((max_length or len(ids)) - len(ids))]))


class _Enc(torch.nn.Module):
    def __init__(self, dim):
        super().__init__()
        torch.manual_seed(0)
        self.emb = torch.nn.Embedding(512, dim)

    def forward(self, ids):
        return (self.emb(ids.to(self.emb.weight.device)),)


def bench_steps(args, dev):
    base = DenoiseEngine(SD15, make_state_dict(SD15, "unet", 101),
                         [make_state_dict(SD15, "controlnet", s) for s in (102, 103)], dev)
    ts, a, ap_ = ddim_schedule(50)
    g = torch.Generator().manual_seed(11)
    variants = {}
    for n in (1, 4):
        ctx = torch.randn(2 * n, 77, SD15.context_dim, generator=g)
        sam = torch.randint(0, 256, (n, 3, 512, 512), generator=g).float()
        lat = torch.randn(n, 4, 64, 64, generator=g)
        for guess in (False, True):
            eng = DenoiseEngine(SD15, None, None, dev, unet_packed=base.unet, controlnets_packed=base.cns[:1])
            if guess:
                eng.prepare(ctx, [sam], [1.0], guess_mode=True, controlnet_rows="conditional")
            else:
                eng.prepare(ctx, [torch.cat([sam, sam])], [1.0], cfg_duplicated=True)
            variants[f"txt2img_N{n}_guess_{'on' if guess else 'off'}"] = (eng, lat)
        if n == 1:
            inp = torch.rand(2, 3, 512, 512, generator=g)
            base.prepare(ctx, [torch.cat([sam, sam]), inp], [1.0, 1.0], cfg_duplicated=True)
            variants["inpaint_2cn_N1"] = (base, lat)
    for eng, lat in variants.values():
        eng.set_schedule(ts, a, ap_)
        eng.begin(lat, guidance=7.5, use_graph=True)
        for _ in range(3):
            eng.step()                     # capture + warm-up
    torch.cuda.synchronize()
    times = {k: [] for k in variants}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(args.rounds):
        for k, (eng, _) in variants.items():
            eng.step_ctr.zero_()
            e0.record()
            for _ in range(args.steps):
                eng.step()
            e1.record()
            torch.cuda.synchronize()
            times[k].append(e0.elapsed_time(e1) / args.steps)
    out = {k: dict(_stats(v), launches=variants[k][0].launches_per_step) for k, v in times.items()}
    del base, variants
    torch.cuda.empty_cache()
    return out


def bench_process(args, dev):
    from editanything_b200 import app
    from editanything_b200.pipeline import StableDiffusionControlNetInpaintPipeline, StableDiffusionControlNetPipeline
    from editanything_b200.schedulers import UniPCMultistepScheduler
    from editanything_b200.vae import VaeEngine, make_vae_state_dict
    from editanything_b200.vae_spec import VaeConfig
    vcfg = VaeConfig()
    vsd = dict(make_vae_state_dict(vcfg, 61, part="encoder"))
    vsd.update(make_vae_state_dict(vcfg, 62))
    eng = DenoiseEngine(SD15, make_state_dict(SD15, "unet", 101), [make_state_dict(SD15, "controlnet", 102)], dev)
    tile_eng = DenoiseEngine(SD15, None, [make_state_dict(SD15, "controlnet", 104)], dev, unet_packed=eng.unet)
    vae, enc, tok = VaeEngine(vcfg, vsd, dev), _Enc(SD15.context_dim).to(dev), _Tok()
    pipe = StableDiffusionControlNetPipeline(eng, vae=vae, text_encoder=enc, tokenizer=tok)
    tile = StableDiffusionControlNetInpaintPipeline(tile_eng, vae=vae, text_encoder=enc, tokenizer=tok)
    for p in (pipe, tile):
        p.scheduler = UniPCMultistepScheduler.from_config(p.scheduler.config)
    model = app.EditAnythingLoraModel(base_model_path="base", lora_model_path=None, use_blip=False,
                                      sam_generator=_Sam(), mask_predictor=object(), tile_model=tile, pipe=pipe)
    model.defalut_enable_all_generate = True      # the pipeline is already the text-to-image one: no rebuild
    image = np.random.RandomState(0).randint(0, 256, (512, 512, 3)).astype(np.uint8)
    a = ({"image": image, "mask": np.zeros_like(image)}, True, None, 1.0, False, "a photo of a house", "lowres", 2,
         512, 512, 20, False, 7.5, 1234, 0.0)
    os.environ["EA_SAVE_INPUT"] = "0"
    variants = {"without_tile_pass": dict(enable_tile=False),
                "with_tile_pass_1024": dict(enable_tile=True, refine_alignment_ratio=0.95, refine_image_resolution=1024)}
    for kw in variants.values():
        model.process(*a, **kw)                   # capture + warm-up
    t = {k: [] for k in variants}
    for _ in range(args.rounds):
        for k, kw in variants.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            model.process(*a, **kw)
            torch.cuda.synchronize()
            t[k].append((time.perf_counter() - t0) * 1e3)
    return {k: _stats(v) for k, v in t.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("needs a GPU: nothing is measured without one")
    dev = torch.device("cuda:0")
    res = {"card": _card(), "config": "sd15_512, captured step with CFG; txt2img = SAM ControlNet only",
           "steps": args.steps, "rounds": args.rounds, "ms_per_step": bench_steps(args, dev)}
    m = res["ms_per_step"]
    for n in (1, 4):
        res[f"N{n}_guess_on_over_off"] = round(m[f"txt2img_N{n}_guess_on"]["median"] /
                                               m[f"txt2img_N{n}_guess_off"]["median"], 3)
    res["process_all_generate_ms"] = dict(bench_process(args, dev), images=2, steps=20, size=512,
                                          note="SAM and the text encoder are stand-ins; VAE included")
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_txt2img.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
