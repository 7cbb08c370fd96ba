"""Generate tests/golden/sam_*.pt with the in-container HF port of SAM's image encoder
(transformers.models.sam.modeling_sam.SamVisionEncoder) — build container or GPU box, CPU only.

    python -m oracle.make_golden_sam [--full]

The reference's own dependency (`segment_anything`, un-vendored and un-pinned, README.md:235) is
absent, so the HF port — a line-for-line re-export of the same network — is the implementation
that is actually RUN to produce the vectors; weights are the deterministic synthetic ones of
editanything_b200.sam_spec.make_sam_state_dict.
"""
import os
import sys

import torch

from oracle.make_golden import golden_sample

from editanything_b200.sam_spec import SAM_TINY, SAM_VIT_H, make_sam_state_dict
from oracle import sam_oracle as S

GOLD = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
CASES = {"sam_tiny": (SAM_TINY, 2, 301, 5)}          # name -> (cfg, batch, weight seed, image seed)
FULL_CASES = {"sam_vit_h": (SAM_VIT_H, 1, 201, 6)}


def make_image(cfg, B, seed):
    """Preprocessed image as Sam.preprocess leaves it: per-channel normalised pixels, the bottom /
    right padding region exactly zero (SURVEY.md §3.5)."""
    g = torch.Generator().manual_seed(seed)
    img = torch.randn(B, cfg.in_chans, cfg.img_size, cfg.img_size, generator=g)
    pad = cfg.img_size // 4
    img[:, :, cfg.img_size - pad:, :] = 0.0
    return img


def run_case(name, spec):
    cfg, B, wseed, iseed = spec
    sd = make_sam_state_dict(cfg, wseed)
    img = make_image(cfg, B, iseed)
    m = S.hf_encoder(cfg, sd)
    with torch.no_grad():
        out = m(img).last_hidden_state
    rec = {"meta": dict(name=name, B=B, weight_seed=wseed, image_seed=iseed, generator="transformers SamVisionEncoder"),
           "embedding": out.to(torch.float16) if cfg.embed_dim >= 1280 else out.clone()}
    if name == "sam_vit_h":   # files stay below 1 MB: a fixed, seeded sample of 96 of the 256 channels
        idx = golden_sample(rec["embedding"].shape[1], 96, 1024)
        rec["embedding"] = rec["embedding"].index_select(1, idx).clone()
        rec["embedding_index"] = (1, idx)
    torch.save(rec, os.path.join(GOLD, name + ".pt"))
    print(name, tuple(out.shape), float(out.abs().max()), float(out.std()))


if __name__ == "__main__":
    os.makedirs(GOLD, exist_ok=True)
    torch.set_num_threads(os.cpu_count())
    for n, s in (FULL_CASES if "--full" in sys.argv else CASES).items():
        run_case(n, s)
