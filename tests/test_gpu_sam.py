"""-m gpu: the SAM ViT image encoder on the CUDA path against the HF-generated golden vectors and
the CPU oracle.

Tolerance: BASELINE.json's SAM gate is mask IoU >= 0.999, which needs real SAM weights and the mask
decoder (neither exists in this environment).  With synthetic weights the gate is on the encoder
output itself (the tensor the mask decoder consumes, LayerNorm2d-normalised to O(1)): max-abs
< 3e-2 and relative Frobenius error < 5e-3 in fp16 storage / fp32 accumulation vs the fp32 reference."""
import os

import pytest
import torch

from editanything_b200.sam import SamEncoderEngine
from editanything_b200.sam_spec import SAM_TINY, SAM_VIT_H, make_sam_state_dict
from oracle import sam_oracle as S
from oracle.make_golden_sam import make_image

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
MAX_ABS, REL_FRO = 3e-2, 5e-3


def _check(out, ref, what):
    out, ref = out.float().cpu(), ref.float()
    err = (out - ref).abs().max().item()
    rel = ((out - ref).norm() / ref.norm()).item()
    print(f"{what}: max-abs {err:.3e} rel-fro {rel:.3e} ref-max {ref.abs().max().item():.2f}")
    assert err < MAX_ABS and rel < REL_FRO, (what, err, rel)


def test_tiny_encoder_vs_golden_and_oracle():
    g = torch.load(os.path.join(GOLD, "sam_tiny.pt"))
    m = g["meta"]
    sd = make_sam_state_dict(SAM_TINY, m["weight_seed"])
    eng = SamEncoderEngine(SAM_TINY, sd, torch.device("cuda:0"))
    img = make_image(SAM_TINY, m["B"], m["image_seed"])
    _check(eng.encode(img), g["embedding"], "sam_tiny vs HF golden")
    img2 = make_image(SAM_TINY, 3, 77)           # fresh input, odd batch
    with torch.no_grad():
        ref = S.image_encoder(sd, SAM_TINY, img2)
    _check(eng.encode(img2), ref, "sam_tiny fresh vs oracle")


def test_vit_h_1024_vs_golden():
    """Full SAM ViT-H (637 M parameters, 1024x1024 -> 256x64x64): 28 windowed + 4 global blocks."""
    g = torch.load(os.path.join(GOLD, "sam_vit_h.pt"))
    m = g["meta"]
    sd = make_sam_state_dict(SAM_VIT_H, m["weight_seed"])
    eng = SamEncoderEngine(SAM_VIT_H, sd, torch.device("cuda:0"))
    del sd
    out = eng.encode(make_image(SAM_VIT_H, m["B"], m["image_seed"]))
    assert torch.isfinite(out).all()
    dim, idx = g["embedding_index"]             # the golden file keeps a fixed, seeded sample of the channels
    _check(out.cpu().index_select(dim, idx), g["embedding"], "sam_vit_h vs HF golden")


def test_encoder_rejects_wrong_shape():
    sd = make_sam_state_dict(SAM_TINY, 1)
    eng = SamEncoderEngine(SAM_TINY, sd, torch.device("cuda:0"))
    with pytest.raises(ValueError):
        eng.encode(torch.zeros(1, 3, 128, 128))
