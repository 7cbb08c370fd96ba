"""tests/golden/host_reference.pt: what the REFERENCE's own host functions return on the fixed inputs of
tests/test_host_semantics_cpu.py and tests/test_app_cpu.py, as bit-exact fingerprints (tests compare against it).

    python -m oracle.make_golden_host        (needs the reference tree; EA_REFERENCE_ROOT, default /root/reference)

annotator/util.py is imported as is; show_anns / make_inpaint_condition / get_pipeline_embeds and
EditAnythingLoraModel.process / get_sam_control live in editany_lora.py, whose module-level imports (diffusers,
gradio, segment_anything) are absent, so exactly those definitions are compiled out of the reference file (ast) and
executed unmodified in a namespace of stand-ins.  Nothing of the reference's source is stored."""
import ast
import os
import random
import sys

import numpy as np
import torch
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
REF = os.environ.get("EA_REFERENCE_ROOT", "/root/reference")
OUT = os.path.join(ROOT, "tests", "golden", "host_reference.pt")


def _ref_util():
    if REF not in sys.path:
        sys.path.insert(0, REF)
    import annotator.util as U
    return U


def _ref_namespace():
    from editanything_b200 import host
    import cv2
    import einops
    U = _ref_util()
    import PIL.Image  # noqa: F401
    return {"np": np, "torch": torch, "cv2": cv2, "einops": einops, "random": random, "Image": Image,
            "PIL": __import__("PIL"), "os": os, "HWC3": U.HWC3, "resize_image": U.resize_image,
            "get_bounding_box": U.get_bounding_box, "seed_everything": host.seed_everything,
            "StableDiffusionControlNetInpaintMixingPipeline": type("Mix", (), {}), "prepare_mask_image": None,
            "obtain_generation_model": None}


def _compile_reference():
    """The reference's helper functions and an EditAnythingLoraModel with ONLY `process` and `get_sam_control`."""
    ns = _ref_namespace()
    tree = ast.parse(open(os.path.join(REF, "editany_lora.py")).read())
    for node in tree.body:
        if isinstance(node, ast.FunctionDef) and node.name in ("show_anns", "make_inpaint_condition", "get_pipeline_embeds"):
            exec(compile(ast.Module([node], []), "editany_lora.py", "exec"), ns)
        if isinstance(node, ast.ClassDef) and node.name == "EditAnythingLoraModel":
            keep = [n for n in node.body if isinstance(n, ast.FunctionDef) and n.name in ("process", "get_sam_control")]
            for n in keep:
                n.decorator_list = []          # @torch.inference_mode() / @save_input_to_file: not part of the arithmetic
            node.body = keep
            exec(compile(ast.Module([node], []), "editany_lora.py", "exec"), ns)
    return ns


def main():
    from tests import test_app_cpu as A
    from tests import test_host_semantics_cpu as H
    if not os.path.isfile(os.path.join(REF, "editany_lora.py")):
        sys.exit(f"reference tree not found at {REF}")
    ns = _compile_reference()
    fp = H.fingerprint
    out = {"show_anns": fp(H.show_anns_cases(ns["show_anns"])),
           "make_inpaint_condition": fp(H.inpaint_condition_case(ns["make_inpaint_condition"])),
           "image_helpers": fp(H.image_helper_cases(_ref_util())),
           "get_pipeline_embeds": fp(H.pipeline_embeds_cases(ns["get_pipeline_embeds"]))}
    cuda, save = torch.Tensor.cuda, os.environ.get("EA_SAVE_INPUT")
    torch.Tensor.cuda = lambda self, *a, **k: self          # the reference hard-codes .cuda()
    os.environ["EA_SAVE_INPUT"] = "0"
    try:
        calls, tile_calls, (r_tile, r_res, r_masks, r_prompt) = A.run_process(ns["EditAnythingLoraModel"])
    finally:
        torch.Tensor.cuda = cuda
        if save is None:
            os.environ.pop("EA_SAVE_INPUT", None)
    out["process"] = {"calls": [fp(c) for c in calls], "tile_calls": [fp(c) for c in tile_calls],
                      "results_tile": fp(r_tile), "results": fp(r_res), "masks": fp(r_masks), "prompt": r_prompt}
    torch.save(out, OUT)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
