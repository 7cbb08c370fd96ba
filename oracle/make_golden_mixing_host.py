"""tests/golden/host_mixing.pt: what the REFERENCE's own EditAnythingLoraModel.process hands an alpha-mixing generation
pipeline and tile pipeline (editany_lora.py:829-856, :902-918) on the fixed inputs of tests/test_app_cpu.py with
alpha_weight 0.3, with and without use_scale_map, as bit-exact fingerprints.

    python -m oracle.make_golden_mixing_host   (needs the reference tree; EA_REFERENCE_ROOT, default /root/reference)

`process` is compiled out of editany_lora.py as oracle/make_golden_host.py does, with the name
StableDiffusionControlNetInpaintMixingPipeline bound to the spy class of tests/test_mixing_cpu.py (so the reference
takes its mixing branch) and prepare_mask_image compiled unmodified out of the reference's
utils/stable_diffusion_controlnet_inpaint.py.  Nothing of the reference's source is stored."""
import ast
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from oracle.make_golden_host import REF, _compile_reference  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "host_mixing.pt")


def _ref_prepare_mask_image():
    import numpy as np
    import PIL.Image
    ns = {"np": np, "torch": torch, "PIL": PIL}
    tree = ast.parse(open(os.path.join(REF, "utils", "stable_diffusion_controlnet_inpaint.py")).read())
    node = next(n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == "prepare_mask_image")
    exec(compile(ast.Module([node], []), "stable_diffusion_controlnet_inpaint.py", "exec"), ns)
    return ns["prepare_mask_image"]


def main():
    from tests import test_mixing_cpu as T
    from tests.test_host_semantics_cpu import fingerprint as fp
    if not os.path.isfile(os.path.join(REF, "editany_lora.py")):
        sys.exit(f"reference tree not found at {REF}")
    ns = _compile_reference()
    cls = ns["EditAnythingLoraModel"]
    # process() reads both names from its module's globals
    cls.process.__globals__["StableDiffusionControlNetInpaintMixingPipeline"] = T.SpyMixingPipe
    cls.process.__globals__["prepare_mask_image"] = _ref_prepare_mask_image()
    cuda, save = torch.Tensor.cuda, os.environ.get("EA_SAVE_INPUT")
    torch.Tensor.cuda = lambda self, *a, **k: self          # the reference hard-codes .cuda()
    os.environ["EA_SAVE_INPUT"] = "0"
    out = {}
    try:
        for use_scale_map in (False, True):
            calls, tile_calls, (r_tile, r_res, r_masks, r_prompt) = T.run_mixing_process(cls, use_scale_map)
            out[f"scale_map={use_scale_map}"] = {
                "calls": [fp(c) for c in calls], "tile_calls": [fp(c) for c in tile_calls],
                "results_tile": fp(r_tile), "results": fp(r_res), "masks": fp(r_masks), "prompt": r_prompt}
    finally:
        torch.Tensor.cuda = cuda
        if save is None:
            os.environ.pop("EA_SAVE_INPUT", None)
    torch.save(out, OUT)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
