"""tests/golden/lora_reference.pt: the weights the REFERENCE's own `load_lora_weights` (editany_lora.py:197-329)
produces on the synthetic LoRA cases of tests/synth_lora.py, as per-tensor SHA-256 fingerprints.

    python -m oracle.make_golden_lora        (needs the reference tree; EA_REFERENCE_ROOT, default /root/reference)

editany_lora.py's module-level imports (diffusers, gradio, segment_anything) are absent here, so exactly that one
function is compiled out of the reference file (ast) and run unmodified, the way its call sites call it
(`load_lora_weights(pipe, [path, ...], multiplier, "cpu", torch.float32)`, :378-381), on a stand-in pipeline:
`.unet` is an nn.Module tree of the synthetic diffusers-keyed UNet weights in fp16 and `.text_encoder` the tiny fp16
CLIPTextModel of tests/synth_ckpt.py, both what `from_pretrained(torch_dtype=torch.float16)` would hold.  The LoRA
factors are dyadic rationals, so the fingerprints do not depend on the CPU's BLAS.  Nothing of the reference's
source is stored."""
import ast
import os
import sys
import tempfile
from collections import defaultdict
from types import SimpleNamespace

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
REF = os.environ.get("EA_REFERENCE_ROOT", "/root/reference")
OUT = os.path.join(ROOT, "tests", "golden", "lora_reference.pt")


def _compile_reference():
    from safetensors.torch import load_file
    ns = {"torch": torch, "defaultdict": defaultdict, "load_file": load_file, "print": lambda *a, **k: None}
    tree = ast.parse(open(os.path.join(REF, "editany_lora.py")).read())
    for node in tree.body:
        if isinstance(node, ast.FunctionDef) and node.name == "load_lora_weights":
            exec(compile(ast.Module([node], []), "editany_lora.py", "exec"), ns)
    return ns["load_lora_weights"]


def run_case(load_lora_weights, name, tmp):
    """{"unet": {diffusers key: fingerprint}, "text_encoder": {key: fingerprint}} of every tensor the case changes."""
    from tests import synth_ckpt
    from tests import synth_lora as SL
    cfg = SL.CASES[name][0]
    root = os.path.join(tmp, f"te{cfg.context_dim}")
    if not os.path.isdir(root):
        synth_ckpt.write_text_encoder_and_tokenizer(root, cfg.context_dim)
    te = SL.text_encoder_fp16(root)
    te_before = {k: v.clone() for k, v in te.state_dict().items()}
    usd = {k: v.to(torch.float16) for k, v in SL.unet_diffusers_state_dict(cfg).items()}
    pipe = SimpleNamespace(unet=SL.module_tree(usd), text_encoder=te)
    paths, mult, _ = SL.write_case(name, tmp, {k: v.shape for k, v in te_before.items()})
    load_lora_weights(pipe, paths, mult, "cpu", torch.float32)
    out = {"unet": {}, "text_encoder": {}}
    for k, v in pipe.unet.state_dict().items():
        if not torch.equal(v, usd[k]):
            out["unet"][k] = SL.fingerprint(v)
    for k, v in te.state_dict().items():
        if not torch.equal(v, te_before[k]):
            out["text_encoder"][k] = SL.fingerprint(v)
    return out


def main():
    from tests import synth_lora as SL
    if not os.path.isfile(os.path.join(REF, "editany_lora.py")):
        sys.exit(f"reference tree not found at {REF}")
    fn = _compile_reference()
    with tempfile.TemporaryDirectory() as tmp:
        out = {name: run_case(fn, name, tmp) for name in SL.CASES}
    torch.save(out, OUT)
    print(OUT, os.path.getsize(OUT), "bytes", {k: (len(v["unet"]), len(v["text_encoder"])) for k, v in out.items()})


if __name__ == "__main__":
    main()
