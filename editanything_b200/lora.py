"""Kohya-format LoRA files merged into the base weights before packing (editany_lora.py:197-329).

The reference's `load_lora_weights(pipe, [path], lora_weight, "cpu", torch.float32)` walks `pipe.unet` and
`pipe.text_encoder` and adds `multiplier * scale * up @ down` to each target weight in place.  The engines here
pre-pack their weights (fused q/k/v, LayerNorm gammas folded into the GEMMs, cross-attention K/V projected per
request), which cannot be undone, so the merge runs on the host state dict before packing.  The result is the
reference's, bit for bit:

* a file is grouped by `layer, elem = key.split(".", 1)`; a layer whose name contains "text" targets the text
  encoder, every other one the UNet;
* the layer name resolves with the reference's greedy walk: pop one `_`-separated token and look it up as a child,
  parameter or buffer (what `nn.Module.__getattr__` sees); on failure join the next token with `_` and retry.  The
  UNet is walked as the prefix tree of its diffusers parameter names, which is the module tree of
  `UNet2DConditionModel`; a name that never resolves raises `IndexError` like the reference's `pop(0)`;
* `up` and `down` are cast to fp32, scale = alpha / rank when `alpha` is truthy, else 1 (so alpha = 0 means 1, and
  a file without `alpha` raises `KeyError`), and the delta is added in fp32 to the fp16 weight that
  `from_pretrained(torch_dtype=torch.float16)` holds, rounding once;
* 3x3 ("LoCon") entries fail, as they do inside the reference's `torch.mm`, with `RuntimeError`.

One deliberate difference: every entry of every file is resolved and checked before any weight changes, so a bad
file leaves the weights untouched (the reference leaves them half merged).  Several files apply in list order, each
rounding to fp16.
"""
import os
from collections import defaultdict

import torch

LORA_PREFIX_UNET = "lora_unet"
LORA_PREFIX_TEXT_ENCODER = "lora_te"


def read_lora(path):
    """{layer: {elem: tensor}} of one kohya `.safetensors` file, grouped like editany_lora.py:205-211."""
    from safetensors.torch import load_file
    updates = defaultdict(dict)
    for key, value in load_file(path, device="cpu").items():
        layer, elem = key.split(".", 1)
        updates[layer][elem] = value
    return updates


def normalize(lora):
    """[(path, multiplier), ...] with real paths and float multipliers; None or () for no LoRA."""
    return [(os.path.realpath(p), float(m)) for p, m in (lora or ())]


class KeyTree:
    """The module tree a list of parameter names implies: its nodes are the dotted prefixes of the names.  `child`
    looks a name up the way `nn.Module.__getattr__` does (child modules, parameters and buffers), so the LoRA layer
    names resolve on a diffusers-keyed state dict without building the model."""

    def __init__(self, names):
        self.children = defaultdict(set)
        for n in names:
            parts = n.split(".")
            for i in range(len(parts)):
                self.children[".".join(parts[:i])].add(parts[i])

    def child(self, node, name):
        if name not in self.children.get(node, ()):
            raise AttributeError(name)
        return f"{node}.{name}" if node else name


def walk(tokens, root, child):
    """The reference's greedy name walk (editany_lora.py:226-238), restated: the node the tokens lead to."""
    tokens = list(tokens)
    cur = root
    temp_name = tokens.pop(0)
    while True:
        try:
            cur = child(cur, temp_name)
            if tokens:
                temp_name = tokens.pop(0)
            else:
                return cur
        except Exception:
            if len(temp_name) > 0:
                temp_name += "_" + tokens.pop(0)        # IndexError once the tokens run out
            else:
                temp_name = tokens.pop(0)


def _module_child(module, name):
    return module.__getattr__(name)


def layer_tokens(layer):
    """(target, tokens): "text_encoder" or "unet", and the `_`-split name below the prefix."""
    if "text" in layer:
        return "text_encoder", layer.split(LORA_PREFIX_TEXT_ENCODER + "_")[-1].split("_")
    return "unet", layer.split(LORA_PREFIX_UNET + "_")[-1].split("_")


def _factors(elems):
    """(up, down, scale) of one layer: fp32 factors as 2-D matrices and the scalar alpha / rank (or 1)."""
    up = elems["lora_up.weight"].to(torch.float32)
    down = elems["lora_down.weight"].to(torch.float32)
    alpha = elems["alpha"]
    if alpha:
        alpha = alpha.item() / up.shape[1]
    else:
        alpha = 1.0
    return up, down, alpha


def _check_shapes(layer, up, down, weight_shape):
    """The shape errors the reference's torch.mm and in-place add raise, found before anything is merged."""
    if up.dim() == 4:
        if up.shape[2:] != (1, 1) or down.dim() != 4 or down.shape[2:] != (1, 1):
            raise RuntimeError(f"LoRA layer {layer}: only 1x1 convolutions are supported, got up {tuple(up.shape)} "
                               f"and down {tuple(down.shape)}")
        out_shape = (up.shape[0], down.shape[1], 1, 1)
    else:
        if up.dim() != 2 or down.dim() != 2:
            raise RuntimeError(f"LoRA layer {layer}: up {tuple(up.shape)} and down {tuple(down.shape)} are not matrices")
        out_shape = (up.shape[0], down.shape[1])
    if up.shape[1] != down.shape[0]:
        raise RuntimeError(f"LoRA layer {layer}: up {tuple(up.shape)} and down {tuple(down.shape)} cannot be multiplied")
    if tuple(weight_shape) != out_shape:
        raise RuntimeError(f"LoRA layer {layer}: a delta of shape {out_shape} does not fit the weight "
                           f"{tuple(weight_shape)}")


def delta(up, down, scale, multiplier):
    """multiplier * scale * up @ down in fp32 (editany_lora.py:314-328), back in 4-D for a 1x1 convolution."""
    if len(up.shape) == 4:
        return (multiplier * scale * torch.mm(up.squeeze(3).squeeze(2), down.squeeze(3).squeeze(2))
                ).unsqueeze(2).unsqueeze(3)
    return multiplier * scale * torch.mm(up, down)


def plan(lora, unet_keys=None, unet_shapes=None, text_encoder=None):
    """Read, resolve and check every entry of every file in `lora` ([(path, multiplier), ...]) without changing a
    weight.  unet_keys / unet_shapes: the diffusers parameter names and their shapes (a dict name -> shape);
    text_encoder: the CLIPTextModel.  Entries for a target that is None are skipped (a network shared with another
    pipeline that already carries the same merge).  Returns [(target, name or module, up, down, scale, multiplier)] in
    application order; `target` is "unet" (name: the diffusers weight key) or "text_encoder"."""
    if unet_keys is None and text_encoder is None:
        return []
    tree = KeyTree(unet_keys) if unet_keys is not None else None
    entries = []
    for path, multiplier in lora:
        for layer, elems in read_lora(path).items():
            target, tokens = layer_tokens(layer)
            if target == "unet":
                if tree is None:
                    continue
                node = walk(tokens, "", tree.child)
                name = node + ".weight"
                if name not in unet_shapes:
                    raise AttributeError(f"LoRA layer {layer}: '{node}' has no weight")
                shape = unet_shapes[name]
            else:
                if text_encoder is None:
                    continue
                name = walk(tokens, text_encoder, _module_child)
                shape = name.weight.shape
            up, down, scale = _factors(elems)
            _check_shapes(layer, up, down, shape)
            entries.append((target, name, up, down, scale, multiplier))
    return entries


def apply(entries, unet_sd=None):
    """Merge planned entries in order.  UNet weights in `unet_sd` (diffusers keys) become fp16 with the delta added
    in fp32 and rounded once; text-encoder weights (fp16 modules) take the CPU-computed delta on their device with
    the same single rounding.  Untouched tensors are left as they are."""
    for target, name, up, down, scale, multiplier in entries:
        d = delta(up, down, scale, multiplier)
        if target == "unet":
            w = unet_sd[name]
            if w.dtype != torch.float16:
                w = w.to(torch.float16)
            else:
                w = w.clone()                 # the loaded dict may share storage with the file's tensors
            w += d
            unet_sd[name] = w
        else:
            w = name.weight.data
            w += d.to(w.device)


def merge(lora, unet_sd=None, text_encoder=None):
    """Merge [(path, multiplier), ...] into a diffusers-keyed UNet state dict (replaced entries, in place) and/or a
    text encoder (in place).  Nothing changes if any entry fails to resolve or check."""
    if not lora:
        return
    shapes = None if unet_sd is None else {k: v.shape for k, v in unet_sd.items()}
    entries = plan(lora, None if unet_sd is None else list(unet_sd), shapes, text_encoder)
    with torch.no_grad():
        apply(entries, unet_sd)
