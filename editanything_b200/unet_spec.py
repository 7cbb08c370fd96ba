"""Topology of the SD UNet / ControlNet as a flat block table + synthetic weights.

Restated from the reference constructors (no code shared with them):
  UNetModel.__init__            ldm/modules/diffusionmodules/openaimodel.py:442-736
  ControlNet.__init__           cldm/cldm.py:48-282 (same encoder + hint stack + zero convs)
  SD2.1 values                  models/cldm_v21.yaml:21-55
  SD1.5 values                  not shipped (tools/tool_add_control_sd15.py:27); the usual
                                model_channels 320, mult (1,2,4,4), 8 heads, context 768
Parameter names follow the ldm/cldm state-dict convention so real checkpoints (after the
diffusers->ldm key map of SURVEY.md App. B) load unchanged.
"""
from dataclasses import dataclass, field, replace
from typing import List, Optional, Tuple

import torch


@dataclass(frozen=True)
class UNetConfig:
    in_channels: int = 4
    out_channels: int = 4
    model_channels: int = 320
    num_res_blocks: int = 2
    attention_resolutions: Tuple[int, ...] = (4, 2, 1)
    channel_mult: Tuple[int, ...] = (1, 2, 4, 4)
    num_heads: int = 8                 # used when num_head_channels == -1 (SD1.5)
    num_head_channels: int = -1        # 64 for SD2.1
    context_dim: int = 768
    use_linear_in_transformer: bool = False
    hint_channels: int = 3

    def heads_for(self, ch):
        if self.num_head_channels == -1:
            return self.num_heads, ch // self.num_heads
        return ch // self.num_head_channels, self.num_head_channels


SD15 = UNetConfig()
SD21 = UNetConfig(num_head_channels=64, context_dim=1024, use_linear_in_transformer=True)
# reduced-width configuration used by the fast parity tests (same topology, every tensor-core
# shape constraint still met: channels multiples of 64)
TINY = UNetConfig(model_channels=64, num_heads=8, context_dim=64)
TINY21 = UNetConfig(model_channels=64, num_head_channels=16, context_dim=128, use_linear_in_transformer=True)
# inpainting base models (stabilityai/stable-diffusion-2-inpainting): the UNet also reads the mask and the VAE latents
# of the masked image, 4 + 1 + 4 = 9 input channels (utils/stable_diffusion_controlnet_inpaint.py:955-979)
SD2_INPAINT = replace(SD21, in_channels=9)
TINY21_INPAINT = replace(TINY21, in_channels=9)


def controlnet_config(cfg: UNetConfig) -> UNetConfig:
    """The ControlNet belonging to a UNet: the same topology on the 4 latent channels only (models/cldm_v21.yaml:44;
    the 9-channel branch feeds the ControlNets the plain latents, utils/...inpaint.py:1607-1615)."""
    return replace(cfg, in_channels=4)

HINT_CHANNELS = (16, 16, 32, 32, 96, 96, 256)      # cldm/cldm.py:147-163
HINT_STRIDES = (1, 1, 2, 1, 2, 1, 2, 1)


@dataclass
class Block:
    """One TimestepEmbedSequential entry: ('res'|'attn'|'down'|'up'|'conv_in', prefix, cin, cout)."""
    kind: str
    prefix: str
    cin: int
    cout: int


@dataclass
class Topology:
    cfg: UNetConfig
    input_blocks: List[List[Block]] = field(default_factory=list)
    middle: List[Block] = field(default_factory=list)
    output_blocks: List[List[Block]] = field(default_factory=list)
    input_chans: List[int] = field(default_factory=list)     # channels of each saved skip


def build_topology(cfg: UNetConfig, with_decoder: bool = True) -> Topology:
    t = Topology(cfg)
    mc = cfg.model_channels
    t.input_blocks.append([Block("conv_in", "input_blocks.0.0", cfg.in_channels, mc)])
    chans = [mc]
    ch, ds, idx = mc, 1, 1
    for level, mult in enumerate(cfg.channel_mult):
        for _ in range(cfg.num_res_blocks):
            layers = [Block("res", f"input_blocks.{idx}.0", ch, mult * mc)]
            ch = mult * mc
            if ds in cfg.attention_resolutions:
                layers.append(Block("attn", f"input_blocks.{idx}.1", ch, ch))
            t.input_blocks.append(layers)
            chans.append(ch)
            idx += 1
        if level != len(cfg.channel_mult) - 1:
            t.input_blocks.append([Block("down", f"input_blocks.{idx}.0", ch, ch)])
            chans.append(ch)
            idx += 1
            ds *= 2
    t.input_chans = list(chans)
    t.middle = [Block("res", "middle_block.0", ch, ch), Block("attn", "middle_block.1", ch, ch),
                Block("res", "middle_block.2", ch, ch)]
    if with_decoder:
        oidx = 0
        for level, mult in list(enumerate(cfg.channel_mult))[::-1]:
            for i in range(cfg.num_res_blocks + 1):
                ich = chans.pop()
                layers = [Block("res", f"output_blocks.{oidx}.0", ch + ich, mc * mult)]
                ch = mc * mult
                if ds in cfg.attention_resolutions:
                    layers.append(Block("attn", f"output_blocks.{oidx}.{len(layers)}", ch, ch))
                if level and i == cfg.num_res_blocks:
                    layers.append(Block("up", f"output_blocks.{oidx}.{len(layers)}", ch, ch))
                    ds //= 2
                t.output_blocks.append(layers)
                oidx += 1
    return t


def param_shapes(cfg: UNetConfig, kind: str):
    """Ordered {name: (shape, role)} for kind in {'unet', 'controlnet'}.  role drives the synthetic
    init: 'w' weight (fan-in scaled), 'b' bias, 'g' norm gain, 'nb' norm bias."""
    topo = build_topology(cfg, with_decoder=(kind == "unet"))
    mc, ted = cfg.model_channels, cfg.model_channels * 4
    P = {}

    def conv(p, cin, cout, k):
        P[p + ".weight"] = ((cout, cin, k, k), "w")
        P[p + ".bias"] = ((cout,), "b")

    def lin(p, cin, cout, bias=True):
        P[p + ".weight"] = ((cout, cin), "w")
        if bias:
            P[p + ".bias"] = ((cout,), "b")

    def norm(p, c):
        P[p + ".weight"] = ((c,), "g")
        P[p + ".bias"] = ((c,), "nb")

    def res(p, cin, cout):
        norm(p + ".in_layers.0", cin)
        conv(p + ".in_layers.2", cin, cout, 3)
        lin(p + ".emb_layers.1", ted, cout)
        norm(p + ".out_layers.0", cout)
        conv(p + ".out_layers.3", cout, cout, 3)
        if cin != cout:
            conv(p + ".skip_connection", cin, cout, 1)

    def attn(p, c):
        heads, dh = cfg.heads_for(c)
        inner = heads * dh
        norm(p + ".norm", c)
        if cfg.use_linear_in_transformer:
            lin(p + ".proj_in", c, inner)
        else:
            conv(p + ".proj_in", c, inner, 1)
        tb = p + ".transformer_blocks.0"
        for a, cd in (("attn1", inner), ("attn2", cfg.context_dim)):
            lin(f"{tb}.{a}.to_q", inner, inner, bias=False)
            lin(f"{tb}.{a}.to_k", cd, inner, bias=False)
            lin(f"{tb}.{a}.to_v", cd, inner, bias=False)
            lin(f"{tb}.{a}.to_out.0", inner, inner)
        lin(tb + ".ff.net.0.proj", inner, inner * 8)
        lin(tb + ".ff.net.2", inner * 4, inner)
        for n in ("norm1", "norm2", "norm3"):
            norm(f"{tb}.{n}", inner)
        if cfg.use_linear_in_transformer:
            lin(p + ".proj_out", inner, c)
        else:
            conv(p + ".proj_out", inner, c, 1)

    lin("time_embed.0", mc, ted)
    lin("time_embed.2", ted, ted)

    def emit(blocks):
        for b in blocks:
            if b.kind == "conv_in":
                conv(b.prefix, b.cin, b.cout, 3)
            elif b.kind == "res":
                res(b.prefix, b.cin, b.cout)
            elif b.kind == "attn":
                attn(b.prefix, b.cin)
            elif b.kind == "down":
                conv(b.prefix + ".op", b.cin, b.cout, 3)
            elif b.kind == "up":
                conv(b.prefix + ".conv", b.cin, b.cout, 3)

    for layers in topo.input_blocks:
        emit(layers)
    emit(topo.middle)
    if kind == "unet":
        for layers in topo.output_blocks:
            emit(layers)
        norm("out.0", mc)
        conv("out.2", mc, cfg.out_channels, 3)
    else:
        cin = cfg.hint_channels
        for i, cout in enumerate(HINT_CHANNELS + (mc,)):
            conv(f"input_hint_block.{2 * i}", cin, cout, 3)
            cin = cout
        for i, c in enumerate(topo.input_chans):
            conv(f"zero_convs.{i}.0", c, c, 1)
        conv("middle_block_out.0", topo.middle[-1].cout, topo.middle[-1].cout, 1)
    return P


def make_state_dict(cfg: UNetConfig, kind: str, seed: int, dtype=torch.float32, device="cpu"):
    """Deterministic synthetic weights (CPU generator).  Weights ~ N(0, 1/fan_in) so activations
    keep O(1) scale through the network; the reference's zero-initialised tensors
    (zero_module: openaimodel.py:228-231,729; attention.py:312-318; cldm/cldm.py:162,282) are drawn
    like every other weight — with them at zero every golden vector would be identically 0."""
    g = torch.Generator(device=device).manual_seed(seed)
    sd = {}
    for name, (shape, role) in param_shapes(cfg, kind).items():
        if role == "w":
            fan_in = 1
            for s in shape[1:]:
                fan_in *= s
            t = torch.randn(shape, generator=g, device=device) * (fan_in ** -0.5)
        elif role == "b":
            t = torch.randn(shape, generator=g, device=device) * 0.05
        elif role == "g":
            t = 1.0 + 0.1 * torch.randn(shape, generator=g, device=device)
        else:
            t = 0.1 * torch.randn(shape, generator=g, device=device)
        sd[name] = t.to(dtype)
    return sd
