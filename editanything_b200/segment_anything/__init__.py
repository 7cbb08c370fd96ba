"""Import-compatible stand-in for the `segment_anything` package the reference depends on (an un-vendored git
dependency: editany_lora.py:44-66; SURVEY.md §8b row B4):

    from segment_anything import sam_model_registry, SamAutomaticMaskGenerator, SamPredictor      # reference
    from editanything_b200.segment_anything import ...                                             # this backend

`sam_model_registry["default"](checkpoint=path)` builds a `Sam` whose image encoder is the H100 engine
(`editanything_b200.sam.SamEncoderEngine`, built when the model is moved to a CUDA device) and whose prompt encoder /
mask decoder are PyTorch modules with upstream parameter names, so the official .pth checkpoints load as they are."""
import torch

from ..sam_spec import SAM_VIT_H, SamEncoderConfig
from .amg import SamAutomaticMaskGenerator, remove_small_regions  # noqa: F401
from .modeling import MaskDecoder, PromptEncoder, Sam, TwoWayTransformer, _EncoderModule
from .predictor import ResizeLongestSide, SamPredictor  # noqa: F401

SAM_VIT_L = SamEncoderConfig(embed_dim=1024, depth=24, num_heads=16, mlp_dim=4096, global_attn_indexes=(5, 11, 17, 23))
SAM_VIT_B = SamEncoderConfig(embed_dim=768, depth=12, num_heads=12, mlp_dim=3072, global_attn_indexes=(2, 5, 8, 11))


def build_sam_from_state_dict(cfg: SamEncoderConfig, state_dict):
    """`state_dict`: upstream names (image_encoder.*, prompt_encoder.*, mask_decoder.*)."""
    pe_dim = cfg.out_chans
    enc_sd = {k: v for k, v in state_dict.items() if k.startswith("image_encoder.")}
    sam = Sam(_EncoderModule(cfg, enc_sd),
              PromptEncoder(embed_dim=pe_dim, image_embedding_size=(cfg.grid, cfg.grid),
                            input_image_size=(cfg.img_size, cfg.img_size), mask_in_chans=16),
              MaskDecoder(transformer_dim=pe_dim, transformer=TwoWayTransformer(2, pe_dim, 8, 2048)))
    rest = {k: v for k, v in state_dict.items() if not k.startswith("image_encoder.")}
    if rest:
        missing, unexpected = sam.load_state_dict(rest, strict=False)
        bad = [k for k in missing if not k.startswith("image_encoder.")] + list(unexpected)
        if bad:
            raise KeyError(f"SAM checkpoint does not match: {bad[:5]}")
    return sam.eval()


def config_from_state_dict(sd):
    """The encoder configuration a checkpoint was trained with, read off its tensor shapes (the registry keys only
    name the default sizes; a checkpoint of another size - e.g. the test-sized ones - still loads)."""
    pe = sd["image_encoder.pos_embed"]
    grid, dim = pe.shape[1], pe.shape[-1]
    patch = sd["image_encoder.patch_embed.proj.weight"].shape[-1]
    depth = 1 + max(int(k.split(".")[2]) for k in sd if k.startswith("image_encoder.blocks."))
    head_dim = sd["image_encoder.blocks.0.attn.rel_pos_h"].shape[1]
    lens = [sd[f"image_encoder.blocks.{i}.attn.rel_pos_h"].shape[0] for i in range(depth)]
    glob = tuple(i for i, n in enumerate(lens) if n == 2 * grid - 1)
    win = [(n + 1) // 2 for i, n in enumerate(lens) if i not in glob]
    return SamEncoderConfig(img_size=grid * patch, patch_size=patch, embed_dim=dim, depth=depth, num_heads=dim // head_dim,
                            mlp_dim=sd["image_encoder.blocks.0.mlp.lin1.weight"].shape[0],
                            out_chans=sd["image_encoder.neck.0.weight"].shape[0], window_size=win[0] if win else 0,
                            global_attn_indexes=glob)


def _builder(cfg):
    def build(checkpoint=None):
        if checkpoint is None:
            raise ValueError("a checkpoint path is required (synthetic weights: build_sam_from_state_dict)")
        sd = torch.load(checkpoint, map_location="cpu", weights_only=True)
        return build_sam_from_state_dict(config_from_state_dict(sd), sd)
    return build


build_sam_vit_h, build_sam_vit_l, build_sam_vit_b = _builder(SAM_VIT_H), _builder(SAM_VIT_L), _builder(SAM_VIT_B)
build_sam = build_sam_vit_h
sam_model_registry = {"default": build_sam_vit_h, "vit_h": build_sam_vit_h, "vit_l": build_sam_vit_l, "vit_b": build_sam_vit_b}
