"""The `segment_anything` stand-in (editanything_b200/segment_anything): prompt encoder + two-way mask decoder against
the in-container HF port of the same network (transformers.models.sam) with the same weights; the automatic mask
generator's pure helpers; the predictor / generator plumbing with a stub image encoder (the real one is the H100
engine: tests/test_gpu_sam.py).  Upstream `segment_anything` is absent: parity unpinned against it."""
import numpy as np
import pytest
import torch

from editanything_b200.segment_anything import (MaskDecoder, PromptEncoder, Sam, SamAutomaticMaskGenerator, SamPredictor,
                                                TwoWayTransformer)
from editanything_b200.segment_anything import amg as A


def _to_hf(sd):
    out = {}
    for k, v in sd.items():
        if k == "prompt_encoder.pe_layer.positional_encoding_gaussian_matrix":
            out["shared_image_embedding.positional_embedding"] = v
            out["prompt_encoder.shared_embedding.positional_embedding"] = v
            continue
        k = k.replace("prompt_encoder.point_embeddings.", "prompt_encoder.point_embed.")
        for a, b in (("mask_downscaling.0.", "mask_embed.conv1."), ("mask_downscaling.1.", "mask_embed.layer_norm1."),
                     ("mask_downscaling.3.", "mask_embed.conv2."), ("mask_downscaling.4.", "mask_embed.layer_norm2."),
                     ("mask_downscaling.6.", "mask_embed.conv3."), ("output_upscaling.0.", "upscale_conv1."),
                     ("output_upscaling.1.", "upscale_layer_norm."), ("output_upscaling.3.", "upscale_conv2."),
                     (".norm_final_attn.", ".layer_norm_final_attn.")):
            k = k.replace(a, b)
        for i in (1, 2, 3, 4):
            k = k.replace(f".norm{i}.", f".layer_norm{i}.")
        if "hypernetworks_mlps" in k or "iou_prediction_head" in k:
            k = k.replace(".layers.0.", ".proj_in.").replace(".layers.2.", ".proj_out.").replace(".layers.1.", ".layers.0.")
        out[k] = v
    return out


def _models(dim=64, grid=16, size=256):
    torch.manual_seed(0)
    pe = PromptEncoder(embed_dim=dim, image_embedding_size=(grid, grid), input_image_size=(size, size), mask_in_chans=16)
    md = MaskDecoder(transformer_dim=dim, transformer=TwoWayTransformer(2, dim, 8, 128), iou_head_hidden_dim=dim)
    for p in list(pe.parameters()) + list(md.parameters()):
        torch.nn.init.normal_(p, std=0.3)
    return pe, md


def test_prompt_encoder_and_mask_decoder_match_the_hf_port():
    from transformers import SamConfig, SamMaskDecoderConfig, SamModel, SamPromptEncoderConfig, SamVisionConfig
    dim, grid, size = 64, 16, 256
    pe, md = _models(dim, grid, size)
    vc = SamVisionConfig(hidden_size=32, num_hidden_layers=1, num_attention_heads=2, mlp_dim=64, image_size=size,
                         patch_size=16, output_channels=dim, window_size=4, global_attn_indexes=[0], num_pos_feats=dim // 2)
    cfg = SamConfig(vision_config=vc, prompt_encoder_config=SamPromptEncoderConfig(hidden_size=dim, image_size=size, patch_size=16),
                    mask_decoder_config=SamMaskDecoderConfig(hidden_size=dim, mlp_dim=128, num_attention_heads=8, iou_head_hidden_dim=dim))
    hf = SamModel(cfg).eval()
    sd = {"prompt_encoder." + k: v for k, v in pe.state_dict().items()}
    sd.update({"mask_decoder." + k: v for k, v in md.state_dict().items()})
    missing, unexpected = hf.load_state_dict(_to_hf(sd), strict=False)
    assert not unexpected and all(k.startswith("vision_encoder.") for k in missing), (missing[:3], unexpected[:3])
    g = torch.Generator().manual_seed(1)
    emb = torch.randn(1, dim, grid, grid, generator=g)
    pts = torch.rand(5, 1, 2, generator=g) * size                   # 5 single-point prompts (the AMG pattern)
    labels = torch.ones(5, 1, dtype=torch.int)
    with torch.no_grad():
        sparse, dense = pe(points=(pts, labels), boxes=None, masks=None)
        for multi in (True, False):
            masks, iou = md(image_embeddings=emb, image_pe=pe.get_dense_pe(), sparse_prompt_embeddings=sparse,
                            dense_prompt_embeddings=dense, multimask_output=multi)
            o = hf(image_embeddings=emb, input_points=pts.reshape(1, 5, 1, 2), input_labels=labels.reshape(1, 5, 1),
                   multimask_output=multi)
            assert masks.shape == o.pred_masks[0].shape
            assert torch.allclose(masks, o.pred_masks[0], atol=2e-4, rtol=1e-4), (masks - o.pred_masks[0]).abs().max()
            assert torch.allclose(iou, o.iou_scores[0], atol=2e-4, rtol=1e-4)
        # two points (positive + negative) and a box prompt
        pts2 = torch.rand(2, 2, 2, generator=g) * size
        lab2 = torch.tensor([[1, 0], [1, 1]], dtype=torch.int)
        sparse, dense = pe(points=(pts2, lab2), boxes=None, masks=None)
        masks, iou = md(emb, pe.get_dense_pe(), sparse, dense, True)
        o = hf(image_embeddings=emb, input_points=pts2.reshape(1, 2, 2, 2), input_labels=lab2.reshape(1, 2, 2), multimask_output=True)
        assert torch.allclose(masks, o.pred_masks[0], atol=2e-4, rtol=1e-4)
        box = torch.tensor([[20.0, 30.0, 200.0, 180.0]])
        sparse, dense = pe(points=None, boxes=box, masks=None)
        masks, iou = md(emb, pe.get_dense_pe(), sparse, dense, False)
        o = hf(image_embeddings=emb, input_boxes=box.reshape(1, 1, 4), multimask_output=False)
        assert torch.allclose(masks, o.pred_masks[0], atol=2e-4, rtol=1e-4)


class _StubEncoder(torch.nn.Module):
    """Deterministic stand-in with the image encoder's contract ([B,3,S,S] -> [B,C,S/16,S/16])."""
    img_size = 256

    def __init__(self, dim=64):
        super().__init__()
        torch.manual_seed(3)
        self.proj = torch.nn.Conv2d(3, dim, 16, 16)

    def forward(self, x):
        return torch.tanh(self.proj(x) * 0.05)


def _sam():
    pe, md = _models(64, 16, 256)
    return Sam(_StubEncoder(64), pe, md).eval()


def test_predictor_contract():
    sam = _sam()
    pred = SamPredictor(sam)
    img = np.random.RandomState(0).randint(0, 256, (120, 200, 3)).astype(np.uint8)
    with pytest.raises(RuntimeError):
        pred.predict(point_coords=np.array([[10, 10]]), point_labels=np.array([1]))
    pred.set_image(img)
    assert pred.input_size == (154, 256) and pred.original_size == (120, 200)      # longest side -> 256
    masks, scores, low = pred.predict(point_coords=np.array([[50, 60], [150, 20]]), point_labels=np.array([1, 0]),
                                      multimask_output=False)
    assert masks.shape == (1, 120, 200) and masks.dtype == bool and scores.shape == (1,) and low.shape == (1, 64, 64)
    masks3, scores3, _ = pred.predict(point_coords=np.array([[50, 60]]), point_labels=np.array([1]), multimask_output=True)
    assert masks3.shape == (3, 120, 200) and scores3.shape == (3,)
    # the transform maps original pixel coordinates into the resized frame
    assert np.allclose(pred.transform.apply_coords(np.array([[200.0, 120.0]]), (120, 200)), [[256.0, 154.0]])


def test_automatic_mask_generator_records_and_helpers():
    sam = _sam()
    gen = SamAutomaticMaskGenerator(sam, points_per_side=6, points_per_batch=16, pred_iou_thresh=-1e9,
                                    stability_score_thresh=-1.0, box_nms_thresh=0.7)
    img = np.random.RandomState(1).randint(0, 256, (96, 128, 3)).astype(np.uint8)
    anns = gen.generate(img)
    assert isinstance(anns, list) and len(anns) >= 1
    for a in anns:
        assert set(a) >= {"segmentation", "area", "bbox", "predicted_iou", "point_coords", "stability_score", "crop_box"}
        assert a["segmentation"].shape == (96, 128) and a["segmentation"].dtype == bool
        assert a["area"] == int(a["segmentation"].sum()) and a["crop_box"] == [0, 0, 128, 96]
    # the id map of the reference's show_anns accepts them as they are
    from editanything_b200.host import show_anns
    full, res = show_anns(anns)
    assert res.shape == (96, 128, 3) and res[:, :, 0].max() <= len(anns)
    # helpers
    g = A.build_point_grid(4)
    assert g.shape == (16, 2) and np.allclose(g[0], [0.125, 0.125]) and np.allclose(g[-1], [0.875, 0.875])
    boxes, layers = A.generate_crop_boxes((100, 200), 1, 512 / 1500)
    assert boxes[0] == [0, 0, 200, 100] and len(boxes) == 5 and layers == [0, 1, 1, 1, 1]
    m = torch.zeros(2, 10, 12, dtype=torch.bool)
    m[0, 2:5, 3:9] = True
    assert A.batched_mask_to_box(m).tolist() == [[3, 2, 8, 4], [0, 0, 0, 0]]
    logits = torch.full((1, 8, 8), -5.0)
    logits[0, 2:6, 2:6] = 5.0
    logits[0, 1, 1] = 0.5                                  # inside the -1 threshold, outside the +1 threshold
    assert abs(A.calculate_stability_score(logits, 0.0, 1.0).item() - 16 / 17) < 1e-6
    near = A.is_box_near_crop_edge(torch.tensor([[0, 0, 50, 50], [10, 10, 99, 60]]), [0, 0, 100, 100], [0, 0, 300, 300])
    assert near.tolist() == [False, True]                # touching the crop's right edge, which is not the image's
    hole = np.ones((20, 20), dtype=bool)
    hole[5:7, 5:7] = False
    filled, changed = A.remove_small_regions(hole, 10, "holes")
    assert changed and filled.all()


def test_registry_and_checkpoint_round_trip(tmp_path):
    from editanything_b200 import segment_anything as S
    from editanything_b200.sam_spec import SAM_TINY, make_sam_state_dict
    pe, _ = _models(SAM_TINY.out_chans, SAM_TINY.grid, SAM_TINY.img_size)
    md = MaskDecoder(transformer_dim=SAM_TINY.out_chans, transformer=TwoWayTransformer(2, SAM_TINY.out_chans, 8, 2048))
    sd = {"image_encoder." + k: v for k, v in make_sam_state_dict(SAM_TINY, 5).items()}
    sd.update({"prompt_encoder." + k: v for k, v in pe.state_dict().items()})
    sd.update({"mask_decoder." + k: v for k, v in md.state_dict().items()})
    ck = tmp_path / "sam_tiny.pth"
    torch.save(sd, ck)
    sam = S._builder(SAM_TINY)(checkpoint=str(ck))
    assert torch.equal(sam.mask_decoder.iou_token.weight, md.iou_token.weight)
    assert set(S.sam_model_registry) == {"default", "vit_h", "vit_l", "vit_b"}
    with pytest.raises(RuntimeError):                     # no CPU fallback for the encoder
        sam.image_encoder(torch.zeros(1, 3, 256, 256))
    with pytest.raises(KeyError):
        S.build_sam_from_state_dict(SAM_TINY, {"prompt_encoder.bogus": torch.zeros(1)})
