"""SAM prompt encoder, mask decoder and the `Sam` container (SURVEY.md §8b row B4, §8f N3), in PyTorch.

The image encoder - 5.96 of SAM's ~6 TFLOP per image - is `editanything_b200.sam.SamEncoderEngine` (sm_90a
kernels); the prompt encoder and the two-layer two-way mask decoder are a few MFLOP per prompt batch and stay
PyTorch modules.  Parameter names and tensor layouts follow the upstream `segment_anything` package so the official
checkpoints (`sam_vit_h_4b8939.pth`, editany_lora.py:54-66,85-87) load with `load_state_dict`; upstream itself is an
un-vendored git dependency of the reference and absent here, so the arithmetic is pinned against the in-container
HF port (transformers.models.sam) in tests/test_sam_shim_cpu.py - against upstream: parity unpinned.
"""
import math

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F


class LayerNorm2d(nn.Module):
    def __init__(self, c, eps=1e-6):
        super().__init__()
        self.weight, self.bias, self.eps = nn.Parameter(torch.ones(c)), nn.Parameter(torch.zeros(c)), eps

    def forward(self, x):
        u = x.mean(1, keepdim=True)
        s = (x - u).pow(2).mean(1, keepdim=True)
        return self.weight[:, None, None] * ((x - u) / torch.sqrt(s + self.eps)) + self.bias[:, None, None]


class PositionEmbeddingRandom(nn.Module):
    def __init__(self, num_pos_feats=64, scale=None):
        super().__init__()
        scale = 1.0 if scale is None or scale <= 0.0 else scale
        self.register_buffer("positional_encoding_gaussian_matrix", scale * torch.randn((2, num_pos_feats)))

    def _pe_encoding(self, coords):           # coords in [0, 1]^2
        coords = (2 * coords - 1) @ self.positional_encoding_gaussian_matrix
        coords = 2 * math.pi * coords
        return torch.cat([torch.sin(coords), torch.cos(coords)], dim=-1)

    def forward(self, size):
        h, w = size
        dev = self.positional_encoding_gaussian_matrix.device
        grid = torch.ones((h, w), device=dev, dtype=torch.float32)
        y = (grid.cumsum(0) - 0.5) / h
        x = (grid.cumsum(1) - 0.5) / w
        return self._pe_encoding(torch.stack([x, y], dim=-1)).permute(2, 0, 1)      # C x H x W

    def forward_with_coords(self, coords_input, image_size):
        c = coords_input.clone()
        c[:, :, 0] = c[:, :, 0] / image_size[1]
        c[:, :, 1] = c[:, :, 1] / image_size[0]
        return self._pe_encoding(c.to(torch.float))


class PromptEncoder(nn.Module):
    def __init__(self, embed_dim=256, image_embedding_size=(64, 64), input_image_size=(1024, 1024), mask_in_chans=16):
        super().__init__()
        self.embed_dim, self.input_image_size, self.image_embedding_size = embed_dim, input_image_size, image_embedding_size
        self.pe_layer = PositionEmbeddingRandom(embed_dim // 2)
        self.num_point_embeddings = 4                     # pos / neg point + 2 box corners
        self.point_embeddings = nn.ModuleList([nn.Embedding(1, embed_dim) for _ in range(4)])
        self.not_a_point_embed = nn.Embedding(1, embed_dim)
        self.mask_input_size = (4 * image_embedding_size[0], 4 * image_embedding_size[1])
        self.mask_downscaling = nn.Sequential(
            nn.Conv2d(1, mask_in_chans // 4, kernel_size=2, stride=2), LayerNorm2d(mask_in_chans // 4), nn.GELU(),
            nn.Conv2d(mask_in_chans // 4, mask_in_chans, kernel_size=2, stride=2), LayerNorm2d(mask_in_chans), nn.GELU(),
            nn.Conv2d(mask_in_chans, embed_dim, kernel_size=1))
        self.no_mask_embed = nn.Embedding(1, embed_dim)

    def get_dense_pe(self):
        return self.pe_layer(self.image_embedding_size).unsqueeze(0)

    def _embed_points(self, points, labels, pad):
        points = points + 0.5                              # pixel centre
        if pad:
            points = torch.cat([points, torch.zeros((points.shape[0], 1, 2), device=points.device)], dim=1)
            labels = torch.cat([labels, -torch.ones((labels.shape[0], 1), device=labels.device)], dim=1)
        pe = self.pe_layer.forward_with_coords(points, self.input_image_size)
        pe[labels == -1] = 0.0
        pe[labels == -1] += self.not_a_point_embed.weight
        pe[labels == 0] += self.point_embeddings[0].weight
        pe[labels == 1] += self.point_embeddings[1].weight
        return pe

    def _embed_boxes(self, boxes):
        boxes = boxes + 0.5
        ce = self.pe_layer.forward_with_coords(boxes.reshape(-1, 2, 2), self.input_image_size)
        ce[:, 0, :] += self.point_embeddings[2].weight
        ce[:, 1, :] += self.point_embeddings[3].weight
        return ce

    def forward(self, points, boxes, masks):
        if points is not None:
            bs = points[0].shape[0]
        elif boxes is not None:
            bs = boxes.shape[0]
        elif masks is not None:
            bs = masks.shape[0]
        else:
            bs = 1
        dev = self.point_embeddings[0].weight.device
        sparse = torch.empty((bs, 0, self.embed_dim), device=dev)
        if points is not None:
            coords, labels = points
            sparse = torch.cat([sparse, self._embed_points(coords, labels, pad=(boxes is None))], dim=1)
        if boxes is not None:
            sparse = torch.cat([sparse, self._embed_boxes(boxes)], dim=1)
        if masks is not None:
            dense = self.mask_downscaling(masks)
        else:
            dense = self.no_mask_embed.weight.reshape(1, -1, 1, 1).expand(bs, -1, self.image_embedding_size[0],
                                                                           self.image_embedding_size[1])
        return sparse, dense


class Attention(nn.Module):
    def __init__(self, embedding_dim, num_heads, downsample_rate=1):
        super().__init__()
        self.internal_dim, self.num_heads = embedding_dim // downsample_rate, num_heads
        self.q_proj = nn.Linear(embedding_dim, self.internal_dim)
        self.k_proj = nn.Linear(embedding_dim, self.internal_dim)
        self.v_proj = nn.Linear(embedding_dim, self.internal_dim)
        self.out_proj = nn.Linear(self.internal_dim, embedding_dim)

    def _heads(self, x):
        b, n, c = x.shape
        return x.reshape(b, n, self.num_heads, c // self.num_heads).transpose(1, 2)

    def forward(self, q, k, v):
        q, k, v = self._heads(self.q_proj(q)), self._heads(self.k_proj(k)), self._heads(self.v_proj(v))
        attn = torch.softmax(q @ k.transpose(-1, -2) / math.sqrt(q.shape[-1]), dim=-1)
        out = (attn @ v).transpose(1, 2)
        return self.out_proj(out.reshape(out.shape[0], out.shape[1], -1))


class MLPBlock(nn.Module):
    def __init__(self, embedding_dim, mlp_dim, act=nn.GELU):
        super().__init__()
        self.lin1, self.lin2, self.act = nn.Linear(embedding_dim, mlp_dim), nn.Linear(mlp_dim, embedding_dim), act()

    def forward(self, x):
        return self.lin2(self.act(self.lin1(x)))


class TwoWayAttentionBlock(nn.Module):
    def __init__(self, embedding_dim, num_heads, mlp_dim=2048, activation=nn.ReLU, attention_downsample_rate=2,
                 skip_first_layer_pe=False):
        super().__init__()
        self.self_attn = Attention(embedding_dim, num_heads)
        self.norm1 = nn.LayerNorm(embedding_dim)
        self.cross_attn_token_to_image = Attention(embedding_dim, num_heads, attention_downsample_rate)
        self.norm2 = nn.LayerNorm(embedding_dim)
        self.mlp = MLPBlock(embedding_dim, mlp_dim, activation)
        self.norm3 = nn.LayerNorm(embedding_dim)
        self.norm4 = nn.LayerNorm(embedding_dim)
        self.cross_attn_image_to_token = Attention(embedding_dim, num_heads, attention_downsample_rate)
        self.skip_first_layer_pe = skip_first_layer_pe

    def forward(self, queries, keys, query_pe, key_pe):
        if self.skip_first_layer_pe:
            queries = self.self_attn(queries, queries, queries)
        else:
            q = queries + query_pe
            queries = queries + self.self_attn(q, q, queries)
        queries = self.norm1(queries)
        q, k = queries + query_pe, keys + key_pe
        queries = self.norm2(queries + self.cross_attn_token_to_image(q, k, keys))
        queries = self.norm3(queries + self.mlp(queries))
        q, k = queries + query_pe, keys + key_pe
        keys = self.norm4(keys + self.cross_attn_image_to_token(k, q, queries))
        return queries, keys


class TwoWayTransformer(nn.Module):
    def __init__(self, depth, embedding_dim, num_heads, mlp_dim, activation=nn.ReLU, attention_downsample_rate=2):
        super().__init__()
        self.layers = nn.ModuleList([TwoWayAttentionBlock(embedding_dim, num_heads, mlp_dim, activation,
                                                          attention_downsample_rate, skip_first_layer_pe=(i == 0))
                                     for i in range(depth)])
        self.final_attn_token_to_image = Attention(embedding_dim, num_heads, attention_downsample_rate)
        self.norm_final_attn = nn.LayerNorm(embedding_dim)

    def forward(self, image_embedding, image_pe, point_embedding):
        image_embedding = image_embedding.flatten(2).permute(0, 2, 1)
        image_pe = image_pe.flatten(2).permute(0, 2, 1)
        queries, keys = point_embedding, image_embedding
        for layer in self.layers:
            queries, keys = layer(queries, keys, point_embedding, image_pe)
        q, k = queries + point_embedding, keys + image_pe
        queries = self.norm_final_attn(queries + self.final_attn_token_to_image(q, k, keys))
        return queries, keys


class MLP(nn.Module):
    def __init__(self, input_dim, hidden_dim, output_dim, num_layers, sigmoid_output=False):
        super().__init__()
        h = [hidden_dim] * (num_layers - 1)
        self.num_layers, self.sigmoid_output = num_layers, sigmoid_output
        self.layers = nn.ModuleList(nn.Linear(n, k) for n, k in zip([input_dim] + h, h + [output_dim]))

    def forward(self, x):
        for i, layer in enumerate(self.layers):
            x = F.relu(layer(x)) if i < self.num_layers - 1 else layer(x)
        return torch.sigmoid(x) if self.sigmoid_output else x


class MaskDecoder(nn.Module):
    def __init__(self, transformer_dim=256, transformer=None, num_multimask_outputs=3, iou_head_depth=3,
                 iou_head_hidden_dim=256):
        super().__init__()
        self.transformer_dim = transformer_dim
        self.transformer = transformer if transformer is not None else TwoWayTransformer(2, transformer_dim, 8, 2048)
        self.num_multimask_outputs = num_multimask_outputs
        self.iou_token = nn.Embedding(1, transformer_dim)
        self.num_mask_tokens = num_multimask_outputs + 1
        self.mask_tokens = nn.Embedding(self.num_mask_tokens, transformer_dim)
        self.output_upscaling = nn.Sequential(
            nn.ConvTranspose2d(transformer_dim, transformer_dim // 4, kernel_size=2, stride=2),
            LayerNorm2d(transformer_dim // 4), nn.GELU(),
            nn.ConvTranspose2d(transformer_dim // 4, transformer_dim // 8, kernel_size=2, stride=2), nn.GELU())
        self.output_hypernetworks_mlps = nn.ModuleList([MLP(transformer_dim, transformer_dim, transformer_dim // 8, 3)
                                                        for _ in range(self.num_mask_tokens)])
        self.iou_prediction_head = MLP(transformer_dim, iou_head_hidden_dim, self.num_mask_tokens, iou_head_depth)

    def forward(self, image_embeddings, image_pe, sparse_prompt_embeddings, dense_prompt_embeddings, multimask_output):
        out_tokens = torch.cat([self.iou_token.weight, self.mask_tokens.weight], dim=0)
        out_tokens = out_tokens.unsqueeze(0).expand(sparse_prompt_embeddings.size(0), -1, -1)
        tokens = torch.cat((out_tokens, sparse_prompt_embeddings), dim=1)
        src = torch.repeat_interleave(image_embeddings, tokens.shape[0], dim=0) + dense_prompt_embeddings
        pos_src = torch.repeat_interleave(image_pe, tokens.shape[0], dim=0)
        b, c, h, w = src.shape
        hs, src = self.transformer(src, pos_src, tokens)
        iou_token_out = hs[:, 0, :]
        mask_tokens_out = hs[:, 1:(1 + self.num_mask_tokens), :]
        up = self.output_upscaling(src.transpose(1, 2).reshape(b, c, h, w))
        hyper_in = torch.stack([m(mask_tokens_out[:, i, :]) for i, m in enumerate(self.output_hypernetworks_mlps)], dim=1)
        b, c, h, w = up.shape
        masks = (hyper_in @ up.reshape(b, c, h * w)).reshape(b, -1, h, w)
        iou_pred = self.iou_prediction_head(iou_token_out)
        sl = slice(1, None) if multimask_output else slice(0, 1)
        return masks[:, sl, :, :], iou_pred[:, sl]


class _EncoderModule(nn.Module):
    """`sam.image_encoder`: fp32 NCHW [B, 3, S, S] -> fp32 [B, 256, S/16, S/16] on the H100 engine.  The engine is
    built lazily on `.to(cuda device)` from the checkpoint tensors held until then (there is no CPU path)."""

    def __init__(self, cfg, state_dict):
        super().__init__()
        self.cfg, self._sd, self.engine = cfg, state_dict, None
        self.img_size = cfg.img_size

    def _apply(self, fn, *a, **k):
        from .. import _backend
        probe = fn(torch.zeros(1))
        if (probe.is_cuda or _backend.OPS is not None) and self.engine is None:     # (OPS: the CPU test-suite's seam)
            from ..sam import SamEncoderEngine
            self.engine = SamEncoderEngine(self.cfg, self._sd, probe.device)
            self._sd = None
        return super()._apply(fn, *a, **k)

    def forward(self, x):
        if self.engine is None:
            raise RuntimeError("the SAM image encoder runs on the H100 engine only: call sam.to('cuda') first "
                               "(there is no CPU fallback)")
        return self.engine(x)


class Sam(nn.Module):
    mask_threshold = 0.0
    image_format = "RGB"

    def __init__(self, image_encoder, prompt_encoder, mask_decoder, pixel_mean=(123.675, 116.28, 103.53),
                 pixel_std=(58.395, 57.12, 57.375)):
        super().__init__()
        self.image_encoder, self.prompt_encoder, self.mask_decoder = image_encoder, prompt_encoder, mask_decoder
        self.register_buffer("pixel_mean", torch.tensor(pixel_mean).view(-1, 1, 1), False)
        self.register_buffer("pixel_std", torch.tensor(pixel_std).view(-1, 1, 1), False)

    @property
    def device(self):
        return self.pixel_mean.device

    def preprocess(self, x):
        """Normalise and zero-pad (bottom / right) to the encoder's square input."""
        x = (x - self.pixel_mean) / self.pixel_std
        h, w = x.shape[-2:]
        s = self.image_encoder.img_size
        return F.pad(x, (0, s - w, 0, s - h))

    def postprocess_masks(self, masks, input_size, original_size):
        s = self.image_encoder.img_size
        masks = F.interpolate(masks, (s, s), mode="bilinear", align_corners=False)
        masks = masks[..., :input_size[0], :input_size[1]]
        return F.interpolate(masks, original_size, mode="bilinear", align_corners=False)
