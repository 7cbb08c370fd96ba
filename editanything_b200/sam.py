"""SAM ViT image encoder on the libea_b200 C-ABI operators (SURVEY.md §8a row R1).

Drop-in for `Sam.image_encoder` (the nn.Module `SamAutomaticMaskGenerator.generate` /
`SamPredictor.set_image` call once per image — reference call sites editany_lora.py:82-95,
522-541): `SamEncoderEngine.__call__(x)` takes the preprocessed fp32 NCHW image
[B, 3, 1024, 1024] and returns the fp32 NCHW embedding [B, 256, 64, 64].

Upstream semantics followed (segment_anything/modeling/image_encoder.py; line refs into the
in-container HF port transformers/models/sam/modeling_sam.py, "HF:"):
    PatchEmbed + pos_embed     HF:97-129,1065-1066   im2col kernel -> ea_gemm (+bias, +pos_embed residual)
    Block                      HF:954-972            LN -> [pad+window partition] -> attention ->
                                                     [unpartition] + residual -> LN -> MLP + residual
    Attention                  HF:803-831            qkv ea_gemm (+bias) -> decomposed rel-pos terms
                                                     from the UNSCALED q -> fused wgmma attention with the
                                                     rel-pos bias added to the fp32 logits -> proj ea_gemm
    window partition           HF:900-952            zero padding AFTER LayerNorm; padded tokens are
                                                     real keys (k, v = qkv bias), not masked
    neck                       HF:975-992            1x1 conv (ea_gemm) -> LayerNorm2d -> 3x3 conv
                                                     (implicit GEMM) -> LayerNorm2d
Activations are channels-last half [tokens, C]; all accumulation fp32.
"""
import os

import torch

from . import _lib as L
from ._backend import default_ops, engine_call
from ._graphs import GraphLRU
from .sam_spec import SAM_TINY, SAM_VIT_H, SamEncoderConfig, make_sam_state_dict  # noqa: F401


def _gather_rel_pos(table, S):
    """get_rel_pos for q_size == k_size == S (HF:729-759): R[q, k, :] = table[q - k + S - 1]."""
    if table.shape[0] != 2 * S - 1:
        raise ValueError(f"rel_pos table of length {table.shape[0]} for window {S}: interpolated tables are not supported")
    idx = torch.arange(S)[:, None] - torch.arange(S)[None, :] + (S - 1)
    return table[idx.to(table.device)]


class SamEncoderEngine:
    def __init__(self, cfg: SamEncoderConfig, state_dict, device, backend=None):
        self.cfg, self.dev = cfg, device
        self.ops = backend or default_ops()
        self.hdt = self.ops.half_dtype()
        sd = {k[len("image_encoder."):] if k.startswith("image_encoder.") else k: v for k, v in state_dict.items()}
        H, F = self._half, self._f32
        D, g = cfg.embed_dim, cfg.grid
        w = {}
        w["pe.w"] = H(sd["patch_embed.proj.weight"].reshape(D, -1))
        w["pe.b"] = F(sd["patch_embed.proj.bias"])
        w["pos"] = H(sd["pos_embed"].reshape(g * g, D))
        for i in range(cfg.depth):
            p, q = f"blocks.{i}", f"b{i}"
            S = g if i in cfg.global_attn_indexes else cfg.window_size
            for n in ("norm1", "norm2"):
                w[f"{q}.{n}.g"], w[f"{q}.{n}.b"] = F(sd[f"{p}.{n}.weight"]), F(sd[f"{p}.{n}.bias"])
            w[q + ".qkv.w"], w[q + ".qkv.b"] = H(sd[p + ".attn.qkv.weight"]), F(sd[p + ".attn.qkv.bias"])
            w[q + ".proj.w"], w[q + ".proj.b"] = H(sd[p + ".attn.proj.weight"]), F(sd[p + ".attn.proj.bias"])
            w[q + ".Rh"] = F(_gather_rel_pos(sd[p + ".attn.rel_pos_h"], S))
            w[q + ".Rw"] = F(_gather_rel_pos(sd[p + ".attn.rel_pos_w"], S))
            w[q + ".fc1.w"], w[q + ".fc1.b"] = H(sd[p + ".mlp.lin1.weight"]), F(sd[p + ".mlp.lin1.bias"])
            w[q + ".fc2.w"], w[q + ".fc2.b"] = H(sd[p + ".mlp.lin2.weight"]), F(sd[p + ".mlp.lin2.bias"])
        oc = cfg.out_chans
        w["neck0.w"] = H(sd["neck.0.weight"].reshape(oc, D))
        w["neck1.g"], w["neck1.b"] = F(sd["neck.1.weight"]), F(sd["neck.1.bias"])
        w["neck2.w"] = H(sd["neck.2.weight"].permute(0, 2, 3, 1).reshape(oc, -1))
        w["neck3.g"], w["neck3.b"] = F(sd["neck.3.weight"]), F(sd["neck.3.bias"])
        self.w = w
        self._bufs = {}
        self._graphs = GraphLRU(int(os.environ.get("EA_GRAPH_CACHE", "4")))

    def _half(self, t):
        return t.detach().to(device=self.dev, dtype=self.hdt).contiguous()

    def _f32(self, t):
        return t.detach().to(device=self.dev, dtype=torch.float32).contiguous()

    def weight_bytes(self):
        return sum(t.numel() * t.element_size() for t in self.w.values())

    def _buf(self, name, shape, dtype=None):
        """Named workspace reused across blocks and calls (stable addresses, no allocator traffic)."""
        dtype = dtype or self.hdt
        key = (name, tuple(shape), dtype)
        b = self._bufs.get(key)
        if b is None:
            b = torch.empty(*shape, device=self.dev, dtype=dtype)
            self._bufs[key] = b
        return b

    # ------------------------------------------------------------------------------------------
    def _block(self, i, x, B):
        o, w, cfg = self.ops, self.w, self.cfg
        q = f"b{i}"
        D, g, heads, d = cfg.embed_dim, cfg.grid, cfg.num_heads, cfg.head_dim
        T = B * g * g
        ws = 0 if i in cfg.global_attn_indexes else cfg.window_size
        n1 = self._buf("ln", (T, D))
        o.layernorm(x, w[q + ".norm1.g"], w[q + ".norm1.b"], n1, M=T, C_=D, eps=cfg.ln_eps)
        if ws > 0:
            nW = (g + ws - 1) // ws
            Bw, S = B * nW * nW, ws
            a_in = self._buf("win", (Bw * S * S, D))
            o.window_partition(n1, a_in, B=B, H=g, W=g, C_=D, ws=ws)
        else:
            Bw, S, a_in = B, g, n1
        Tw = Bw * S * S
        qkv = self._buf("qkv", (Tw, 3 * D))
        o.gemm(a_in, w[q + ".qkv.w"], qkv, bias=w[q + ".qkv.b"])
        rel_h = self._buf("relh", (Bw * heads, S * S, S), torch.float32)
        rel_w = self._buf("relw", (Bw * heads, S * S, S), torch.float32)
        o.sam_relpos(qkv, S * S * 3 * D, 3 * D, w[q + ".Rh"], w[q + ".Rw"], rel_h, rel_w, B=Bw, heads=heads, S=S, d=d)
        ao = self._buf("ao", (Tw, D))
        st = (S * S * 3 * D, 3 * D)
        o.attention(qkv, qkv[:, D:], qkv[:, 2 * D:], ao, B=Bw, heads=heads, Nq=S * S, Nkv=S * S, d=d,
                    q_strides=st, k_strides=st, v_strides=st, o_strides=(S * S * D, D), scale=d ** -0.5,
                    rel_h=rel_h, rel_w=rel_w, rel_s=S)
        x1 = self._buf("x1", (T, D))
        if ws > 0:
            pr = self._buf("proj", (Tw, D))
            o.gemm(ao, w[q + ".proj.w"], pr, bias=w[q + ".proj.b"])
            o.window_unpartition(pr, x, x1, B=B, H=g, W=g, C_=D, ws=ws)
        else:
            o.gemm(ao, w[q + ".proj.w"], x1, bias=w[q + ".proj.b"], residual=x)
        n2 = self._buf("ln", (T, D))
        o.layernorm(x1, w[q + ".norm2.g"], w[q + ".norm2.b"], n2, M=T, C_=D, eps=cfg.ln_eps)
        hmid = self._buf("mlp", (T, cfg.mlp_dim))
        o.gemm(n2, w[q + ".fc1.w"], hmid, bias=w[q + ".fc1.b"], act=L.EA_ACT_GELU)
        o.gemm(hmid, w[q + ".fc2.w"], x, bias=w[q + ".fc2.b"], residual=x1)   # x is dead: reuse as output
        return x

    def tokens(self, img):
        """Patch embedding + all transformer blocks: half [B*g*g, D]."""
        o, w, cfg = self.ops, self.w, self.cfg
        B = img.shape[0]
        g, D = cfg.grid, cfg.embed_dim
        img = img.to(self.dev, torch.float32).contiguous()
        K = cfg.in_chans * cfg.patch_size ** 2
        cols = self._buf("cols", (B * g * g, K))
        o.sam_patchify(img, cols, B=B, Cin=cfg.in_chans, H=cfg.img_size, W=cfg.img_size, ps=cfg.patch_size)
        x = self._buf("x", (B * g * g, D))
        for b in range(B):   # pos_embed is per image: residual rows restart at every image
            sl = slice(b * g * g, (b + 1) * g * g)
            o.gemm(cols[sl], w["pe.w"], x[sl], bias=w["pe.b"], residual=w["pos"])
        for i in range(cfg.depth):
            x = self._block(i, x, B)
        return x

    @engine_call
    def encode(self, img, use_graph=True):
        """img: fp32 [B, 3, S, S] preprocessed (Sam.preprocess) -> fp32 [B, out_chans, S/16, S/16].
        On the CUDA backend the ~320 launches of one encode are captured once per batch size into a
        CUDA graph and replayed (the Python/ctypes launch path costs more than the kernels)."""
        cfg = self.cfg
        B = img.shape[0]
        if tuple(img.shape[1:]) != (cfg.in_chans, cfg.img_size, cfg.img_size):
            raise ValueError(f"expected [B,{cfg.in_chans},{cfg.img_size},{cfg.img_size}], got {tuple(img.shape)}")
        if not use_graph or self.dev.type != "cuda":
            return self._encode_eager(img)
        st = self._graphs.get(B)
        if st is None:
            static_in = torch.zeros(B, cfg.in_chans, cfg.img_size, cfg.img_size, device=self.dev, dtype=torch.float32)
            static_in.copy_(img)
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                self._encode_eager(static_in)          # warm-up: allocator, cudaFuncSetAttribute
            torch.cuda.current_stream().wait_stream(s)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                static_out = self._encode_eager(static_in)
            st = (g, static_in, static_out)
            self._graphs.put(B, st)
        g, static_in, static_out = st
        static_in.copy_(img, non_blocking=True)
        g.replay()
        return static_out.clone()

    def _encode_eager(self, img):
        o, w, cfg = self.ops, self.w, self.cfg
        B = img.shape[0]
        g, oc = cfg.grid, cfg.out_chans
        T = B * g * g
        x = self.tokens(img)
        y0 = self._buf("neck0", (T, oc))
        o.gemm(x, w["neck0.w"], y0)
        y1 = self._buf("neck1", (T, oc))
        o.layernorm(y0, w["neck1.g"], w["neck1.b"], y1, M=T, C_=oc, eps=1e-6)
        o.gemm(y1, w["neck2.w"], y0, mode=L.EA_GEMM_CONV_S1, conv=(B, g, g, oc))
        o.layernorm(y0, w["neck3.g"], w["neck3.b"], y1, M=T, C_=oc, eps=1e-6)
        out = torch.empty(B, oc, g, g, device=self.dev, dtype=torch.float32)
        o.nhwc_to_nchw_f32(y1, out, B=B, HW=g * g, C_=oc)
        return out

    __call__ = encode
