"""First-stage (AutoencoderKL) decoder on the libea_b200 C-ABI operators — SURVEY.md §8f row N1, the
step right after the denoising loop (`decode_latents`, utils/stable_diffusion_controlnet_inpaint.py:
718-724: latents / scaling_factor -> vae.decode -> (x / 2 + 0.5).clamp(0, 1)).

Reference semantics followed (paths relative to the reference root):
    AutoencoderKL.decode          ldm/models/autoencoder.py:88-91      post_quant_conv (1x1) -> Decoder
    Decoder.forward               ldm/modules/diffusionmodules/model.py:623-652
    ResnetBlock.forward           model.py:129-148   GN(32, eps 1e-6) -> swish -> conv3x3 -> GN -> swish
                                                     -> conv3x3, + x (or + nin_shortcut 1x1 (x))
    AttnBlock.forward             model.py:181-210   GN -> q, k, v 1x1 -> softmax(q k^T C^-1/2) v -> proj, + x
    Upsample.forward              model.py:60-64     nearest x2 -> conv3x3
and, for the encode side (`prepare_masked_image_latents`, utils/...inpaint.py:1056-1105 -> vae.encode):
    AutoencoderKL.encode          ldm/models/autoencoder.py:82-86      Encoder -> quant_conv (1x1) -> moments
    Encoder.forward               model.py:519-543
    Downsample.forward            model.py:79-86     F.pad(x, (0,1,0,1)) -> conv3x3 stride 2 pad 0 (ea_gemm CONV_S2A)
    DiagonalGaussianDistribution  ldm/modules/distributions/distributions.py:24-45  mean, logvar.clamp(-30, 20)
Execution: channels-last half activations, fp32 accumulation; every 3x3 convolution is the wgmma
implicit GEMM (ea_gemm CONV_S1), the 1x1 shortcut of a channel-changing ResnetBlock rides along as extra
K columns of conv2, GroupNorm + swish is one fused launch, and the single-head attention (d = C, 512 in the
SD VAE) is, above FUSED_ATTN_MIN_TOKENS tokens, one q|k|v GEMM and one ea_attention launch over all images, so
the N x N logits are never stored; shorter sequences run two plain GEMMs around a row-softmax kernel (fp32 logits).
The last convolution (128 -> 3) is padded to 8 output channels so it can use the same GEMM; `ea_image_out`
drops the padding, applies
(x / 2 + 0.5).clamp(0, 1) and writes the fp32 NCHW image the pipeline hands to numpy / PIL.
"""
import types

import os

import torch

from . import _lib as L
from ._backend import default_ops, engine_call
from ._graphs import GraphLRU
from .vae_spec import SD_VAE, VAE_TINY, VaeConfig, decoder_blocks, encoder_blocks, make_vae_state_dict  # noqa: F401


# AttnBlock sequence lengths up to this run the logits as GEMMs around a row softmax, longer ones run ea_attention.
# On an H100 80GB HBM3 (700 W) at C = 512 the fused kernel took 2.1-2.2x the GEMM sequence's time at 64 x 64 latents
# (N = 4096: 64 CTAs of 64 query rows fill half the SMs), 1.04-1.06x at 128 x 128 and 0.91x at 192 x 256, while the
# GEMM sequence stores 6 N^2 bytes of logits (1.6 GB at N = 16384, 46.5 GB at 256 x 344).
FUSED_ATTN_MIN_TOKENS = 128 * 128


def _conv3_pack(w):  # [Cout, Cin, 3, 3] -> [Cout, (kh, kw, Cin)]
    return w.permute(0, 2, 3, 1).reshape(w.shape[0], -1)


class _VaeBase:
    """Weight packing and the ResnetBlock / AttnBlock executors shared by the two halves."""

    def _setup(self, cfg, device, backend):
        self.cfg, self.dev = cfg, device
        self.ops = backend or default_ops()
        self.hdt = self.ops.half_dtype()
        self.config = types.SimpleNamespace(scaling_factor=cfg.scaling_factor, latent_channels=cfg.z_channels,
                                            block_out_channels=cfg.block_out_channels)
        self.w = {}
        self._gn_ws = {}
        self._graphs = GraphLRU(int(os.environ.get("EA_GRAPH_CACHE", "4")))

    def _pack_blocks(self, sd, blocks):
        H, F, w = self._half, self._f32, self.w
        for kind, p, cin, cout in blocks:
            if kind == "res":
                for n in ("norm1", "norm2"):
                    w[f"{p}.{n}.g"], w[f"{p}.{n}.b"] = F(sd[f"{p}.{n}.weight"]), F(sd[f"{p}.{n}.bias"])
                w[p + ".conv1.w"], w[p + ".conv1.b"] = H(_conv3_pack(sd[p + ".conv1.weight"])), F(sd[p + ".conv1.bias"])
                c2, b2 = _conv3_pack(sd[p + ".conv2.weight"]), sd[p + ".conv2.bias"]
                if cin != cout:   # nin_shortcut as extra K columns of conv2 (same trick as the UNet ResBlock)
                    c2 = torch.cat([c2, sd[p + ".nin_shortcut.weight"].reshape(cout, cin)], 1)
                    b2 = b2 + sd[p + ".nin_shortcut.bias"]
                w[p + ".conv2.w"], w[p + ".conv2.b"] = H(c2), F(b2)
            elif kind == "attn":
                w[p + ".norm.g"], w[p + ".norm.b"] = F(sd[p + ".norm.weight"]), F(sd[p + ".norm.bias"])
                c = cin
                qkv = torch.cat([sd[f"{p}.{n}.weight"].reshape(c, c) for n in "qkv"], 0)
                w[p + ".qkv.w"], w[p + ".qkv.b"] = H(qkv), F(torch.cat([sd[f"{p}.{n}.bias"] for n in "qkv"]))
                w[p + ".proj.w"], w[p + ".proj.b"] = H(sd[p + ".proj_out.weight"].reshape(c, c)), F(sd[p + ".proj_out.bias"])
            else:   # upsample.conv / downsample.conv
                w[p + ".conv.w"], w[p + ".conv.b"] = H(_conv3_pack(sd[p + ".conv.weight"])), F(sd[p + ".conv.bias"])

    def _graphed(self, key, x, fn):
        """Run fn(static copy of x) through a CUDA graph captured once per `key` (CUDA backend only)."""
        st = self._graphs.get(key)
        if st is None:
            static_in = torch.zeros(tuple(x.shape), device=self.dev, dtype=torch.float32)
            static_in.copy_(x)
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                fn(static_in)                                      # warm-up: allocator, function attributes
            torch.cuda.current_stream().wait_stream(s)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                static_out = fn(static_in)
            st = self._graphs.put(key, (g, static_in, static_out))
        g, static_in, static_out = st
        static_in.copy_(x, non_blocking=True)
        g.replay()
        return static_out.clone()

    def _half(self, t):
        return t.detach().to(device=self.dev, dtype=self.hdt).contiguous()

    def _f32(self, t):
        return t.detach().to(device=self.dev, dtype=torch.float32).contiguous()

    def _new(self, *shape, dtype=None):
        return torch.empty(*shape, device=self.dev, dtype=dtype or self.hdt)

    def weight_bytes(self):
        return sum(t.numel() * t.element_size() for t in self.w.values())

    # ------------------------------------------------------------------------------------------
    def _gn(self, x, g, b, B, HW, C_, silu):
        out = self._new(B * HW, C_)
        ws = self._gn_ws.get(B)      # zero-initialised once; the kernel leaves it zeroed for the next launch
        if ws is None:
            ws = self._gn_ws[B] = self.ops.gn_workspace(B, self.dev, self.cfg.num_groups)
        self.ops.groupnorm(x, g, b, out, B=B, HW=HW, C_=C_, groups=self.cfg.num_groups, eps=self.cfg.eps,
                           silu=silu, workspace=ws)
        return out

    def _res(self, p, x, B, H, W_, cin, cout):
        o, w = self.ops, self.w
        a1 = self._gn(x, w[p + ".norm1.g"], w[p + ".norm1.b"], B, H * W_, cin, True)
        h1 = self._new(B * H * W_, cout)
        o.gemm(a1, w[p + ".conv1.w"], h1, mode=L.EA_GEMM_CONV_S1, conv=(B, H, W_, cin), bias=w[p + ".conv1.b"])
        a2 = self._gn(h1, w[p + ".norm2.g"], w[p + ".norm2.b"], B, H * W_, cout, True)
        out = self._new(B * H * W_, cout)
        if cin != cout:
            o.gemm(a2, w[p + ".conv2.w"], out, mode=L.EA_GEMM_CONV_S1, conv=(B, H, W_, cout),
                   a_extra=x.view(B, H, W_, cin), ld_extra=cin, bias=w[p + ".conv2.b"])
        else:
            o.gemm(a2, w[p + ".conv2.w"], out, mode=L.EA_GEMM_CONV_S1, conv=(B, H, W_, cout),
                   bias=w[p + ".conv2.b"], residual=x)
        return out

    def _attn(self, p, x, B, H, W_, c):
        o, w = self.ops, self.w
        N = H * W_
        hn = self._gn(x, w[p + ".norm.g"], w[p + ".norm.b"], B, N, c, False)
        qkv_w, qkv_b = w[p + ".qkv.w"], w[p + ".qkv.b"]
        if N <= FUSED_ATTN_MIN_TOKENS:
            # the logits as plain GEMMs around a row softmax, one image at a time
            qk = self._new(B * N, 2 * c)
            o.gemm(hn, qkv_w[:2 * c], qk, bias=qkv_b[:2 * c])
            out = self._new(B * N, c)
            s = self._new(N, N, dtype=torch.float32)
            pr = self._new(N, N)
            vt = self._new(c, N)
            ao = self._new(N, c)
            for b in range(B):
                rows = slice(b * N, (b + 1) * N)
                o.gemm(qk[rows, :c], qk[rows, c:], out_f32=s, K=c, lda=2 * c, ldw=2 * c, out_scale=float(c) ** -0.5)
                o.softmax_rows(s, pr, rows=N, cols=N)
                o.gemm(qkv_w[2 * c:], hn[rows], vt)                                  # V^T = Wv hn^T   [c, N]
                # softmax rows sum to 1, so v's bias passes straight through: P (V + 1 b^T) = P V + b^T
                o.gemm(pr, vt, ao, bias=qkv_b[2 * c:])
                o.gemm(ao, w[p + ".proj.w"], out[rows], bias=w[p + ".proj.b"], residual=x[rows])
            return out
        qkv = self._new(B * N, 3 * c)
        o.gemm(hn, qkv_w, qkv, bias=qkv_b)
        ao = self._new(B * N, c)
        st = (N * 3 * c, 3 * c)                              # one head of d = c per image
        o.attention(qkv, qkv[:, c:], qkv[:, 2 * c:], ao, B=B, heads=1, Nq=N, Nkv=N, d=c, q_strides=st,
                    k_strides=st, v_strides=st, o_strides=(N * c, c), scale=float(c) ** -0.5)
        out = self._new(B * N, c)
        o.gemm(ao, w[p + ".proj.w"], out, bias=w[p + ".proj.b"], residual=x)
        return out


class VaeDecoderEngine(_VaeBase):
    """Drop-in for `pipe.vae` on the decode side: `.decode(z).sample`, `.config.scaling_factor`,
    `.config.block_out_channels` (what StableDiffusionControlNetInpaintPipeline reads), plus
    `decode_latents(latents)` = the pipeline method's tensor part in one call."""

    def __init__(self, cfg: VaeConfig, state_dict, device, backend=None):
        self._setup(cfg, device, backend)
        sd = {k[len("first_stage_model."):] if k.startswith("first_stage_model.") else k: v
              for k, v in state_dict.items()}
        H, F, w = self._half, self._f32, self.w
        # tiny-depth convolutions run on the direct kernels: fp32 weights laid out [kh, kw, Cin, Cout]
        w["pqc.w"] = F(sd["post_quant_conv.weight"].permute(2, 3, 1, 0))
        w["pqc.b"] = F(sd["post_quant_conv.bias"])
        w["cin.w"] = F(sd["decoder.conv_in.weight"].permute(2, 3, 1, 0))
        w["cin.b"] = F(sd["decoder.conv_in.bias"])
        self.blocks, last = decoder_blocks(cfg)
        self._pack_blocks(sd, self.blocks)
        w["nout.g"], w["nout.b"] = F(sd["decoder.norm_out.weight"]), F(sd["decoder.norm_out.bias"])
        co = _conv3_pack(sd["decoder.conv_out.weight"])                       # [3, 9*C]
        self.cout_pad = 8
        cop = torch.zeros(self.cout_pad, co.shape[1], dtype=co.dtype, device=co.device)
        cop[:cfg.out_ch] = co
        bop = torch.zeros(self.cout_pad, dtype=co.dtype, device=co.device)
        bop[:cfg.out_ch] = sd["decoder.conv_out.bias"]
        w["cout.w"], w["cout.b"] = H(cop), F(bop)
        self.last_ch = last

    @engine_call
    def decode(self, z):
        """z: [B, z_channels, h, w] (already divided by scaling_factor) -> object with
        `.sample` = fp32 [B, 3, 8h, 8w] in the decoder's native range (about [-1, 1])."""
        return types.SimpleNamespace(sample=self._decode(z, post=False))

    @engine_call
    def decode_latents(self, latents, use_graph=True):
        """latents as the denoising loop leaves them -> fp32 [B, 3, 8h, 8w] in [0, 1]
        (decode_latents up to the .cpu().permute().numpy() plumbing).  On the CUDA backend the launches (71
        for the SD VAE) are captured once per latent shape into a CUDA graph and replayed."""
        if not use_graph or self.dev.type != "cuda":
            return self._decode(latents.float() / self.cfg.scaling_factor, post=True)
        return self._graphed(("dec",) + tuple(latents.shape), latents,
                             lambda x: self._decode(x / self.cfg.scaling_factor, post=True))

    def _decode(self, z, post):
        o, w, cfg = self.ops, self.w, self.cfg
        B, zc, H, W_ = z.shape
        if zc != cfg.z_channels:
            raise ValueError(f"expected {cfg.z_channels} latent channels, got {zc}")
        zh = z.to(self.dev).permute(0, 2, 3, 1).contiguous().to(self.hdt)          # NHWC half [B,h,w,4]
        y = self._new(B * H * W_, cfg.z_channels)
        o.conv_direct(zh, w["pqc.w"], w["pqc.b"], y, B=B, Hin=H, Win=W_, Cin=cfg.embed_dim, Cout=cfg.z_channels,
                      ksize=1)
        top = cfg.ch * cfg.ch_mult[-1]
        h = self._new(B * H * W_, top)
        o.conv_direct(y, w["cin.w"], w["cin.b"], h, B=B, Hin=H, Win=W_, Cin=cfg.z_channels, Cout=top, ksize=3)
        for kind, p, cin, cout in self.blocks:
            if kind == "res":
                h = self._res(p, h, B, H, W_, cin, cout)
            elif kind == "attn":
                h = self._attn(p, h, B, H, W_, cin)
            else:
                up = self._new(B * 4 * H * W_, cin)
                o.upsample2x(h, up, B=B, H=H, W=W_, C_=cin)
                H, W_ = 2 * H, 2 * W_
                h = self._new(B * H * W_, cin)
                o.gemm(up, w[p + ".conv.w"], h, mode=L.EA_GEMM_CONV_S1, conv=(B, H, W_, cin), bias=w[p + ".conv.b"])
        a = self._gn(h, w["nout.g"], w["nout.b"], B, H * W_, self.last_ch, True)
        y8 = self._new(B * H * W_, self.cout_pad)
        o.gemm(a, w["cout.w"], y8, mode=L.EA_GEMM_CONV_S1, conv=(B, H, W_, self.last_ch), bias=w["cout.b"])
        img = torch.empty(B, cfg.out_ch, H, W_, device=self.dev, dtype=torch.float32)
        if post:
            o.image_out(y8, img, B=B, HW=H * W_, C_=cfg.out_ch, ldx=self.cout_pad, scale=0.5, shift=0.5, lo=0.0, hi=1.0)
        else:
            o.image_out(y8, img, B=B, HW=H * W_, C_=cfg.out_ch, ldx=self.cout_pad, scale=1.0, shift=0.0,
                        lo=-3.0e38, hi=3.0e38)
        return img


class DiagonalGaussian:
    """`vae.encode(x).latent_dist` (ldm/modules/distributions/distributions.py:24-45; diffusers'
    DiagonalGaussianDistribution has the same arithmetic): moments [B, 2z, h, w] -> mean | logvar."""

    def __init__(self, moments):
        self.mean, logvar = torch.chunk(moments, 2, dim=1)
        self.logvar = torch.clamp(logvar, -30.0, 20.0)
        self.std = torch.exp(0.5 * self.logvar)
        self.var = torch.exp(self.logvar)

    def sample(self, generator=None):
        # plumbing on a [B, z, h, w] tensor; noise drawn on the generator's device like diffusers' randn_tensor
        gdev = generator.device if generator is not None else self.mean.device
        noise = torch.randn(self.mean.shape, generator=generator, device=gdev, dtype=self.mean.dtype)
        return self.mean + self.std * noise.to(self.mean.device)

    def mode(self):
        return self.mean


class VaeEncoderEngine(_VaeBase):
    """Encode side of `pipe.vae`: `.encode(x).latent_dist.sample(generator)` with x the [-1, 1] image
    [B, 3, H, W] (prepare_masked_image_latents, utils/...inpaint.py:1056-1105; the caller multiplies the
    sample by `config.scaling_factor`)."""

    def __init__(self, cfg: VaeConfig, state_dict, device, backend=None):
        self._setup(cfg, device, backend)
        sd = {k[len("first_stage_model."):] if k.startswith("first_stage_model.") else k: v
              for k, v in state_dict.items()}
        H, F, w = self._half, self._f32, self.w
        ci = sd["encoder.conv_in.weight"]                                    # [ch, 3, 3, 3]
        self.in_ch = ci.shape[1]
        cip = torch.zeros(ci.shape[0], 4, 3, 3, dtype=ci.dtype, device=ci.device)   # image padded to 4 channels
        cip[:, :self.in_ch] = ci
        w["cin.w"], w["cin.b"] = F(cip.permute(2, 3, 1, 0)), F(sd["encoder.conv_in.bias"])
        self.blocks, last = encoder_blocks(cfg)
        self._pack_blocks(sd, self.blocks)
        w["nout.g"], w["nout.b"] = F(sd["encoder.norm_out.weight"]), F(sd["encoder.norm_out.bias"])
        w["cout.w"], w["cout.b"] = H(_conv3_pack(sd["encoder.conv_out.weight"])), F(sd["encoder.conv_out.bias"])
        w["qc.w"], w["qc.b"] = F(sd["quant_conv.weight"].permute(2, 3, 1, 0)), F(sd["quant_conv.bias"])
        self.last_ch = last
        if (2 * cfg.z_channels) % 8 != 0:
            raise ValueError("2 * z_channels must be a multiple of 8 (GEMM output width)")

    @engine_call
    def encode(self, x, use_graph=True):
        if x.dim() != 4 or x.shape[1] != self.in_ch:
            raise ValueError(f"expected [B, {self.in_ch}, H, W], got {tuple(x.shape)}")
        f = 2 ** (self.cfg.num_resolutions - 1)
        if x.shape[2] % f or x.shape[3] % f:
            raise ValueError(f"image sides must be multiples of {f}")
        if use_graph and self.dev.type == "cuda":
            m = self._graphed(("enc",) + tuple(x.shape), x, self._moments)
        else:
            m = self._moments(x.float())
        return types.SimpleNamespace(latent_dist=DiagonalGaussian(m))

    def _moments(self, x):
        """fp32 NCHW image -> fp32 NCHW moments [B, 2z, H/f, W/f] (AutoencoderKL.encode before sampling)."""
        o, w, cfg = self.ops, self.w, self.cfg
        B, _, H, W_ = x.shape
        xh = torch.zeros(B, H, W_, 4, device=self.dev, dtype=self.hdt)
        xh[..., :self.in_ch] = x.to(self.dev).permute(0, 2, 3, 1)                  # NHWC half, 4th channel zero
        h = self._new(B * H * W_, cfg.ch)
        o.conv_in(xh, w["cin.w"], w["cin.b"], h, B=B, H=H, W=W_, Cin=4, Cout=cfg.ch)
        for kind, p, cin, cout in self.blocks:
            if kind == "res":
                h = self._res(p, h, B, H, W_, cin, cout)
            elif kind == "attn":
                h = self._attn(p, h, B, H, W_, cin)
            else:   # Downsample: pad (0,1,0,1), conv3x3 stride 2
                H, W_ = H // 2, W_ // 2
                d = self._new(B * H * W_, cin)
                o.gemm(h, w[p + ".conv.w"], d, mode=L.EA_GEMM_CONV_S2A, conv=(B, H, W_, cin), bias=w[p + ".conv.b"])
                h = d
        a = self._gn(h, w["nout.g"], w["nout.b"], B, H * W_, self.last_ch, True)
        zc2 = 2 * cfg.z_channels
        m0 = self._new(B * H * W_, zc2)
        o.gemm(a, w["cout.w"], m0, mode=L.EA_GEMM_CONV_S1, conv=(B, H, W_, self.last_ch), bias=w["cout.b"])
        m1 = self._new(B * H * W_, 2 * cfg.embed_dim)
        o.conv_direct(m0, w["qc.w"], w["qc.b"], m1, B=B, Hin=H, Win=W_, Cin=zc2, Cout=2 * cfg.embed_dim, ksize=1)
        out = torch.empty(B, 2 * cfg.embed_dim, H, W_, device=self.dev, dtype=torch.float32)
        o.nhwc_to_nchw_f32(m1, out, B=B, HW=H * W_, C_=2 * cfg.embed_dim)
        return out


class VaeEngine:
    """Both halves behind the one object the pipeline holds as `pipe.vae` (encode, decode,
    decode_latents, config)."""

    def __init__(self, cfg: VaeConfig, state_dict, device, backend=None):
        self.encoder = VaeEncoderEngine(cfg, state_dict, device, backend)
        self.decoder = VaeDecoderEngine(cfg, state_dict, device, backend)
        self.config = self.decoder.config
        self.encode, self.decode, self.decode_latents = self.encoder.encode, self.decoder.decode, self.decoder.decode_latents
