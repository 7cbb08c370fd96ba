"""Host-side executor of the SD UNet / ControlNet on the libea_b200 C-ABI operators.

Mirrors the reference call contracts (SURVEY.md §8b B3):
    controlnet(sample, t, encoder_hidden_states, controlnet_cond, conditioning_scale) -> residuals
    unet(sample, t, encoder_hidden_states, down_block_additional_residuals, mid_...)  -> eps
but executes them channels-last on hand-written sm_90a kernels, with the ControlNet residuals
never materialised as separate tensors: every zero-conv GEMM accumulates `scale * residual`
straight into the UNet's skip-concat buffers (cldm/cldm.py:34-41), and CFG + the DDIM update run in
the epilogue of the final convolution (cldm/ddim_hacked.py:190-231).

Reference semantics followed (paths relative to the reference root):
    ControlledUnetModel.forward   cldm/cldm.py:22-45
    ControlNet.forward            cldm/cldm.py:284-305
    ResBlock._forward             ldm/modules/diffusionmodules/openaimodel.py:254-274
    SpatialTransformer.forward    ldm/modules/attention.py:321-340
    BasicTransformerBlock         ldm/modules/attention.py:271-275
"""
import os
from dataclasses import replace

import torch

from . import _lib as L
from ._backend import default_ops
from .unet_spec import HINT_STRIDES, UNetConfig, build_topology


def _conv3_pack(w):  # [Cout, Cin, 3, 3] -> [Cout, (kh, kw, Cin)]
    return w.permute(0, 2, 3, 1).reshape(w.shape[0], -1)


def _geglu_interleave(n_inner):
    """Row permutation so each 128-row block of the GEGLU projection holds 64 value rows followed
    by their 64 gate rows (attention.py:54-56 chunks [value | gate] along the last dim)."""
    idx = []
    for j in range(n_inner // 64):
        idx.append(torch.arange(j * 64, j * 64 + 64))
        idx.append(n_inner + torch.arange(j * 64, j * 64 + 64))
    return torch.cat(idx)


class PackedNet:
    """Device-resident, kernel-layout weights of one UNet or ControlNet (built once, after any LoRA
    merge — editany_lora.py:197-329 merges LoRA deltas into the weights in place)."""

    def __init__(self, cfg: UNetConfig, kind: str, state_dict, device, backend=None):
        self.cfg, self.kind = cfg, kind
        self.ops = backend or default_ops()
        # LayerNorm folded into the GEMMs around it (ea_gemm_args.rowstats_out / ln_*): no LayerNorm launch, no
        # normalised tensor.  EA_LN_FOLD=0 keeps the separate ea_layernorm launches (A/B, debugging).
        self.ln_fold = os.environ.get("EA_LN_FOLD", "1") != "0"
        self.dev = device
        self.hdt = self.ops.half_dtype()
        self.topo = build_topology(cfg, with_decoder=(kind == "unet"))
        # channels of the per-step input x: the latents only, also for a 9-channel inpainting UNet
        self.x_channels = 4 if (kind == "unet" and cfg.in_channels == 9) else cfg.in_channels
        sd = state_dict
        self.w = {}
        H, F = self._half, self._f32

        # time embedding MLP + every ResBlock's emb projection as ONE matrix
        self.w["te0.w"], self.w["te0.b"] = H(sd["time_embed.0.weight"]), F(sd["time_embed.0.bias"])
        self.w["te2.w"], self.w["te2.b"] = H(sd["time_embed.2.weight"]), F(sd["time_embed.2.bias"])
        emb_w, emb_b, self.emb_off = [], [], {}
        off = 0
        blocks = [b for layers in self.topo.input_blocks for b in layers] + list(self.topo.middle)
        if kind == "unet":
            blocks += [b for layers in self.topo.output_blocks for b in layers]
        for b in blocks:
            if b.kind == "res":
                p = b.prefix
                emb_w.append(sd[p + ".emb_layers.1.weight"])
                # conv1 bias folded into the per-(batch, channel) row vector
                emb_b.append(sd[p + ".emb_layers.1.bias"] + sd[p + ".in_layers.2.bias"])
                self.emb_off[p] = off
                off += b.cout
        self.emb_total = off
        self.w["emb.w"], self.w["emb.b"] = H(torch.cat(emb_w, 0)), F(torch.cat(emb_b, 0))

        for b in blocks:
            p = b.prefix
            if b.kind == "conv_in":
                wt = sd[p + ".weight"]
                if self.x_channels != b.cin:
                    # 9-channel UNet: conv(cat[x, c], W) + b = conv(x, W_x) + (conv(c, W_c) + b).  W_x (the latent's
                    # 4 channels) runs every step; W_c (mask + masked-image latents, zero-padded to 8 channels) runs
                    # once per request in precompute_condition and is added through conv_in's `add`
                    wc = torch.zeros(wt.shape[0], 8, 3, 3, dtype=wt.dtype, device=wt.device)
                    wc[:, :b.cin - 4] = wt[:, 4:]
                    self.w[p + ".wc"] = F(wc.permute(2, 3, 1, 0))
                    wt = wt[:, :4]
                self.w[p + ".w"] = F(wt.permute(2, 3, 1, 0))  # [k,k,Cin,Cout]
                self.w[p + ".b"] = F(sd[p + ".bias"])
            elif b.kind == "res":
                for n in ("in_layers.0", "out_layers.0"):
                    self.w[f"{p}.{n}.g"], self.w[f"{p}.{n}.b"] = F(sd[f"{p}.{n}.weight"]), F(sd[f"{p}.{n}.bias"])
                self.w[p + ".conv1.w"] = H(_conv3_pack(sd[p + ".in_layers.2.weight"]))
                w2 = _conv3_pack(sd[p + ".out_layers.3.weight"])
                b2 = sd[p + ".out_layers.3.bias"]
                if b.cin != b.cout:  # fold the 1x1 skip conv in as extra K columns
                    w2 = torch.cat([w2, sd[p + ".skip_connection.weight"].reshape(b.cout, b.cin)], 1)
                    b2 = b2 + sd[p + ".skip_connection.bias"]
                self.w[p + ".conv2.w"], self.w[p + ".conv2.b"] = H(w2), F(b2)
            elif b.kind == "attn":
                self._pack_attn(sd, p, b.cin)
            elif b.kind == "down":
                self.w[p + ".w"], self.w[p + ".b"] = H(_conv3_pack(sd[p + ".op.weight"])), F(sd[p + ".op.bias"])
            elif b.kind == "up":
                self.w[p + ".w"], self.w[p + ".b"] = H(_conv3_pack(sd[p + ".conv.weight"])), F(sd[p + ".conv.bias"])
        if kind == "unet":
            self.w["out.g"], self.w["out.b"] = F(sd["out.0.weight"]), F(sd["out.0.bias"])
            self.w["out.w"] = F(sd["out.2.weight"].permute(0, 2, 3, 1))  # [4,3,3,C]
            self.w["out.cb"] = F(sd["out.2.bias"])
        else:
            for i in range(len(HINT_STRIDES)):
                p = f"input_hint_block.{2 * i}"
                self.w[p + ".w"] = F(sd[p + ".weight"].permute(2, 3, 1, 0))
                self.w[p + ".b"] = F(sd[p + ".bias"])
                if i > 0:
                    # tensor-core form of layers 2..8: channels zero-padded to multiples of 64 (the implicit-GEMM
                    # convolution needs Cin % 64 == 0); padded output channels get zero weights and bias, so they
                    # stay exactly 0 through SiLU and feed zeros into the next layer's padded inputs
                    wt = sd[p + ".weight"]
                    co, ci = wt.shape[0], wt.shape[1]
                    co_p = co if i == len(HINT_STRIDES) - 1 else -(-co // 64) * 64
                    ci_p = -(-ci // 64) * 64
                    wp = torch.zeros(co_p, 3, 3, ci_p, dtype=wt.dtype, device=wt.device)
                    wp[:co, :, :, :ci] = wt.permute(0, 2, 3, 1)
                    bp = torch.zeros(co_p, dtype=wt.dtype, device=wt.device)
                    bp[:co] = sd[p + ".bias"]
                    self.w[p + ".wp"], self.w[p + ".bp"] = H(wp.reshape(co_p, -1)), F(bp)
            for i, c in enumerate(self.topo.input_chans):
                p = f"zero_convs.{i}.0"
                self.w[p + ".w"], self.w[p + ".b"] = H(sd[p + ".weight"].reshape(c, c)), F(sd[p + ".bias"])
            c = self.topo.middle[-1].cout
            self.w["mid_out.w"] = H(sd["middle_block_out.0.weight"].reshape(c, c))
            self.w["mid_out.b"] = F(sd["middle_block_out.0.bias"])

    def _half(self, t):
        return t.detach().to(device=self.dev, dtype=self.hdt).contiguous()

    def _f32(self, t):
        return t.detach().to(device=self.dev, dtype=torch.float32).contiguous()

    def _pack_attn(self, sd, p, c):
        H, F = self._half, self._f32
        heads, dh = self.cfg.heads_for(c)
        inner = heads * dh
        tb = p + ".transformer_blocks.0"
        self.w[p + ".norm.g"], self.w[p + ".norm.b"] = F(sd[p + ".norm.weight"]), F(sd[p + ".norm.bias"])
        self.w[p + ".proj_in.w"] = H(sd[p + ".proj_in.weight"].reshape(inner, c))
        self.w[p + ".proj_in.b"] = F(sd[p + ".proj_in.bias"])
        self.w[p + ".proj_out.w"] = H(sd[p + ".proj_out.weight"].reshape(c, inner))
        self.w[p + ".proj_out.b"] = F(sd[p + ".proj_out.bias"])
        qkv1 = torch.cat([sd[f"{tb}.attn1.to_q.weight"], sd[f"{tb}.attn1.to_k.weight"], sd[f"{tb}.attn1.to_v.weight"]], 0)
        q2 = sd[f"{tb}.attn2.to_q.weight"]
        idx = _geglu_interleave(inner * 4)
        ff1, ff1b = sd[f"{tb}.ff.net.0.proj.weight"][idx], sd[f"{tb}.ff.net.0.proj.bias"][idx]
        if self.ln_fold:
            # LN(x) W^T + b = rstd * (x (W*gamma)^T - mean * g) + (W beta + b)   (attention.py:263-275)
            for name, wt, bt, nrm in (("qkv1", qkv1, None, "norm1"), ("q2", q2, None, "norm2"), ("ff1", ff1, ff1b, "norm3")):
                gam, bet = sd[f"{tb}.{nrm}.weight"].double(), sd[f"{tb}.{nrm}.bias"].double()
                wg = H((wt.double() * gam[None, :]).float())
                self.w[f"{p}.{name}.w"] = wg
                self.w[f"{p}.{name}.g"] = F(wg.double().sum(1).float())     # of the ROUNDED weights: exact cancellation
                c = wt.double() @ bet
                self.w[f"{p}.{name}.b"] = F((c + bt.double() if bt is not None else c).float())
        else:
            self.w[p + ".qkv1.w"], self.w[p + ".q2.w"] = H(qkv1), H(q2)
            self.w[p + ".ff1.w"], self.w[p + ".ff1.b"] = H(ff1), F(ff1b)
        self.w[p + ".o1.w"], self.w[p + ".o1.b"] = H(sd[f"{tb}.attn1.to_out.0.weight"]), F(sd[f"{tb}.attn1.to_out.0.bias"])
        self.w[p + ".kv2.w"] = H(torch.cat([sd[f"{tb}.attn2.to_k.weight"], sd[f"{tb}.attn2.to_v.weight"]], 0))
        self.w[p + ".o2.w"], self.w[p + ".o2.b"] = H(sd[f"{tb}.attn2.to_out.0.weight"]), F(sd[f"{tb}.attn2.to_out.0.bias"])
        self.w[p + ".ff2.w"], self.w[p + ".ff2.b"] = H(sd[f"{tb}.ff.net.2.weight"]), F(sd[f"{tb}.ff.net.2.bias"])
        for n in ("norm1", "norm2", "norm3"):
            self.w[f"{p}.{n}.g"], self.w[f"{p}.{n}.b"] = F(sd[f"{tb}.{n}.weight"]), F(sd[f"{tb}.{n}.bias"])

    def weight_bytes(self):
        return sum(t.numel() * t.element_size() for t in self.w.values())

    # ------------------------------------------------------------------ per-prompt / per-image
    def attn_prefixes(self):
        out = []
        groups = list(self.topo.input_blocks) + [self.topo.middle] + list(self.topo.output_blocks)
        for layers in groups:
            out += [b.prefix for b in layers if b.kind == "attn"]
        return out

    def precompute_context(self, ctx):
        """Cross-attention K/V depend only on the prompt: project them once per request
        (attention.py:168-169 recomputes them every step)."""
        B, Lc, D = ctx.shape
        ctx2 = ctx.to(self.hdt).reshape(B * Lc, D).contiguous()
        kv = {}
        for p in self.attn_prefixes():
            kv[p] = self.ops.gemm(ctx2, self.w[p + ".kv2.w"])  # [B*L, 2*inner]
        return {"kv": kv, "B": B, "L": Lc}

    def precompute_hint(self, hint_nchw):
        """ControlNet.input_hint_block (cldm/cldm.py:147-163): independent of x and t, so hoisted
        out of the denoising loop (the reference recomputes it every step, cldm/cldm.py:288)."""
        o = self.ops
        B, C, Hh, Wh = hint_nchw.shape
        x = hint_nchw.permute(0, 2, 3, 1).contiguous().to(self.hdt)
        n = len(HINT_STRIDES)
        tc = os.environ.get("EA_HINT_TC", "1") != "0" and Hh % 8 == 0 and Wh % 8 == 0
        cin = C
        for i, s in enumerate(HINT_STRIDES):
            p = f"input_hint_block.{2 * i}"
            cout = self.w[p + ".w"].shape[-1]
            Ho, Wo = (Hh + s - 1) // s, (Wh + s - 1) // s
            if not tc:
                y = torch.empty(B, Ho, Wo, cout, device=self.dev, dtype=self.hdt)
                o.conv_direct(x, self.w[p + ".w"], self.w[p + ".b"], y, B=B, Hin=Hh, Win=Wh, Cin=cin, Cout=cout,
                              ksize=3, stride=s, silu=(i != n - 1))
            elif i == 0:
                # first layer (3 input channels, un-normalised 0..255 id map: fp32 weights) on the direct kernel,
                # written into a buffer whose channels are padded to 64 for the tensor-core layers that follow
                cp = -(-cout // 64) * 64
                y = torch.zeros(B, Ho, Wo, cp, device=self.dev, dtype=self.hdt)
                o.conv_direct(x, self.w[p + ".w"], self.w[p + ".b"], y, B=B, Hin=Hh, Win=Wh, Cin=cin, Cout=cout,
                              ksize=3, stride=s, silu=True, ldo=cp)
            else:
                # layers 2..8 as implicit-GEMM convolutions on the tensor cores (1.5 GFLOP per image on CUDA cores
                # cost several ms per request; padded to 64-channel multiples they are ~64 GFLOP of tensor-core work)
                wp = self.w[p + ".wp"]
                y = torch.empty(B, Ho, Wo, wp.shape[0], device=self.dev, dtype=self.hdt)
                o.gemm(x, wp, y.view(B * Ho * Wo, -1), mode=L.EA_GEMM_CONV_S1 if s == 1 else L.EA_GEMM_CONV_S2,
                       conv=(B, Ho, Wo, x.shape[-1]), bias=self.w[p + ".bp"],
                       act=L.EA_ACT_SILU if i != n - 1 else L.EA_ACT_NONE)
            x, cin, Hh, Wh = y, cout, Ho, Wo
        return x

    def precompute_condition(self, c_nhwc):
        """conv(c, W_c) + b of a 9-channel UNet's conv_in for c = [mask, masked-image latents, 0, 0, 0] (NHWC, 8
        channels): constant over the denoising loop (utils/...inpaint.py:1550-1558 concatenates the same mask and
        masked-image latents every step), so it is computed once per request and added to the per-step conv_in."""
        B, H, W_, C = c_nhwc.shape
        if self.x_channels == self.cfg.in_channels or C != 8:
            raise ValueError(f"precompute_condition needs a 9-channel UNet and an 8-channel input, got {C} channels "
                             f"for in_channels={self.cfg.in_channels}")
        p = self.topo.input_blocks[0][0].prefix
        cout = self.cfg.model_channels
        out = self._new(B, H, W_, cout)
        self.ops.conv_in(c_nhwc.to(self.hdt).contiguous(), self.w[p + ".wc"], self.w[p + ".b"], out, B=B, H=H, W=W_,
                         Cin=8, Cout=cout)
        return out

    # ------------------------------------------------------------------ execution
    def _emb(self, t_dev, B):
        o = self.ops
        mc = self.cfg.model_channels
        te = torch.empty(B, mc, device=self.dev, dtype=torch.float32)
        o.timestep_embedding(t_dev, te, B=B, dim=mc)
        e1 = torch.empty(B, 4 * mc, device=self.dev, dtype=torch.float32)
        o.small_linear(te, self.w["te0.w"], self.w["te0.b"], e1, M=B, N=4 * mc, K=mc, silu_out=True)
        # emb = te2(e1); every consumer applies SiLU first (openaimodel.py:204-205) -> silu_out here
        e2 = torch.empty(B, 4 * mc, device=self.dev, dtype=torch.float32)
        o.small_linear(e1, self.w["te2.w"], self.w["te2.b"], e2, M=B, N=4 * mc, K=4 * mc, silu_out=True)
        ea = torch.empty(B, self.emb_total, device=self.dev, dtype=torch.float32)
        o.small_linear(e2, self.w["emb.w"], self.w["emb.b"], ea, M=B, N=self.emb_total, K=4 * mc)
        return ea

    def _new(self, *shape):
        return torch.empty(*shape, device=self.dev, dtype=self.hdt)


class BlockRunner:
    """Executes ResBlocks / SpatialTransformers / resampling convolutions for ONE network or for n networks of
    the same topology in lockstep (the UNet encoder and the ControlNets: cldm/cldm.py:22-45 vs 284-305 - the same
    layers, different weights, the same latent).  In lockstep the activations are stacked along the batch dimension
    ([n*B, H, W, C], network g = images [g*B, (g+1)*B)), every GEMM is ONE grouped launch (ea_gemm_grouped: group
    g = network g's weights on its slice), GroupNorm takes one (gamma, beta) per network, attention simply sees
    n*B batch entries.  `out2` (the UNet's skip-concat dual store) applies to network 0 only."""

    def __init__(self, nets):
        self.nets, self.n = list(nets), len(nets)
        n0 = self.nets[0]
        self.cfg, self.dev, self.hdt, self.ln_fold = n0.cfg, n0.dev, n0.hdt, n0.ln_fold
        self.emb_off = n0.emb_off

    @property
    def ops(self):
        # looked up at every use: a runner lives as long as its networks, whose operator table a caller may swap
        return self.nets[0].ops

    def _new(self, *shape):
        return torch.empty(*shape, device=self.dev, dtype=self.hdt)

    def _chunk(self, t, g):
        return t if self.n == 1 else t.chunk(self.n, 0)[g]

    def gemm(self, a, wkey, out=None, *, bias=None, rowvec=None, residual=None, out2=None, conv=None,
             rowstats_out=None, ln=None, a_extra=None, M=None, **kw):
        """bias / ln[1]: weight-dict keys; rowvec: one tensor per network; rowstats_out / ln[0]: [n, C/32, M, 2]."""
        n, nets = self.n, self.nets
        if n == 1:
            w = nets[0].w
            return self.ops.gemm(a, w[wkey], out, bias=w[bias] if bias else None,
                                 rowvec=rowvec[0] if rowvec is not None else None, residual=residual, out2=out2,
                                 conv=conv, rowstats_out=rowstats_out[0] if rowstats_out is not None else None,
                                 ln=(ln[0][0], w[ln[1]], ln[2]) if ln is not None else None, a_extra=a_extra, M=M, **kw)
        w0 = nets[0].w[wkey]
        if out is None:
            rows = conv[0] * conv[1] * conv[2] if conv is not None else a.shape[0]
            out = self._new(rows, w0.shape[0] // 2 if kw.get("act") == L.EA_ACT_GEGLU else w0.shape[0])
        calls = []
        for g in range(n):
            w = nets[g].w
            kwg = dict(kw)
            kwg["bias"] = w[bias] if bias else None
            if rowvec is not None:
                kwg["rowvec"] = rowvec[g]
            if residual is not None:
                kwg["residual"] = self._chunk(residual, g)
            if out2 is not None and g == 0:
                kwg["out2"] = out2
            else:
                kwg.pop("ldo2", None)
            if conv is not None:
                kwg["conv"] = (conv[0] // n,) + tuple(conv[1:])
            if rowstats_out is not None:
                kwg["rowstats_out"] = rowstats_out[g]
            if ln is not None:
                kwg["ln"] = (ln[0][g], w[ln[1]], ln[2])
            if a_extra is not None:
                kwg["a_extra"] = self._chunk(a_extra, g)
            if M is not None:
                kwg["M"] = M // n
            calls.append((self._chunk(a, g), w[wkey], self._chunk(out, g), kwg))
        self.ops.gemm_grouped(calls)
        return out

    def groupnorm(self, x, key, out, **kw):
        if self.n == 1:
            w = self.nets[0].w
            return self.ops.groupnorm(x, w[key + ".g"], w[key + ".b"], out, **kw)
        return self.ops.groupnorm(x, [nt.w[key + ".g"] for nt in self.nets], [nt.w[key + ".b"] for nt in self.nets],
                                  out, **kw)

    def _res(self, blk, x, embs, gn_ws, out=None, out2=None):
        """x: NHWC view [B,H,W,cin] (may be a concat buffer).  Returns [B,H,W,cout].  embs: one [B, emb_total]
        row-vector table per network."""
        p = blk.prefix
        B, H, W_, cin = x.shape
        cout = blk.cout
        a1 = self._new(B, H, W_, cin)
        self.groupnorm(x, p + ".in_layers.0", a1, B=B, HW=H * W_, C_=cin, eps=1e-5, silu=True, workspace=gn_ws,
                       ldx=x.stride(2))
        h1 = self._new(B, H, W_, cout)
        off = self.emb_off[p]
        self.gemm(a1, p + ".conv1.w", h1, mode=L.EA_GEMM_CONV_S1, conv=(B, H, W_, cin),
                  rowvec=[e[:, off:off + cout] for e in embs])
        a2 = self._new(B, H, W_, cout)
        self.groupnorm(h1, p + ".out_layers.0", a2, B=B, HW=H * W_, C_=cout, eps=1e-5, silu=True, workspace=gn_ws)
        if out is None:
            out = self._new(B, H, W_, cout)
        if cin != cout:
            self.gemm(a2, p + ".conv2.w", out, mode=L.EA_GEMM_CONV_S1, conv=(B, H, W_, cout), a_extra=x,
                      ld_extra=x.stride(2), bias=p + ".conv2.b", out2=out2)
        else:
            self.gemm(a2, p + ".conv2.w", out, mode=L.EA_GEMM_CONV_S1, conv=(B, H, W_, cout),
                      bias=p + ".conv2.b", residual=x, out2=out2)
        return out

    def _attn(self, blk, x, ctxc, gn_ws, out=None, out2=None):
        o, p, n = self.ops, blk.prefix, self.n
        B, H, W_, c = x.shape
        heads, dh = self.cfg.heads_for(c)
        inner = heads * dh
        N, M = H * W_, B * H * W_
        xn = self._new(B, H, W_, c)
        self.groupnorm(x, p + ".norm", xn, B=B, HW=N, C_=c, eps=1e-6, silu=False, workspace=gn_ws, ldx=x.stride(2))
        fold = self.ln_fold

        def stats():   # per-row partial (sum, sumsq) per 32-column chunk, written by the producing GEMM
            return torch.empty(n, inner // 32, M // n, 2, device=self.dev, dtype=torch.float32) if fold else None

        def normed(t, st, name, nrm, **kw):   # GEMM on LayerNorm(t): folded, or LayerNorm launch + plain GEMM
            if fold:
                return self.gemm(t, f"{p}.{name}.w", bias=f"{p}.{name}.b", ln=(st, f"{p}.{name}.g", 1e-5), **kw)
            w = self.nets[0].w                 # (lockstep needs the fold: UNetRunner checks)
            nn_ = self._new(M, inner)
            o.layernorm(t, w[f"{p}.{nrm}.g"], w[f"{p}.{nrm}.b"], nn_, M=M, C_=inner)
            return self.gemm(nn_, f"{p}.{name}.w", bias=f"{p}.{name}.b" if f"{p}.{name}.b" in w else None, **kw)

        st0, st1, st2 = stats(), stats(), stats()
        t0 = self.gemm(xn.view(M, c), p + ".proj_in.w", bias=p + ".proj_in.b", rowstats_out=st0)
        qkv = normed(t0, st0, "qkv1", "norm1")                  # [M, 3*inner]
        ao = self._new(M, inner)
        o.attention(qkv, qkv[:, inner:], qkv[:, 2 * inner:], ao, B=B, heads=heads, Nq=N, Nkv=N, d=dh,
                    q_strides=(N * 3 * inner, 3 * inner), k_strides=(N * 3 * inner, 3 * inner),
                    v_strides=(N * 3 * inner, 3 * inner), o_strides=(N * inner, inner), scale=dh ** -0.5)
        t1 = self.gemm(ao, p + ".o1.w", bias=p + ".o1.b", residual=t0, rowstats_out=st1)
        q2 = normed(t1, st1, "q2", "norm2")
        kv = ctxc["kv"][p]                                       # [B*L, 2*inner] (stacked like x in lockstep)
        Lc = ctxc["L"]
        ao2 = self._new(M, inner)
        o.attention(q2, kv, kv[:, inner:], ao2, B=B, heads=heads, Nq=N, Nkv=Lc, d=dh,
                    q_strides=(N * inner, inner), k_strides=(Lc * 2 * inner, 2 * inner),
                    v_strides=(Lc * 2 * inner, 2 * inner), o_strides=(N * inner, inner), scale=dh ** -0.5)
        t2 = self.gemm(ao2, p + ".o2.w", bias=p + ".o2.b", residual=t1, rowstats_out=st2)
        g = normed(t2, st2, "ff1", "norm3", act=L.EA_ACT_GEGLU)   # [M, 4*inner]
        t3 = self.gemm(g, p + ".ff2.w", bias=p + ".ff2.b", residual=t2)
        if out is None:
            out = self._new(B, H, W_, c)
        self.gemm(t3, p + ".proj_out.w", out.view(M, -1) if out.is_contiguous() else out, M=M, bias=p + ".proj_out.b",
                  residual=x, ldr=x.stride(2), ldo=out.stride(2), out2=out2,
                  ldo2=(out2.stride(2) if out2 is not None else None))
        return out

    def _run_layers(self, layers, h, embs, ctxc, gn_ws, final_out=None, final_out2=None):
        """Run one TimestepEmbedSequential; the LAST operator writes to final_out / final_out2."""
        o = self.ops
        for i, blk in enumerate(layers):
            last = i == len(layers) - 1
            fo = final_out if last else None
            fo2 = final_out2 if last else None
            B, H, W_, _ = h.shape
            if blk.kind == "res":
                h = self._res(blk, h, embs, gn_ws, out=fo, out2=fo2)
            elif blk.kind == "attn":
                h = self._attn(blk, h, ctxc, gn_ws, out=fo, out2=fo2)
            elif blk.kind == "down":
                out = fo if fo is not None else self._new(B, H // 2, W_ // 2, blk.cout)
                self.gemm(h, blk.prefix + ".w", out, mode=L.EA_GEMM_CONV_S2, conv=(B, H // 2, W_ // 2, blk.cin),
                          bias=blk.prefix + ".b", out2=fo2)
                h = out
            elif blk.kind == "up":
                up = self._new(B, 2 * H, 2 * W_, blk.cin)
                o.upsample2x(h, up, B=B, H=H, W=W_, C_=blk.cin)
                out = fo if fo is not None else self._new(B, 2 * H, 2 * W_, blk.cout)
                self.gemm(up, blk.prefix + ".w", out, mode=L.EA_GEMM_CONV_S1, conv=(B, 2 * H, 2 * W_, blk.cin),
                          bias=blk.prefix + ".b", out2=fo2)
                h = out
            else:
                raise ValueError(blk.kind)
        return h


class UNetRunner:
    """One denoising-step network: UNet + k ControlNets sharing skip-concat buffers."""

    def __init__(self, unet: PackedNet, controlnets, device):
        self.unet, self.cns, self.dev = unet, list(controlnets), device
        self.ops = unet.ops
        self.hdt = unet.hdt
        self.concurrent = os.environ.get("EA_CONCURRENT", "1") != "0"
        self._streams = []
        self._gn_ws = {}
        # Lockstep: the UNet encoder and the ControlNets as ONE sequence of grouped launches (BlockRunner) instead of
        # one stream per network.  Needs identical topologies (conv_in, run per network, may differ in its input
        # channels), the LayerNorm fold and at most 3 networks (ea_gemm_grouped); EA_LOCKSTEP=0 falls back to the
        # concurrent streams (A/B).
        nets = [unet] + self.cns
        same = replace(unet.cfg, in_channels=0)
        self.lockstep = (os.environ.get("EA_LOCKSTEP", "1") != "0" and 2 <= len(nets) <= 3 and unet.ln_fold
                         and all(replace(n.cfg, in_channels=0) == same and n.ln_fold for n in nets))
        self.solo = [BlockRunner([n]) for n in nets]      # the UNet, then each ControlNet, on its own
        self.group = BlockRunner(nets) if self.lockstep else None

    def _workspaces(self, B, n):
        """n zeroed GroupNorm workspaces for batch B (one per concurrent stream), allocated once."""
        key = (B, n)
        if key not in self._gn_ws:
            self._gn_ws[key] = [self.ops.gn_workspace(B, self.dev) for _ in range(n)]
        return self._gn_ws[key]

    def _encoder(self, R: BlockRunner, x_half, embs, ctxc, gn_ws, sinks, hints, scales, cond_in=None, deferred=None):
        """input_blocks + middle of the networks of R (the UNet, if there, first), stacked along the batch.  embs,
        hints, scales: one per network of R (hint and scale None for the UNet).  The UNet's skips are dual-stored into
        the decoder's concat slots; each ControlNet's zero-conv then accumulates `scale * zero_conv(h)` into the same
        slot instead of materialising the residual (cldm/cldm.py:34-41,293-303), at once or, given `deferred`, later
        by the caller.  cond_in: a 9-channel UNet's conv_in contribution of the condition channels, bias included
        (PackedNet.precompute_condition)."""
        n, nets = R.n, R.nets
        has_unet = nets[0].kind == "unet"
        topo = nets[0].topo
        B, H, W_, _ = x_half.shape
        h = None
        for i, layers in enumerate(topo.input_blocks):
            slot = sinks["skip"][i]
            if layers[0].kind == "conv_in":
                p, cout = layers[0].prefix, layers[0].cout
                h = R._new(n * B, H, W_, cout)
                for g, nt in enumerate(nets):
                    un = nt.kind == "unet"
                    R.ops.conv_in(x_half, nt.w[p + ".w"], None if un and cond_in is not None else nt.w[p + ".b"],
                                  h.chunk(n, 0)[g], B=B, H=H, W=W_, Cin=nt.x_channels, Cout=cout,
                                  out2=slot if un else None, ldo2=slot.stride(2) if un else 0,
                                  add=cond_in if un else hints[g])
            else:
                h = R._run_layers(layers, h, embs, ctxc, gn_ws, final_out2=slot if has_unet else None)
            self._zero_convs(R, h, i, slot, scales, deferred)
        # the UNet on its own writes the middle output straight into the decoder's first concat; stacked with
        # ControlNets, its slice of the stacked output is dual-stored there
        mid = sinks["mid"]
        h = R._run_layers(topo.middle, h, embs, ctxc, gn_ws, final_out=mid if has_unet and n == 1 else None,
                          final_out2=mid if has_unet and n > 1 else None)
        self._zero_convs(R, h, None, mid, scales, deferred)
        return h

    def _zero_convs(self, R, h, i, slot, scales, deferred):
        """slot += scale * zero_conv_i(h) for every ControlNet of R (i = None: middle_block_out), or the same GEMMs
        appended to `deferred` as (a, w, out, kwargs)."""
        c = h.shape[-1]
        M = h.shape[0] // R.n * h.shape[1] * h.shape[2]
        p = "mid_out" if i is None else f"zero_convs.{i}.0"
        for g, nt in enumerate(R.nets):
            if nt.kind == "unet":
                continue
            f, rs = self.zc_scale(scales[g], i, h.shape)
            call = (h.chunk(R.n, 0)[g].reshape(M, c), nt.w[p + ".w"], slot,
                    dict(M=M, bias=nt.w[p + ".b"], out_scale=f, row_scale=rs, accumulate=True, ldo=slot.stride(2)))
            if deferred is not None:
                deferred.append(call)
            else:
                R.ops.gemm(*call[:3], **call[3])

    @staticmethod
    def zc_scale(scale, i, shape):
        """(out_scale, row_scale) of zero-conv i (0..11 = down residuals, None = mid) for one net's conditioning
        scale: a float, or the dict DenoiseEngine.prepare builds for guess mode (per-residual logspace factors) and
        spatial maps (utils/stable_diffusion_controlnet.py:777-802)."""
        if not isinstance(scale, dict):
            return float(scale), None
        f = scale["base"]
        if scale.get("per_res") is not None:
            f *= scale["per_res"][-1 if i is None else i]
        rs = None
        if scale.get("maps") is not None:
            rs = scale["maps"][(shape[1], shape[2])]
        return f, rs

    def precompute_context_lockstep(self, ctx):
        """Cross-attention K/V of the encoder + middle attention layers of every network, stacked along the batch
        like the lockstep activations: kv[p] = [n * B * L, 2 * inner] (network g = rows [g*B*L, (g+1)*B*L))."""
        nets = [self.unet] + self.cns
        n = len(nets)
        B, Lc, D = ctx.shape
        ctx2 = ctx.to(self.hdt).reshape(B * Lc, D).contiguous()
        topo = self.unet.topo
        kv = {}
        for layers in list(topo.input_blocks) + [topo.middle]:
            for b in layers:
                if b.kind == "attn":
                    p = b.prefix
                    out = torch.empty(n * B * Lc, self.unet.w[p + ".kv2.w"].shape[0], device=self.dev, dtype=self.hdt)
                    self.ops.gemm_grouped([(ctx2, nt.w[p + ".kv2.w"], out.chunk(n, 0)[g], {}) for g, nt in enumerate(nets)])
                    kv[p] = out
        return {"kv": kv, "B": n * B, "L": Lc}

    def alloc_sinks(self, B, H, W_):
        """Skip-concat buffers of the decoder: cat_i = [h (C1) | skip_i + control_i (C2)]."""
        topo = self.unet.topo
        chans = list(topo.input_chans)
        sizes = []  # spatial size of each skip
        hh, ww = H, W_
        for layers in topo.input_blocks:
            if layers[0].kind == "down":
                hh, ww = hh // 2, ww // 2
            sizes.append((hh, ww))
        cats, skip_slots = [], [None] * len(chans)
        for oi, layers in enumerate(topo.output_blocks):
            si = len(chans) - 1 - oi
            c2 = chans[si]
            c1 = layers[0].cin - c2
            sh, sw = sizes[si]
            cat = torch.empty(B, sh, sw, c1 + c2, device=self.dev, dtype=self.hdt)
            cats.append((cat, c1))
            skip_slots[si] = cat[..., c1:]
        mh, mw = sizes[-1]
        mid = cats[0][0][..., :cats[0][1]]  # mid output IS the h-part of the first decoder concat
        return {"cats": cats, "skip": skip_slots, "mid": mid}

    def compute_embs(self, t_dev, B):
        """Per-ResBlock time-embedding projections of every net for timestep(s) t_dev: a list of
        [B, emb_total] fp32 tensors (UNet first).  They depend on t only, so the engine caches them
        per timestep instead of re-streaming ~93 MB of embedding weights every step."""
        return [n._emb(t_dev, B) for n in [self.unet] + self.cns]

    def eps_features(self, x_half, t_dev, ctx_cache, hints, scales, gn_ws=None, embs=None, ctx_ls=None, cond_in=None):
        """Runs UNet encoder, ControlNets, UNet decoder; returns the GroupNorm+SiLU'd input of the
        final convolution [B,H,W,mc] (the out conv itself is fused with CFG/DDIM).  x_half holds the 4 latent
        channels; a 9-channel UNet also needs cond_in [B,H,W,mc] (PackedNet.precompute_condition)."""
        un = self.unet
        o = self.ops
        B, H, W_, _ = x_half.shape
        if (un.x_channels != un.cfg.in_channels) != (cond_in is not None):
            raise ValueError(f"cond_in is required by a {un.cfg.in_channels}-channel UNet exactly when it reads "
                             "condition channels")
        if cond_in is not None and tuple(cond_in.shape) != (B, H, W_, un.cfg.model_channels):
            raise ValueError(f"cond_in {tuple(cond_in.shape)} does not match the latents {(B, H, W_)}")
        if gn_ws is None:
            gn_ws = o.gn_workspace(B, self.dev)
        sinks = self.alloc_sinks(B, H, W_)
        if embs is None:
            embs = self.compute_embs(t_dev, B)
        n = 1 + len(self.cns)
        hints, scales = [None] + list(hints), [None] + list(scales)     # one per network, UNet first
        if self.lockstep and ctx_ls is not None:
            o.set_lane(0, False)
            self._encoder(self.group, x_half, embs, ctx_ls, self._workspaces(n * B, 1)[0], sinks, hints, scales,
                          cond_in)
        elif self.concurrent and n > 1 and x_half.is_cuda:
            # The UNet encoder and every ControlNet only READ x and write their own activations: run
            # them on parallel streams (many of their launches cannot fill 132 SMs on their own), join,
            # then apply the zero-conv accumulations into the shared skip slots on the main stream.
            # Inside the concurrent region GroupNorm / split-K use their variants without inter-CTA
            # waits, and each stream has its own scratch lane.
            main = torch.cuda.current_stream()
            if len(self._streams) < len(self.cns):
                self._streams = [torch.cuda.Stream() for _ in self.cns]
            lanes_ws = self._workspaces(B, n)
            deferred = []
            for s in self._streams:
                s.wait_stream(main)
            o.set_lane(0, True)
            self._encoder(self.solo[0], x_half, embs[:1], ctx_cache[0], lanes_ws[0], sinks, hints[:1], scales[:1],
                          cond_in)
            for g in range(1, n):
                with torch.cuda.stream(self._streams[g - 1]):
                    o.set_lane(g, True)
                    self._encoder(self.solo[g], x_half, embs[g:g + 1], ctx_cache[g], lanes_ws[g], sinks,
                                  hints[g:g + 1], scales[g:g + 1], deferred=deferred)
            for s in self._streams:
                main.wait_stream(s)
            o.set_lane(0, False)
            for a_, w_, out_, kw_ in deferred:
                o.gemm(a_, w_, out_, **kw_)
        else:
            for g, R in enumerate(self.solo):
                self._encoder(R, x_half, embs[g:g + 1], ctx_cache[g], gn_ws, sinks, hints[g:g + 1], scales[g:g + 1],
                              cond_in)
        topo = un.topo
        cats = sinks["cats"]
        h = None
        for oi, layers in enumerate(topo.output_blocks):
            cat, c1 = cats[oi]
            if oi + 1 < len(cats):
                nxt, n1 = cats[oi + 1]
                dst = nxt[..., :n1]
            else:
                dst = None
            h = self.solo[0]._run_layers(layers, cat, embs[:1], ctx_cache[0], gn_ws, final_out=dst)
        mc = un.cfg.model_channels
        xn = un._new(B, H, W_, mc)
        o.groupnorm(h, un.w["out.g"], un.w["out.b"], xn, B=B, HW=H * W_, C_=mc, eps=1e-5, silu=True,
                    workspace=gn_ws, ldx=h.stride(2))
        return xn
