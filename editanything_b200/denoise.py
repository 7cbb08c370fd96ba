"""The per-step engine: ControlNet(s) -> UNet -> CFG -> DDIM on the H100 kernels.

This is the seam SURVEY.md §8b calls B3: what
utils/stable_diffusion_controlnet_inpaint.py:1607-1636 does with `self.controlnet(...)`,
`self.unet(...)`, the guidance combine and `scheduler.step(...)`, as ONE stream-ordered sequence
of libea_b200 launches (optionally replayed as a CUDA graph).
"""
import math
import os

import numpy as np
import torch

from ._backend import default_ops, engine_call
from .nets import PackedNet, UNetRunner
from .unet_spec import UNetConfig, controlnet_config


def ddim_schedule(num_steps, linear_start=0.00085, linear_end=0.012, T=1000):
    """DDIM 'uniform' schedule of the reference sampler: betas (util.py:21-25, cldm_v21.yaml:4-5),
    alphas_cumprod (ddpm.py:145-147), timesteps range(0,T,T//S)+1 (util.py:46-60), a_prev
    (util.py:63-74).  Returned in SAMPLING order (descending t).  S=30 yields 31 steps like the
    reference (1000//30 = 33)."""
    betas = np.linspace(linear_start ** 0.5, linear_end ** 0.5, T, dtype=np.float64) ** 2
    ac = np.cumprod(1.0 - betas, axis=0)
    ts = np.asarray(list(range(0, T, T // num_steps))) + 1
    a = ac[ts]
    a_prev = np.asarray([ac[0]] + ac[ts[:-1]].tolist())
    return ts[::-1].copy(), a[::-1].copy(), a_prev[::-1].copy()


def _fits(old, new):
    """Whether `new` can be copied into `old`: the same nesting of lists / dicts, equal plain values, and tensors of
    the same shape and dtype."""
    if torch.is_tensor(new):
        return torch.is_tensor(old) and old.shape == new.shape and old.dtype == new.dtype
    if isinstance(new, list):
        return isinstance(old, list) and len(old) == len(new) and all(map(_fits, old, new))
    if isinstance(new, dict):
        return isinstance(old, dict) and old.keys() == new.keys() and all(_fits(old[k], new[k]) for k in new)
    return not torch.is_tensor(old) and old == new


def _copy_into(old, new):
    if torch.is_tensor(new):
        old.copy_(new)
    elif isinstance(new, (list, dict)):
        for k in (new if isinstance(new, dict) else range(len(new))):
            _copy_into(old[k], new[k])


class DenoiseEngine:
    def __init__(self, cfg: UNetConfig, unet_sd, controlnet_sds, device, backend=None, unet_packed=None):
        """unet_packed: an already packed UNet (another engine's `.unet`) to share instead of packing `unet_sd`
        again - the reference's tile pipeline runs the same base model as the main one (editany_lora.py:395-405)."""
        if cfg.in_channels not in (4, 9):
            raise ValueError(f"the UNet takes 4 latent channels, or 9 (latents, mask, masked-image latents) for an "
                             f"inpainting base model; got in_channels={cfg.in_channels}")
        self.cfg, self.dev = cfg, device
        self.ops = backend or default_ops()
        self.unet = unet_packed if unet_packed is not None else PackedNet(cfg, "unet", unet_sd, device, backend)
        self.cns = [PackedNet(controlnet_config(cfg), "controlnet", sd, device, backend) for sd in controlnet_sds]
        self.runner = UNetRunner(self.unet, self.cns, device)
        self.hdt = self.unet.hdt
        self._graph = None
        self.launches_per_step = None

    def weight_bytes(self):
        return self.unet.weight_bytes() + sum(c.weight_bytes() for c in self.cns)

    # -- per request -------------------------------------------------------------------------
    def _keep(self, name, new):
        """Store `new` (a tensor, or a list / dict of tensors and plain values) under self.<name>, copying it into the
        existing buffers (same addresses => a captured CUDA graph stays valid) when the structure, plain values and
        every tensor's shape / dtype match; otherwise adopt it and invalidate the graph."""
        old = getattr(self, name, None)
        if _fits(old, new):
            _copy_into(old, new)
            new = old
        else:
            self._graph = None
            if torch.is_tensor(new) and new.is_inference():
                new = new.clone()     # a caller under torch.inference_mode(): persistent buffers must be normal tensors
        setattr(self, name, new)
        return new

    def _norm_scale(self, s, guess_mode, B, lat_hw):
        """One net's conditioning scale in the form nets.UNetRunner.zc_scale reads: a plain float, or - for guess mode
        / a spatial map (ControlNetModel2.forward, utils/stable_diffusion_controlnet.py:777-802) - a dict with the 13
        logspace(-1, 0, 13) per-residual factors and / or the map resized (bilinear, align_corners=True) to every
        residual resolution, flattened to one factor per output row [B * h * w]."""
        if not guess_mode and not torch.is_tensor(s):
            return float(s)
        out = {"base": 1.0 if torch.is_tensor(s) else float(s), "per_res": None, "maps": None}
        if guess_mode:
            if torch.is_tensor(s):
                raise NotImplementedError("guess_mode with a spatial conditioning_scale map")
            out["per_res"] = [float(v) for v in torch.logspace(-1, 0, len(self.unet.topo.input_chans) + 1)]
        if torch.is_tensor(s):
            m = s.to(self.dev, torch.float32)
            m = m[None, None] if m.dim() == 2 else m[None] if m.dim() == 3 else m
            maps = {}
            h, w = lat_hw
            for _ in range(len(self.cfg.channel_mult)):
                r = torch.nn.functional.interpolate(m, (h, w), mode="bilinear", align_corners=True)
                maps[(h, w)] = r.expand(B, 1, h, w).reshape(-1).contiguous()
                h, w = h // 2, w // 2
            out["maps"] = maps
        return out

    @engine_call
    def prepare(self, ctx, hints, scales, guess_mode=False, cfg_duplicated=False):
        """ctx: [B, L, D] prompt embeddings ([negative; positive] stacked for CFG,
        utils/stable_diffusion_controlnet_inpaint.py:1339-1347); hints: list of NCHW conditioning
        images [B, 3, 8h, 8w] (un-normalised, editany_lora.py:771-778,814-828); scales: list."""
        ctx = ctx.to(self.dev)
        self.B = ctx.shape[0]
        nets = [self.unet] + self.cns
        # lockstep (nets.UNetRunner): the encoder-side K/V of all networks live stacked in ctx_ls; only the UNet
        # (whose decoder runs alone) keeps its own per-layer cache
        ls = self.runner.lockstep
        self._keep("ctx_cache", [n.precompute_context(ctx) for n in (nets[:1] if ls else nets)])
        self._keep("ctx_ls", self.runner.precompute_context_lockstep(ctx) if ls else None)
        # cfg_duplicated: the conditioning images are [x; x] (prepare_controlnet_conditioning_image doubles them for
        # classifier-free guidance, utils/...inpaint.py:380-381) - run the hint stack on one half only
        if cfg_duplicated and all(h.shape[0] % 2 == 0 for h in hints):
            new_hints = []
            for c, h in zip(self.cns, hints):
                g = c.precompute_hint(h[:h.shape[0] // 2].to(self.dev))
                new_hints.append(torch.cat([g, g]))
        else:
            new_hints = [c.precompute_hint(h.to(self.dev)) for c, h in zip(self.cns, hints)]
        self._keep("hints", new_hints)
        lat_hw = (hints[0].shape[-2] // 8, hints[0].shape[-1] // 8) if len(hints) else (0, 0)
        new_scales = [self._norm_scale(s, guess_mode, self.B, lat_hw) for s in scales]
        plain = all(not isinstance(s, dict) for s in new_scales)
        if not plain or getattr(self, "scales", None) != new_scales:
            self._graph = None        # scales (and map addresses) are baked into the zero-conv launches
        self.scales = new_scales
        if not hasattr(self, "t_dev") or self.t_dev.shape[0] != self.B:
            self._emb_cache = {}
            nets = [self.unet] + self.cns
            self.emb_bufs = [torch.zeros(self.B, n.emb_total, device=self.dev, dtype=torch.float32) for n in nets]
            self.t_dev = torch.zeros(self.B, device=self.dev, dtype=torch.float32)
            self.coef_dev = torch.zeros(16, device=self.dev, dtype=torch.float32)
            self.step_ctr = torch.zeros(1, device=self.dev, dtype=torch.int32)
            self.gn_ws = self.ops.gn_workspace(self.B, self.dev)
            self._sched_key, self._sched_cap, self.n_steps = None, 0, 0
            self._graph = None

    def _emb_rows(self, t):
        """Time-embedding rows of every net for timestep t (util.py:154-174 + time_embed + every ResBlock
        emb_layers, openaimodel.py:526-531,204-210): computed once per distinct t and cached - the DDIM table
        repeats for every image."""
        key = float(t)
        rows = self._emb_cache.get(key)
        if rows is None:
            self.t_dev.fill_(key)
            rows = [e.clone() for e in self.runner.compute_embs(self.t_dev, self.B)]
            if len(self._emb_cache) < 1100:
                self._emb_cache[key] = rows
        return rows

    def _fill_emb(self, t):
        for buf, r in zip(self.emb_bufs, self._emb_rows(t)):
            buf.copy_(r)

    def _condition(self, mask_n1hw, masked_latents_nchw):
        """conv_in's contribution of the condition channels of a 9-channel UNet: [B, h, w, mc] (half)."""
        m = mask_n1hw.to(self.dev, torch.float32)
        z = masked_latents_nchw.to(self.dev, torch.float32)
        c = torch.cat([m, z, torch.zeros_like(z[:, :3])], 1).permute(0, 2, 3, 1).contiguous()
        return self.unet.precompute_condition(c)

    @engine_call
    def set_unet_condition(self, mask_n1hw, masked_latents_nchw):
        """The per-request input of a 9-channel (inpainting) UNet: the mask resized to the latents [N, 1, h, w] and
        the VAE latents of the masked image [N, 4, h, w] (utils/...inpaint.py:1448-1468), for the N images.  They
        are the same at every step (:1550-1558), so their part of conv_in, bias included, is computed here once;
        the CFG duplication is done here too.  Each step's conv_in then reads the 4 latent channels only."""
        if self.unet.x_channels == self.cfg.in_channels:
            raise ValueError(f"set_unet_condition needs a 9-channel UNet, this one takes {self.cfg.in_channels}")
        if mask_n1hw.shape[1] != 1 or masked_latents_nchw.shape[1] != 4 or \
                mask_n1hw.shape[0] != masked_latents_nchw.shape[0] or mask_n1hw.shape[2:] != masked_latents_nchw.shape[2:]:
            raise ValueError(f"mask {tuple(mask_n1hw.shape)} / masked-image latents {tuple(masked_latents_nchw.shape)}: "
                             "expected [N, 1, h, w] and [N, 4, h, w]")
        g = self._condition(mask_n1hw, masked_latents_nchw)
        self._keep("cond_in", torch.cat([g, g]))

    # -- the sampling schedule as device tables -------------------------------------------------
    @engine_call
    def set_schedule(self, timesteps, alphas, alphas_prev, blend=None, multistep=None):
        """Everything that changes from step to step of the loop (utils/...inpaint.py:1540-1656), as device
        tables with one row per step: the DDIM coefficients (cldm/ddim_hacked.py:203-231), the per-ResBlock
        time-embedding rows of every net, and the inpaint-blend terms.  `blend` = (k_init[S], k_noise[S],
        on[S]): the kept region of step i is k_init[i] * known + k_noise[i] * noise (add_noise at
        timesteps[i + 1], :1650-1652), applied where on[i] (i < len * alignment_ratio, :1648).  Without `blend`
        the kept region is `known` itself on every step.  The captured step indexes the tables with a device
        counter (ea_step_gather), so the host issues ONE graph launch per step."""
        ts = [float(t) for t in timesteps]
        S = len(ts)
        if blend is None:
            blend = ([1.0] * S, [0.0] * S, [1.0] * S)
        rows = [[math.sqrt(a), math.sqrt(1.0 - a), math.sqrt(ap), math.sqrt(1.0 - ap), float(ki), float(kn), float(on), 0.0]
                + [0.0] * 8 for a, ap, ki, kn, on in zip(alphas, alphas_prev, *blend)]
        if multistep is not None:
            # linear multistep predictor-corrector (UniPC): per-step coefficient rows of
            # schedulers.UniPCMultistepScheduler.coefficient_rows(); mode flag coef[7] = 1
            for r, m in zip(rows, multistep):
                r[0], r[1], r[7] = m["alpha"], m["sigma"], 1.0
                r[8:16] = [m["kx"], m["kl"], m["k1"], m["k2"], m["k0"], m["px"], m["p0"], m["p1"]]
        key = (tuple(ts), tuple(map(tuple, rows)), self.B)
        if key == self._sched_key:
            return
        if S > self._sched_cap:
            cap = ((S + 63) // 64) * 64
            self.coef_tab = torch.zeros(cap, 16, device=self.dev, dtype=torch.float32)
            self.emb_tabs = [torch.zeros(cap, *b.shape, device=self.dev, dtype=torch.float32) for b in self.emb_bufs]
            self._sched_cap = cap
            self._graph = None        # table addresses are baked into the captured step
        self.coef_tab[:S].copy_(torch.tensor(rows, dtype=torch.float32), non_blocking=True)
        for i, t in enumerate(ts):
            for tab, r in zip(self.emb_tabs, self._emb_rows(t)):
                tab[i].copy_(r)
        self.n_steps = S
        self._sched_key = key

    # -- parity API: the network output itself ------------------------------------------------
    @engine_call
    def eps(self, x_nchw, t):
        """eps = unet(x, t, ctx, control=sum_k scale_k * controlnet_k(x, hint_k, t, ctx)) as fp32
        NCHW - the quantity the reference calls `noise_pred` before guidance.  For a 9-channel UNet x is
        cat([latents, mask, masked-image latents]) (utils/...inpaint.py:1550-1558) and the ControlNets see
        x[:, :4] (:1607-1615)."""
        B, C, H, W_ = x_nchw.shape
        if C != self.cfg.in_channels:
            raise ValueError(f"x has {C} channels, the UNet takes {self.cfg.in_channels}")
        cond = None
        if C != self.unet.x_channels:
            cond = self._condition(x_nchw[:, 4:5], x_nchw[:, 5:9])
            x_nchw = x_nchw[:, :4]
        xh = x_nchw.to(self.dev).permute(0, 2, 3, 1).contiguous().to(self.hdt)
        self._fill_emb(t)
        xn = self.runner.eps_features(xh, self.t_dev, self.ctx_cache, self.hints, self.scales, self.gn_ws,
                                      embs=self.emb_bufs, ctx_ls=self.ctx_ls, cond_in=cond)
        eps = torch.empty(B, H, W_, 4, device=self.dev, dtype=torch.float32)
        self.ops.out_cfg_ddim(xn, self.unet.w["out.w"], self.unet.w["out.cb"], eps_out=eps, Nimg=B // 2, H=H,
                              W=W_, C_=self.cfg.model_channels)
        return eps.permute(0, 3, 1, 2).contiguous()

    # -- production API: one fused denoising step ----------------------------------------------
    def _step_body(self):
        H, W_ = self.lat.shape[1], self.lat.shape[2]
        self.ops.step_gather(self.step_ctr, self._sched_cap, [self.coef_tab] + self.emb_tabs,
                             [self.coef_dev] + self.emb_bufs)
        xn = self.runner.eps_features(self.x_half, self.t_dev, self.ctx_cache, self.hints, self.scales, self.gn_ws,
                                      embs=self.emb_bufs, ctx_ls=self.ctx_ls, cond_in=self._step_cond())
        self.ops.out_cfg_ddim(xn, self.unet.w["out.w"], self.unet.w["out.cb"], latents=self.lat,
                              coef=self.coef_dev, guidance=self.guidance, known=self.known, noise=self.noise,
                              mask=self.mask, lat_half_out=self.x_half, step_counter=self.step_ctr, hist=self.hist,
                              Nimg=self.B // 2, H=H, W=W_, C_=self.cfg.model_channels)

    def _step_cond(self):
        if self.unet.x_channels == self.cfg.in_channels:
            return None
        if getattr(self, "cond_in", None) is None:
            raise RuntimeError("a 9-channel UNet needs set_unet_condition() before the first step")
        return self.cond_in

    @engine_call
    def begin(self, latents_nchw, guidance, known_nchw=None, mask_n1hw=None, noise_nchw=None, use_graph=True):
        """latents: fp32 [N, 4, h, w] initial noise (N = B/2 images).  known/mask: optional inpaint blend
        tensors (mask == 1 keeps `known`, utils/...inpaint.py:1484-1489,1647-1664); noise: the initial latent
        noise the kept region is re-noised with (:1446,1650).  The blend buffers always exist (an all-zero mask
        is an exact no-op), so switching the blend on, off or ending its window never re-captures the graph."""
        def nhwc(t):
            return t.to(self.dev, torch.float32).permute(0, 2, 3, 1).contiguous()
        lat = nhwc(latents_nchw)
        self._keep("lat", lat)
        self._keep("x_half", torch.cat([lat, lat]).to(self.hdt).contiguous())
        if getattr(self, "guidance", None) != float(guidance):
            self._graph = None
        self.guidance = float(guidance)
        # (each buffer gets its OWN zeros: _keep adopts the tensor it is given on first use, and known / noise / mask
        # must never alias)
        self._keep("known", nhwc(known_nchw) if known_nchw is not None else torch.zeros_like(lat))
        self._keep("noise", nhwc(noise_nchw) if noise_nchw is not None else torch.zeros_like(lat))
        if known_nchw is not None:
            m = mask_n1hw.to(self.dev, torch.float32).reshape(lat.shape[0], lat.shape[1], lat.shape[2]).contiguous()
        else:
            m = torch.zeros(lat.shape[:3], device=self.dev, dtype=torch.float32)
        self._keep("mask", m)
        # history of the multistep schedulers (x0 predictions of the two previous steps, previous corrected sample)
        self._keep("hist", torch.zeros((3,) + tuple(lat.shape), device=self.dev, dtype=torch.float32))
        use = use_graph and self.dev.type == "cuda"
        if use != getattr(self, "_use_graph", None):
            self._graph = None
        self._use_graph = use
        self.step_ctr.zero_()

    @engine_call
    def end_blend(self):
        """Close the blend window from the host (callers that drive the blend themselves)."""
        self.mask.zero_()

    @engine_call
    def blend_now(self, k_init, k_noise):
        """latents = (k_init * known + k_noise * noise) * mask + latents * (1 - mask), outside the fused step
        (utils/...inpaint.py:1647-1656) - for callers that must observe the un-blended latents first."""
        m = self.mask[..., None]
        self.lat.copy_((k_init * self.known + k_noise * self.noise) * m + self.lat * (1 - m))
        self.x_half.copy_(torch.cat([self.lat, self.lat]).to(self.hdt))

    @engine_call
    def set_known(self, known_nchw):
        self.known.copy_(known_nchw.to(self.dev, torch.float32).permute(0, 2, 3, 1))

    @engine_call
    def step(self, t=None, a_t=None, a_prev=None):
        """One fused step.  Without arguments: step number *step_ctr of the schedule given to set_schedule()
        (host work: one graph launch).  With (t, a_t, a_prev): a single DDIM (eta=0) step at timestep t
        (cldm/ddim_hacked.py:181-231) - a one-row schedule."""
        if t is not None:
            self.set_schedule([t], [a_t], [a_prev])
            self.step_ctr.zero_()
        elif self._sched_key is None:
            raise RuntimeError("set_schedule() first, or pass (t, a_t, a_prev)")
        if not self._use_graph:
            self._step_body()
            return
        if self._graph is None:
            # warm-up on a side stream (allocator + cudaFuncSetAttribute), then capture once
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            lat0, xh0, c0 = self.lat.clone(), self.x_half.clone(), self.step_ctr.clone()
            # opt-in experiment (EA_WEIGHT_PREFETCH = look-ahead distance, default 0 = off): the warm-up pass records
            # the step's GEMM sequence and in the captured pass every launch carries a later launch's weights as an L2
            # prefetch hint (ops.WeightLookahead).  Not measured on H100.
            dist = int(os.environ.get("EA_WEIGHT_PREFETCH", "0"))
            mk = getattr(self.ops, "WeightLookahead", None)
            single = self.runner.lockstep or not self.runner.cns     # launch order = execution order
            la = mk(dist, int(os.environ.get("EA_WEIGHT_PREFETCH_MAXM", "512"))) if (mk is not None and dist > 0 and single) else None
            with torch.cuda.stream(s):
                if la is not None:
                    with self.ops.weight_lookahead(la):
                        self._step_body()
                else:
                    self._step_body()
            torch.cuda.current_stream().wait_stream(s)
            self.lat.copy_(lat0)
            self.x_half.copy_(xh0)
            self.step_ctr.copy_(c0)
            g = torch.cuda.CUDAGraph()
            n0 = self.ops.launch_count()
            with torch.cuda.graph(g):
                if la is not None:
                    with self.ops.weight_lookahead(la.replay()):
                        self._step_body()
                else:
                    self._step_body()
            self.launches_per_step = self.ops.launch_count() - n0
            self._graph = g
            self.lat.copy_(lat0)
            self.x_half.copy_(xh0)
            self.step_ctr.copy_(c0)
        self._graph.replay()

    @engine_call
    def latents(self):
        return self.lat.permute(0, 3, 1, 2).contiguous()
