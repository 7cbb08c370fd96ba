"""Thin torch-tensor wrappers over the C ABI (include/editanything_b200.h).

PyTorch is used here only for device memory and streams; every function below launches
hand-written sm_90a kernels from libea_b200.so on torch's current stream.
"""
import ctypes as C

import torch

from . import _lib as L

_DT = {"float16": torch.float16, "bfloat16": torch.bfloat16}


def half_dtype():
    return _DT[L.load().ea_dtype_name().decode()]


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def launch_count():
    return L.load().ea_launch_count()


def reset_launch_count():
    L.load().ea_reset_launch_count()


_GEMM_WS = {}
GEMM_WS_BYTES = 65536 + 48 * 1024 * 1024
_LANE = [0]          # workspace lane: kernels on concurrently running streams must not share scratch
_CONCURRENT = [False]


def set_lane(lane, concurrent):
    """Select the scratch lane of the calling stream and whether other streams run concurrently
    (then GroupNorm and split-K GEMMs use their variants without inter-CTA waits)."""
    _LANE[0] = lane
    _CONCURRENT[0] = bool(concurrent)


def gemm_workspace(device):
    """Per-device (and per concurrent lane) split-K scratch of ea_gemm (64 KB zeroed counters + fp32
    partial tiles); shared by every GEMM on a stream, allocated once so CUDA-graph captures see a
    stable address."""
    key = (device.type, device.index, _LANE[0])
    ws = _GEMM_WS.get(key)
    if ws is None:
        ws = torch.zeros(GEMM_WS_BYTES, device=device, dtype=torch.uint8)
        _GEMM_WS[key] = ws
    return ws


def _fill_gemm(g, a, w, out=None, *, mode=L.EA_GEMM_LINEAR, M=None, N=None, K=None, lda=None, ldw=0,
               conv=None, a_extra=None, bias=None, rowvec=None, rows_per_batch=0, residual=None,
               out2=None, out_f32=None, act=L.EA_ACT_NONE, out_scale=1.0, accumulate=False,
               ldo=None, ldr=None, ldo2=None, ld_extra=0, force_bn=0, force_splits=0, force_2cta=0,
               force_persistent=0, rowstats_out=None, ln=None, row_scale=None):
    """Fills one ea_gemm_args; returns the output tensor (allocated when the caller gave none)."""
    g.mode = mode
    g.N = N if N is not None else w.shape[0]
    if mode == L.EA_GEMM_LINEAR:
        g.M = M if M is not None else a.shape[0]
        g.K = K if K is not None else a.shape[-1]
        g.lda = lda if lda is not None else a.stride(0)
    else:
        B, H, W_, Cin = conv
        g.M = B * H * W_
        g.K = 0
        g.Bsz, g.H, g.W, g.Cin = B, H, W_, Cin
        g.lda = lda if lda is not None else 0
    g.a = a.data_ptr()
    g.w = w.data_ptr()
    g.ldw = ldw
    if a_extra is not None:
        g.a_extra = a_extra.data_ptr()
        g.Cin_extra = a_extra.shape[-1]
        g.ld_extra = ld_extra
    g.bias = bias.data_ptr() if bias is not None else None
    if rowvec is not None:
        g.rowvec = rowvec.data_ptr()
        g.rowvec_ld = rowvec.stride(0)
    g.rows_per_batch = rows_per_batch
    n_out = g.N // 2 if act == L.EA_ACT_GEGLU else g.N
    if out is None and out_f32 is None:
        out = torch.empty((g.M, n_out), device=a.device, dtype=half_dtype())
    if residual is not None:
        g.residual = residual.data_ptr()
        g.ldr = ldr if ldr is not None else residual.stride(-2)
    if out is not None:
        g.out = out.data_ptr()
        g.ldo = ldo if ldo is not None else out.stride(-2)
    if out2 is not None:
        g.out2 = out2.data_ptr()
        g.ldo2 = ldo2 if ldo2 is not None else out2.stride(-2)
    if out_f32 is not None:
        g.out_f32 = out_f32.data_ptr()
        g.ldo = ldo if ldo is not None else out_f32.stride(-2)
    g.act = act
    g.out_scale = out_scale
    g.accumulate = 1 if accumulate else 0
    g.force_bn = force_bn
    g.force_splits = force_splits
    g.force_2cta = force_2cta
    g.force_persistent = force_persistent
    g.no_spin = 1 if _CONCURRENT[0] else 0
    if row_scale is not None:
        g.row_scale = row_scale.data_ptr()
    if rowstats_out is not None:
        g.rowstats_out = rowstats_out.data_ptr()
    if ln is not None:
        stats, lg, eps = ln
        g.ln_stats, g.ln_g, g.ln_parts, g.ln_eps = stats.data_ptr(), lg.data_ptr(), stats.shape[0], eps
    ws = gemm_workspace(a.device)
    g.workspace = ws.data_ptr()
    g.workspace_bytes = ws.numel()
    return out if out is not None else out_f32


class WeightLookahead:
    """L2 prefetch hints for a REPEATED sequence of GEMM launches (one denoising step): the `record` pass notes every
    launch's weight operands; in the `replay` pass launch i carries the weights of launch i + distance (wrapping to the
    next step's first launches) in ea_gemm_args.prefetch, so HBM streams them into L2 while launch i computes.  The
    step moves 3.16 GB of weights through a 50 MB L2, and HBM idles behind the latency chain of short launches;
    weight-bound layers (8x8 / 16x16 latents, M = 128 / 512) then start from L2."""
    MIN_BYTES = 1 << 20      # smaller operands arrive within the launch's own first wave anyway

    def __init__(self, distance=1, max_m=1 << 30):
        self.distance, self.seq, self.mode, self.idx, self.max_m = distance, [], "record", 0, max_m   # max_m: only for
        # launches with at most that many rows (weight-bound layers)

    def replay(self):
        self.mode, self.idx = "replay", 0
        return self

    def visit(self, gs, ws):
        if self.mode == "record":
            self.seq.append([(w.data_ptr(), w.numel() * w.element_size(), int(g.M)) for g, w in zip(gs, ws)])
            return
        n = len(self.seq)
        if n == 0:
            return
        tgt = [t[:2] for t in self.seq[(self.idx + self.distance) % n] if t[1] >= self.MIN_BYTES and t[2] <= self.max_m]
        self.idx += 1
        slots = [(g, k) for k in range(3) for g in gs]          # spread the ranges over the groups' slots
        for (ptr, nbytes), (g, k) in zip(tgt, slots):
            g.prefetch[k] = ptr
            g.prefetch_bytes[k] = nbytes


_LOOKAHEAD = [None]


class weight_lookahead:
    """with ops.weight_lookahead(la): every gemm / gemm_grouped call inside visits `la` (None = off)."""

    def __init__(self, la):
        self.la = la

    def __enter__(self):
        self.prev, _LOOKAHEAD[0] = _LOOKAHEAD[0], self.la
        return self.la

    def __exit__(self, *exc):
        _LOOKAHEAD[0] = self.prev
        return False


def gemm(a, w, out=None, **kw):
    """out = epilogue(A @ W^T).  conv = (B, H, W, Cin) output-space geometry for CONV modes.
    rowstats_out: fp32 [N/32, M, 2] per row and 32-column chunk of the stored (half) values: (sum, sum of squared
    deviations from the chunk mean sum / 32) (LayerNorm fold, producer);
    ln = (stats [K/32, M, 2], g [N], eps): the consumer side - `w` is W*gamma, `bias` is W beta + b."""
    lib = L.lib()
    g = L.GemmArgs()
    res = _fill_gemm(g, a, w, out, **kw)
    if _LOOKAHEAD[0] is not None:
        _LOOKAHEAD[0].visit([g], [w])
    L.check(lib.ea_gemm(C.byref(g), _stream()), "ea_gemm")
    return res


def gemm_grouped(calls):
    """calls: list (1..3) of (a, w, out, kwargs) with the same shape and flags - ONE launch (ea_gemm_grouped).
    Returns the list of outputs."""
    lib = L.lib()
    n = len(calls)
    arr = (L.GemmArgs * n)()
    outs = [_fill_gemm(arr[i], a, w, out, **kw) for i, (a, w, out, kw) in enumerate(calls)]
    if _LOOKAHEAD[0] is not None:
        _LOOKAHEAD[0].visit([arr[i] for i in range(n)], [c[1] for c in calls])
    L.check(lib.ea_gemm_grouped(arr, n, _stream()), "ea_gemm_grouped")
    return outs


def attention(q, k, v, out, *, B, heads, Nq, Nkv, d, q_strides, k_strides, v_strides, o_strides,
              scale, rel_h=None, rel_w=None, rel_s=0):
    """q/k/v are base tensors; *_strides = (batch_stride, row_stride) in elements."""
    lib = L.lib()
    a = L.AttnArgs()
    a.q, a.k, a.v, a.out = q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr()
    a.B, a.heads, a.Nq, a.Nkv, a.d = B, heads, Nq, Nkv, d
    a.q_bs, a.q_ns = q_strides
    a.k_bs, a.k_ns = k_strides
    a.v_bs, a.v_ns = v_strides
    a.o_bs, a.o_ns = o_strides
    a.scale = scale
    if rel_h is not None:
        a.rel_h, a.rel_w, a.rel_s = rel_h.data_ptr(), rel_w.data_ptr(), rel_s
    L.check(lib.ea_attention(C.byref(a), _stream()), "ea_attention")
    return out


def gn_workspace(B, device, groups=32):
    """Zeroed ea_groupnorm workspace for B images (EA_GN_WS_FLOATS: counters + one partial slot per (image, CTA))."""
    return torch.zeros(2 * B + 2 * groups * 256, device=device, dtype=torch.float32)


def groupnorm(x, gamma, beta, out, *, B, HW, C_, groups=32, eps=1e-5, silu=True, workspace=None,
              x2=None, C1=0, ldx=None, ldx2=None, ldo=None):
    lib = L.lib()
    g = L.GnArgs()
    g.x = x.data_ptr()
    g.ldx = ldx if ldx is not None else (C1 if x2 is not None else C_)
    if x2 is not None:
        g.x2 = x2.data_ptr()
        g.C1 = C1
        g.ldx2 = ldx2 if ldx2 is not None else (C_ - C1)
    if isinstance(gamma, (list, tuple)):     # one (gamma, beta) per stacked network (ea_gn_args.n_nets)
        g.n_nets = len(gamma)
        for i in range(1, len(gamma)):
            g.gamma_more[i - 1], g.beta_more[i - 1] = gamma[i].data_ptr(), beta[i].data_ptr()
        gamma, beta = gamma[0], beta[0]
    g.gamma, g.beta = gamma.data_ptr(), beta.data_ptr()
    g.out = out.data_ptr()
    g.ldo = ldo if ldo is not None else C_
    g.B, g.HW, g.C, g.groups = B, HW, C_, groups
    g.eps, g.silu = eps, 1 if silu else 0
    g.two_pass = 1 if _CONCURRENT[0] else 0
    if workspace is None:
        workspace = gn_workspace(B, x.device, groups)
    g.workspace = workspace.data_ptr()
    L.check(lib.ea_groupnorm(C.byref(g), _stream()), "ea_groupnorm")
    return out


def layernorm(x, gamma, beta, out, *, M, C_, eps=1e-5, ldx=None, ldo=None):
    lib = L.lib()
    L.check(lib.ea_layernorm(_p(x), ldx if ldx is not None else C_, _p(gamma), _p(beta), _p(out),
                             ldo if ldo is not None else C_, M, C_, eps, _stream()), "ea_layernorm")
    return out


def conv_direct(x, w, bias, out, *, B, Hin, Win, Cin, Cout, ksize=3, stride=1, silu=False, add=None, ldo=0):
    """w: fp32 [k, k, Cin, Cout]."""
    lib = L.lib()
    L.check(lib.ea_conv_direct(_p(x), _p(w), _p(bias), _p(out), B, Hin, Win, Cin, Cout, ksize, stride,
                               1 if silu else 0, _p(add), ldo, _stream()), "ea_conv_direct")
    return out


def conv_in(x, w, bias, out, *, B, H, W, Cin, Cout, out2=None, add=None, ldo=0, ldo2=0):
    """w: fp32 [3, 3, Cin, Cout]; out2 = optional second destination, add = optional dense addend."""
    lib = L.lib()
    L.check(lib.ea_conv_in(_p(x), _p(w), _p(bias), _p(out), ldo, _p(out2), ldo2, _p(add), B, H, W, Cin, Cout,
                           _stream()), "ea_conv_in")
    return out


def upsample2x(x, out, *, B, H, W, C_):
    lib = L.lib()
    L.check(lib.ea_upsample2x(_p(x), _p(out), B, H, W, C_, _stream()), "ea_upsample2x")
    return out


def small_linear(x, w, bias, y, *, M, N, K, silu_in=False, silu_out=False):
    lib = L.lib()
    L.check(lib.ea_small_linear(_p(x), _p(w), _p(bias), _p(y), M, N, K, 1 if silu_in else 0,
                                1 if silu_out else 0, _stream()), "ea_small_linear")
    return y


def timestep_embedding(t, out, *, B, dim):
    lib = L.lib()
    L.check(lib.ea_timestep_embedding(_p(t), _p(out), B, dim, _stream()), "ea_timestep_embedding")
    return out


def check_out_buffers(what, copies, xn, w, bias, latents, eps_out, coef, known, noise, mask, lat_half_out,
                      step_counter, hist, Nimg, H, W, C_):
    """The element count of every buffer of ea_out_cfg_ddim (copies = 2: the network rows are the two guidance
    halves) or ea_out_ddim (copies = 1), checked before the launch: the kernels index them from (Nimg, H, W, C_)
    alone, so a buffer sized for the other entry point would be read or written out of bounds."""
    if min(Nimg, H, W, C_) < 1:
        raise ValueError(f"{what}: Nimg, H, W, C must be positive, got {(Nimg, H, W, C_)}")
    px = Nimg * H * W
    want = {"xn": (xn, copies * px * C_), "w": (w, 36 * C_), "bias": (bias, 4), "latents": (latents, px * 4),
            "eps_out": (eps_out, copies * px * 4), "known": (known, px * 4),
            "noise": (noise, px * 4), "mask": (mask, px), "lat_half_out": (lat_half_out, copies * px * 4),
            "step_counter": (step_counter, 1), "hist": (hist, 3 * px * 4)}
    for name, (t, n) in want.items():
        if t is not None and t.numel() != n:
            raise ValueError(f"{what}: {name} has {t.numel()} elements, Nimg={Nimg}, H={H}, W={W}, C={C_} needs {n}")
    # coef: the DDIM terms always, the blend terms with noise, the multistep row with hist
    n_coef = 16 if hist is not None else 7 if noise is not None else 4
    if latents is not None and (coef is None or coef.numel() < n_coef):
        raise ValueError(f"{what}: coef needs at least {n_coef} elements, has {None if coef is None else coef.numel()}")


PREDICTION_TYPES = ("epsilon", "v_prediction")


def check_prediction(what, prediction):
    """The network-output parameterisations the fused update implements: eps (SD1.5, SD2-inpainting) and v
    (SD2.1-768, diffusers' "v_prediction")."""
    if prediction not in PREDICTION_TYPES:
        raise ValueError(f"{what}: prediction must be one of {PREDICTION_TYPES}, got {prediction!r}")


def out_cfg_ddim(xn, w, bias, *, latents=None, eps_out=None, coef=None, guidance=1.0, known=None, noise=None,
                 mask=None, lat_half_out=None, step_counter=None, hist=None, Nimg, H, W, C_, prediction="epsilon"):
    """ea_out_cfg_ddim, or ea_out_cfg_vpred with prediction="v_prediction" (the network output is v)."""
    check_prediction("out_cfg_ddim", prediction)
    check_out_buffers("out_cfg_ddim", 2, xn, w, bias, latents, eps_out, coef, known, noise, mask, lat_half_out,
                      step_counter, hist, Nimg, H, W, C_)
    lib = L.lib()
    name = "ea_out_cfg_ddim" if prediction == "epsilon" else "ea_out_cfg_vpred"
    L.check(getattr(lib, name)(_p(xn), _p(w), _p(bias), _p(latents), _p(eps_out), _p(coef),
                               float(guidance), _p(known), _p(noise), _p(mask), _p(lat_half_out),
                               _p(step_counter), _p(hist), Nimg, H, W, C_, _stream()), name)


def out_ddim(xn, w, bias, *, latents=None, eps_out=None, coef=None, known=None, noise=None, mask=None,
             lat_half_out=None, step_counter=None, hist=None, Nimg, H, W, C_, prediction="epsilon"):
    """ea_out_ddim: the out conv and update of out_cfg_ddim without guidance; every buffer holds the Nimg images
    once.  prediction="v_prediction": ea_out_vpred."""
    check_prediction("out_ddim", prediction)
    check_out_buffers("out_ddim", 1, xn, w, bias, latents, eps_out, coef, known, noise, mask, lat_half_out,
                      step_counter, hist, Nimg, H, W, C_)
    lib = L.lib()
    name = "ea_out_ddim" if prediction == "epsilon" else "ea_out_vpred"
    L.check(getattr(lib, name)(_p(xn), _p(w), _p(bias), _p(latents), _p(eps_out), _p(coef), _p(known), _p(noise),
                               _p(mask), _p(lat_half_out), _p(step_counter), _p(hist), Nimg, H, W, C_, _stream()),
            name)


def check_mix_buffers(latents, known, mask, noise, mix, step_counter, lat_half_out, copies, Nimg, H, W):
    """The element counts of ea_latent_mix's buffers, checked before the launch (the kernel indexes them from
    (Nimg, H, W) and the step counter alone).  `mix` is [n_rows, 4] and the noise table holds n_rows rows of
    [Nimg, H, W, 4]."""
    if min(Nimg, H, W) < 1 or copies not in (1, 2):
        raise ValueError(f"latent_mix: Nimg, H, W must be positive and copies 1 or 2, got {(Nimg, H, W, copies)}")
    px = Nimg * H * W
    want = {"latents": (latents, px * 4), "known": (known, px * 4), "mask": (mask, px), "step_counter": (step_counter, 1),
            "lat_half_out": (lat_half_out, copies * px * 4)}
    for name, (t, n) in want.items():
        if t is not None and t.numel() != n:
            raise ValueError(f"latent_mix: {name} has {t.numel()} elements, Nimg={Nimg}, H={H}, W={W} needs {n}")
    if mix.dim() != 2 or mix.shape[1] != 4 or mix.shape[0] < 1:
        raise ValueError(f"latent_mix: mix must be [n_rows, 4], got {tuple(mix.shape)}")
    if noise.numel() != mix.shape[0] * px * 4:
        raise ValueError(f"latent_mix: noise has {noise.numel()} elements, {mix.shape[0]} rows of {px * 4} needed")


def latent_mix(latents, known, mask, noise, mix, *, alpha, step_counter, lat_half_out=None, copies=1, Nimg, H, W):
    """ea_latent_mix: the alpha-mixing pipeline's per-step mix of the latents with the re-noised source, row
    *step_counter - 1 of `mix` = [n_rows, 4] {k_init, k_noise, in_window, active} and of the noise table."""
    check_mix_buffers(latents, known, mask, noise, mix, step_counter, lat_half_out, copies, Nimg, H, W)
    lib = L.lib()
    L.check(lib.ea_latent_mix(_p(latents), _p(known), _p(mask), _p(noise), _p(mix), float(alpha), _p(step_counter),
                              int(mix.shape[0]), _p(lat_half_out), int(copies), Nimg, H, W, _stream()),
            "ea_latent_mix")


def step_gather(step_counter, n_rows, tables, dsts):
    """dsts[k][:] = tables[k][min(*step_counter, n_rows - 1)] for fp32 tables [rows, ...] (one launch)."""
    lib = L.lib()
    n = len(tables)
    src = (C.c_void_p * n)(*[t.data_ptr() for t in tables])
    dst = (C.c_void_p * n)(*[d.data_ptr() for d in dsts])
    rows = (C.c_longlong * n)(*[d.numel() for d in dsts])
    L.check(lib.ea_step_gather(_p(step_counter), int(n_rows), n, src, dst, rows, _stream()), "ea_step_gather")


def sam_relpos(q, q_bs, q_ns, Rh, Rw, rel_h, rel_w, *, B, heads, S, d):
    lib = L.lib()
    L.check(lib.ea_sam_relpos(_p(q), q_bs, q_ns, _p(Rh), _p(Rw), _p(rel_h), _p(rel_w), B, heads, S, d,
                              _stream()), "ea_sam_relpos")


def window_partition(x, out, *, B, H, W, C_, ws):
    lib = L.lib()
    L.check(lib.ea_window_partition(_p(x), _p(out), B, H, W, C_, ws, _stream()), "ea_window_partition")
    return out


def window_unpartition(xw, residual, out, *, B, H, W, C_, ws):
    lib = L.lib()
    L.check(lib.ea_window_unpartition(_p(xw), _p(residual), _p(out), B, H, W, C_, ws, _stream()),
            "ea_window_unpartition")
    return out


def sam_patchify(img, out, *, B, Cin, H, W, ps):
    lib = L.lib()
    L.check(lib.ea_sam_patchify(_p(img), _p(out), B, Cin, H, W, ps, _stream()), "ea_sam_patchify")
    return out


def nhwc_to_nchw_f32(x, out, *, B, HW, C_):
    lib = L.lib()
    L.check(lib.ea_nhwc_to_nchw_f32(_p(x), _p(out), B, HW, C_, _stream()), "ea_nhwc_to_nchw_f32")
    return out


def softmax_rows(s, p, *, rows, cols, lds=None, ldp=None):
    """p = softmax(s, dim=-1): fp32 logits [rows, cols] -> half probabilities (VAE AttnBlock)."""
    lib = L.lib()
    L.check(lib.ea_softmax_rows(_p(s), lds if lds is not None else cols, _p(p), ldp if ldp is not None else cols,
                                rows, cols, _stream()), "ea_softmax_rows")
    return p


def image_out(x, out, *, B, HW, C_, ldx, scale=0.5, shift=0.5, lo=0.0, hi=1.0):
    """half NHWC rows (first C_ channels of ldx) -> fp32 NCHW, clamp(x * scale + shift, lo, hi)."""
    lib = L.lib()
    L.check(lib.ea_image_out(_p(x), ldx, _p(out), B, HW, C_, scale, shift, lo, hi, _stream()), "ea_image_out")
    return out

