"""An auditing ops backend: every launch an engine makes, checked on its own inputs against float64.

`Auditor(backend)` stands in for the operator table of DenoiseEngine, SamEncoderEngine or the VAE engines (like
`Recorder` in tests/test_step_trace_cpu.py) and forwards each call to `backend` (editanything_b200.ops on the GPU,
tests/cpu_ops.py on the CPU).  For every call it

 1. declares, from the C ABI (include/editanything_b200.h) and the keywords of the ops.* call - never from the
    marshalled ctypes struct - the elements of each tensor operand the call may read or write: LINEAR A is M rows x K
    at row stride lda, a conv input is the input-resolution NHWC pixels x Cin at pixel stride lda, W is N rows x the
    total K at ldw, a row vector is batches x N at its row stride, out / out2 / residual / out_f32 are M x n_out at
    their own strides, attention operands follow from (batch stride, row stride), heads and d, ...;
 2. synchronises, snapshots every storage it touches, runs the call unchanged on the current stream (with whatever
    lane the engine selected), synchronises again;
 3. recomputes the written operands in float64 from the snapshot and applies the per-element bound of that kernel's
    suite (tests/test_gpu_kernels_fp64.py, tests/test_gpu_conv_fp64.py, tests/test_gpu_attention.py); layout and copy
    kernels must be bit-exact, a grouped GEMM is checked group by group.  The float64 side is built in bands of at
    most CHUNK_ELEMS outputs (rows of a GEMM; output rows of one image for a convolution, with the input rows they
    reach; pixel rows of one image for GroupNorm, whose statistics are merged over the bands first; query rows of one
    batch element for attention), and only the slice of each operand a band reads is upcast, so that the full
    2048 x 2752 tile-refinement layers (2.9 GB fp16 activations) are checked in bounded memory;
 4. requires every element of a written storage outside the declared written extent to be bit-identical to the
    snapshot, the GEMM split-K and GroupNorm workspace counters to be zero again and the step counter to be +1;
 5. re-runs the call on relocated copies of every storage: each a fresh allocation with a NaN margin of at least
    max(2 MiB, 128 rows) before and after, every element outside the declared read extents NaN, every operand at its
    old byte offset (same alignment) and views of one storage still sharing one.  The outputs must equal the
    production run bit for bit and every NaN outside the written extents must still be there: a read outside the
    declared operands that reaches a result, or a store outside them, shows here.  Integer storages and scratch
    workspaces are copied whole.

A failure (AuditError) names the case, the call index, the op and its call site, the operand, the worst element and
its got / ref / bound.  `Auditor.worst` keeps the worst error / bound per (op, call site)."""
import inspect
import os
import traceback

import numpy as np
import torch
import torch.nn.functional as F

from tests import attn_ref, cpu_ops
from tests import fp64_refs as R

U = R.U32
NORM_K = 16.0                 # fp32 ulps on each term of a normalisation's affine map (test_gpu_kernels_fp64.py)
MARGIN_BYTES = 2 << 20
MARGIN_ROWS = 128
LINEAR, CONV_S1, CONV_S2, CONV_S2A = 0, 1, 2, 3
ACT = {0: "none", 1: "silu", 2: "gelu", 3: "geglu"}
GEMM_WS_COUNTER_BYTES = 65536
CHUNK_ELEMS = 1 << 24       # float64 references are built at most this many outputs at a time (at least one row)
# operator-table entries that launch nothing
PASSTHROUGH = {"half_dtype", "launch_count", "reset_launch_count", "gn_workspace", "gemm_workspace",
               "weight_lookahead", "WeightLookahead", "check_out_buffers", "check_prediction"}


class AuditError(AssertionError):
    pass


class Operand:
    """One declared extent: the elements as_strided(storage of `t`, size, stride, offset) (in t's dtype).
    role: "r" read, "w" written, "rw" both, "scratch" (written freely; the storage is copied, not fenced)."""

    def __init__(self, name, t, size, stride, offset, role):
        self.name, self.t, self.role = name, t, role
        self.size, self.stride, self.offset = tuple(int(s) for s in size), tuple(int(s) for s in stride), int(offset)

    def view(self, flat, shift=0):
        return torch.as_strided(flat, self.size, self.stride, self.offset + shift)

    @property
    def reads(self):
        return self.role in ("r", "rw")

    @property
    def writes(self):
        return self.role in ("w", "rw", "scratch")


def rows(name, t, n_rows, n_cols, ld, role="r"):
    """n_rows x n_cols at row stride ld from t's first element."""
    return Operand(name, t, (n_rows, n_cols), (ld, 1), t.storage_offset(), role)


def dense(name, t, shape, role="r"):
    """`shape` contiguous from t's first element."""
    st = torch.empty(shape, device="meta").stride()
    return Operand(name, t, shape, st, t.storage_offset(), role)


def _flat(t):
    """The whole storage of t as a 1-D tensor of t's dtype."""
    st = t.untyped_storage()
    return torch.empty(0, dtype=t.dtype, device=t.device).set_(st, 0, (st.nbytes() // t.element_size(),), (1,))


def _bits(t):
    return t.view({2: torch.int16, 4: torch.int32, 1: torch.uint8, 8: torch.int64}[t.element_size()])


def _key(t):
    return t.untyped_storage().data_ptr()


def _sync(dev):
    if dev.type == "cuda":
        torch.cuda.synchronize(dev)


class Spec:
    """The operands of one call and its float64 check: check(snap, got) yields (operand, got, ref, bound) with
    bound None for bit-exact, snap(name) / got(name) the pre-call / the post-call declared view, both in the stored
    dtype (a check upcasts the slices it reads with _d)."""

    def __init__(self, op, operands, check, after=None):
        self.op, self.operands, self.check, self.after = op, operands, check, after


def _d(t):
    """float64 (integer storages: int64) copy of a slice of an operand."""
    return t.double() if t.is_floating_point() else t.long()


def bands(n, per):
    """[lo, hi) ranges covering range(n), at most max(1, per) long."""
    per = max(1, int(per))
    return [(lo, min(n, lo + per)) for lo in range(0, n, per)]


def _whole(snap):
    """snap for a check of small operands: each one upcast whole."""
    return lambda name: _d(snap(name))


def _tag(parts, label):
    """The band an operand's check covers, in its name when there is more than one band."""
    return f" [{label}]" if len(parts) > 1 else ""


def conv_rows(x, w, k, stride, top, wpad, y0, y1):
    """Output rows [y0, y1) of a k x k convolution without bias: x NHWC [B, Hin, Win, Cin] in any dtype, of which only
    the input rows the band reaches are upcast; w [k, k, Cin, Cout] float64.  The input is zero-padded by `top` rows
    above row 0 (and below the last row as far as the kernel reaches) and by wpad = (left, right) columns; output row
    y reads padded rows stride * y .. stride * y + k - 1.  Returns (out [B, y1 - y0, Wo, Cout], sum of |x w|)."""
    Hin = x.shape[1]
    p0, p1 = stride * y0 - top, stride * (y1 - 1) - top + k       # input rows read, in image coordinates
    lo, hi = max(0, p0), min(Hin, p1)
    xb = F.pad(x[:, lo:hi].double().permute(0, 3, 1, 2), (wpad[0], wpad[1], lo - p0, p1 - hi))
    wt = w.permute(3, 2, 0, 1)
    out = F.conv2d(xb, wt, stride=stride).permute(0, 2, 3, 1)
    mag = F.conv2d(xb.abs(), wt.abs(), stride=stride).permute(0, 2, 3, 1)
    return out, mag


# ea_gemm's convolution modes as (stride, zero rows above row 0, zero columns (left, right)) - R.conv_gemm's padding
CONV_GEOM = {CONV_S1: (1, 1, (1, 1)), CONV_S2: (2, 1, (1, 1)), CONV_S2A: (2, 0, (0, 1))}


def conv_gemm_rows(x, w, mode, y0, y1, extra=None):
    """R.conv_gemm(x, w, mode, extra)[:, y0:y1] built from the input rows those outputs reach: +-1 row for CONV_S1,
    rows 2y - 1 .. 2y + 1 for CONV_S2, 2y .. 2y + 2 (the last one the bottom zero pad) for CONV_S2A, and extra's rows
    y0 .. y1 - 1.  x / extra in any dtype (sliced, then upcast), w [Cout, 9 Cin (+ Cin_extra)] float64."""
    cout, cin = w.shape[0], x.shape[-1]
    s, top, wpad = CONV_GEOM[mode]
    out, mag = conv_rows(x, w[:, :9 * cin].reshape(cout, 3, 3, cin).permute(1, 2, 3, 0), 3, s, top, wpad, y0, y1)
    if extra is not None:
        we = w[:, 9 * cin:]
        e = extra[:, y0:y1].double()
        out, mag = out + e @ we.T, mag + e.abs() @ we.abs().T
    return out, mag


def groupnorm_stats(band_iter, B, groups):
    """Per (image, group) float64 (count, mean, M2) over bands of one image's pixel rows, merged pairwise (Chan, Golub
    & LeVeque): n = na + nb, mean = mean_a + d nb / n, M2 = M2_a + M2_b + d^2 na nb / n with d = mean_b - mean_a.
    band_iter yields (image, band [rows, groups, C / groups] float64)."""
    n = [0.0] * B
    mean = m2 = None
    for b, xg in band_iter:
        if mean is None:
            mean = torch.zeros(B, groups, dtype=torch.float64, device=xg.device)
            m2 = torch.zeros_like(mean)
        nb = float(xg.shape[0] * xg.shape[2])
        mb = xg.mean(dim=(0, 2))
        m2b = ((xg - mb[:, None]) ** 2).sum(dim=(0, 2))
        na, tot = n[b], n[b] + nb
        d = mb - mean[b]
        mean[b] += d * (nb / tot)
        m2[b] += m2b + d * d * (na * nb / tot)
        n[b] = tot
    return n, mean, m2


# ================================================ handlers ======================================================
def _gemm_spec(a, w, out, kw, hdt, prefix=""):
    """One ea_gemm problem.  Returns (Spec, the output tensor the call returns)."""
    mode = kw.get("mode", LINEAR)
    act = kw.get("act", 0)
    N = kw.get("N") or w.shape[0]
    n_out = N // 2 if act == 3 else N
    ops_ = []
    P = prefix
    if mode == LINEAR:
        M = kw.get("M") or a.shape[0]
        K = kw.get("K") or a.shape[-1]
        lda = kw.get("lda") or a.stride(0)
        ops_.append(rows(P + "a", a, M, K, lda))
        Ktot = K
        batch_rows = kw.get("rows_per_batch", 0)
    else:
        B, H, W_, Cin = kw["conv"]
        M = B * H * W_
        s = 1 if mode == CONV_S1 else 2
        Hin, Win = s * H, s * W_
        lda = kw.get("lda") or Cin
        ops_.append(Operand(P + "a", a, (B, Hin, Win, Cin), (Hin * Win * lda, Win * lda, lda, 1), a.storage_offset(), "r"))
        Ktot = 9 * Cin
        xe = kw.get("a_extra")
        if xe is not None:
            ce = xe.shape[-1]
            lde = kw.get("ld_extra") or ce
            ops_.append(Operand(P + "a_extra", xe, (B, H, W_, ce), (H * W_ * lde, W_ * lde, lde, 1), xe.storage_offset(),
                                "r"))
            Ktot += ce
        batch_rows = H * W_
    ops_.append(rows(P + "w", w, N, Ktot, kw.get("ldw") or Ktot))
    bias, rv, res = kw.get("bias"), kw.get("rowvec"), kw.get("residual")
    if bias is not None:
        ops_.append(dense(P + "bias", bias, (N,)))
    if rv is not None:
        nb = (-(-M // batch_rows) if batch_rows else 1)
        ops_.append(rows(P + "rowvec", rv, nb, N, rv.stride(0)))
    if res is not None:
        ops_.append(rows(P + "residual", res, M, n_out, kw.get("ldr") or res.stride(-2)))
    o32 = kw.get("out_f32")
    acc = bool(kw.get("accumulate"))
    if out is None and o32 is None:
        out = torch.empty((M, n_out), device=a.device, dtype=hdt)
    dst = o32 if o32 is not None else out
    ops_.append(rows(P + ("out_f32" if o32 is not None else "out"), dst, M, n_out, kw.get("ldo") or dst.stride(-2),
                     "rw" if acc else "w"))
    o2 = kw.get("out2")
    if o2 is not None:
        ops_.append(rows(P + "out2", o2, M, n_out, kw.get("ldo2") or o2.stride(-2), "w"))
    rso = kw.get("rowstats_out")
    if rso is not None:
        ops_.append(dense(P + "rowstats_out", rso, (N // 32, M, 2), "w"))
    ln = kw.get("ln")
    if ln is not None:
        ops_.append(dense(P + "ln_stats", ln[0], (Ktot // 32, M, 2)))
        ops_.append(dense(P + "ln_g", ln[1], (N,)))
    rs = kw.get("row_scale")
    if rs is not None:
        ops_.append(dense(P + "row_scale", rs, (M,)))
    dname = P + ("out_f32" if o32 is not None else "out")

    def chunks():
        """(first row, end row, label, image, first output row, end output row) of the bands the float64 reference
        is built in, at most CHUNK_ELEMS outputs (and for a LINEAR problem CHUNK_ELEMS A elements) each: rows of M,
        or for a convolution whole output rows of one image."""
        if mode == LINEAR:
            return [(r0, r1, f"rows {r0}-{r1 - 1}", None, None, None)
                    for r0, r1 in bands(M, CHUNK_ELEMS // max(N, Ktot, 1))]
        B, H, W_ = kw["conv"][:3]
        return [(b * H * W_ + y0 * W_, b * H * W_ + y1 * W_, f"image {b} rows {y0}-{y1 - 1}", b, y0, y1)
                for b in range(B) for y0, y1 in bands(H, CHUNK_ELEMS // max(N * W_, 1))]

    def check(snap, got):
        A, Wd = snap(P + "a"), _d(snap(P + "w"))
        bd = _d(snap(P + "bias")) if bias is not None else None
        rvd = _d(snap(P + "rowvec")) if rv is not None else None
        rsd = _d(snap(P + "row_scale")) if rs is not None else None
        g_all = got(dname)
        parts = chunks()
        for r0, r1, label, b, y0, y1 in parts:
            tag = _tag(parts, label)
            if mode == LINEAR:
                Ac = _d(A[r0:r1])
                if ln is not None:
                    mu = Ac.mean(-1, keepdim=True)
                    r = (Ac.var(-1, correction=0, keepdim=True) + ln[2]).rsqrt()
                    pre = ((Ac - mu) * r) @ Wd.T
                    e = (Ktot + 2) * U * r * (Ac.abs() @ Wd.abs().T + mu.abs() * _d(snap(P + "ln_g")).abs())
                else:
                    pre = Ac @ Wd.T
                    mag = Ac.abs() @ Wd.abs().T
                del Ac
            else:
                xe_ = snap(P + "a_extra")[b:b + 1] if xe is not None else None
                pre, mag = conv_gemm_rows(A[b:b + 1], Wd, mode, y0, y1, xe_)
                pre, mag = pre.reshape(r1 - r0, N), mag.reshape(r1 - r0, N)
            if ln is not None:
                if bd is not None:
                    pre = pre + bd
                    e = e + 2 * U * bd.abs()
            else:
                if bd is not None:
                    pre, mag = pre + bd, mag + bd.abs()
                if rvd is not None:
                    rows_ = torch.arange(r0, r1, device=rvd.device)
                    idx = rows_ // batch_rows if batch_rows else torch.zeros_like(rows_)
                    pre, mag = pre + rvd[idx], mag + rvd[idx].abs()
                e = (Ktot + 2) * U * mag
                del mag
            y, err = R.gemm_act(ACT[act], pre, e)
            del pre, e
            scale = float(kw.get("out_scale", 1.0))
            n_scale = int(scale != 1.0)
            if rsd is not None:
                scale = scale * rsd[r0:r1, None]
                n_scale += 1
            extras = []
            if res is not None:
                extras.append(_d(snap(P + "residual")[r0:r1]))
            if acc:
                extras.append(_d(snap(dname)[r0:r1]))
            ref, bound = R.gemm_out(y, err, scale, extras, None if o32 is not None else hdt, n_scale)
            del y, err
            g = g_all[r0:r1]
            yield dname + tag, g, ref, bound
            del ref, bound
            if o2 is not None:
                yield P + "out2" + tag, got(P + "out2")[r0:r1], g, None
            if rso is not None:
                xc = g.double().reshape(r1 - r0, N // 32, 32).permute(1, 0, 2)
                sm = xc.sum(-1)
                m2 = ((xc - sm[..., None] / 32) ** 2).sum(-1)
                sabs = xc.abs().sum(-1)
                st = got(P + "rowstats_out")[:, r0:r1]
                yield P + "rowstats_out[sum]" + tag, st[..., 0], sm, 32 * U * sabs
                yield P + "rowstats_out[M2]" + tag, st[..., 1], m2, 40 * U * m2 + 32 * (U * sabs) ** 2

    return Spec("gemm", ops_, check), out


def h_gemm(be, a, hdt):
    kw = {k: v for k, v in a.items() if k not in ("a", "w", "out")}
    spec, a["out"] = _gemm_spec(a["a"], a["w"], a["out"], kw, hdt)
    return spec


def h_gemm_grouped(be, a, hdt):
    calls = []
    specs = []
    for g, (x, w, out, kw) in enumerate(a["calls"]):
        spec, out = _gemm_spec(x, w, out, kw, hdt, prefix=f"g{g}.")
        calls.append((x, w, out, kw))
        specs.append(spec)
    a["calls"] = calls

    def check(snap, got):
        for s in specs:
            yield from s.check(snap, got)
    return Spec("gemm_grouped", [o for s in specs for o in s.operands], check)


def h_attention(be, a, hdt):
    B, heads, Nq, Nkv, d = a["B"], a["heads"], a["Nq"], a["Nkv"], a["d"]
    q, k, v, out = a["q"], a["k"], a["v"], a["out"]
    hd = heads * d
    o = [Operand("q", q, (B, Nq, hd), (a["q_strides"][0], a["q_strides"][1], 1), q.storage_offset(), "r"),
         Operand("k", k, (B, Nkv, hd), (a["k_strides"][0], a["k_strides"][1], 1), k.storage_offset(), "r"),
         Operand("v", v, (B, Nkv, hd), (a["v_strides"][0], a["v_strides"][1], 1), v.storage_offset(), "r"),
         Operand("out", out, (B, Nq, hd), (a["o_strides"][0], a["o_strides"][1], 1), out.storage_offset(), "w")]
    rel = a.get("rel_h") is not None
    S = a.get("rel_s", 0)
    if rel:
        o += [dense("rel_h", a["rel_h"], (B * heads, Nq, S)), dense("rel_w", a["rel_w"], (B * heads, Nq, S))]

    def check(snap, got):
        """One batch element and at most CHUNK_ELEMS outputs at a time: attention_bound upcasts K and V of one
        (element, head) and builds its logits in chunks of query rows, so no float64 tensor is larger than those
        plus one band's output and bound."""
        sh = lambda t, n: t.reshape(1, n, heads, d)
        parts = [(b, r0, r1) for b in range(B) for r0, r1 in bands(Nq, CHUNK_ELEMS // hd)]
        for b, r0, r1 in parts:
            hs = slice(b * heads, (b + 1) * heads)
            ref, bound = attn_ref.attention_bound(sh(snap("q")[b:b + 1, r0:r1], r1 - r0), sh(snap("k")[b:b + 1], Nkv),
                                                  sh(snap("v")[b:b + 1], Nkv), a["scale"],
                                                  snap("rel_h")[hs, r0:r1] if rel else None,
                                                  snap("rel_w")[hs, r0:r1] if rel else None, S, dtype=hdt)
            yield ("out" + _tag(parts, f"batch {b} rows {r0}-{r1 - 1}"), got("out")[b:b + 1, r0:r1],
                   ref.reshape(1, r1 - r0, hd), bound.reshape(1, r1 - r0, hd))
    return Spec("attention", o, check)


def h_groupnorm(be, a, hdt):
    B, HW, C, groups = a["B"], a["HW"], a["C_"], a["groups"]
    x, x2, out = a["x"], a.get("x2"), a["out"]
    C1 = a.get("C1", 0) if x2 is not None else C
    ldx = a.get("ldx") or (C1 if x2 is not None else C)
    o = [rows("x", x, B * HW, C1, ldx)]
    if x2 is not None:
        o.append(rows("x2", x2, B * HW, C - C1, a.get("ldx2") or (C - C1)))
    gam, bet = a["gamma"], a["beta"]
    gl = list(gam) if isinstance(gam, (list, tuple)) else [gam]
    bl = list(bet) if isinstance(bet, (list, tuple)) else [bet]
    for i, (g, b) in enumerate(zip(gl, bl)):
        o += [dense(f"gamma{i}", g, (C,)), dense(f"beta{i}", b, (C,))]
    o.append(rows("out", out, B * HW, C, a.get("ldo") or C, "w"))
    if a.get("workspace") is None:
        a["workspace"] = be.gn_workspace(B, x.device, groups)
    ws = a["workspace"]
    o.append(dense("workspace", ws, (2 * B + 2 * groups * 256,), "scratch"))

    def check(snap, got):
        """R.groupnorm in two passes.  Pass 1 walks each image one CTA's pixels at a time in the kernel's launch
        geometry (R.gn_geometry): the per-(image, group) mean and M2 merged over the CTAs, and the running error
        bound of the kernel's fp32 sums in their order (R.gn_cta_sums, R.gn_cross_cta).  Pass 2 builds y, the
        pre-SiLU value, the rounding terms and the bound in bands of pixel rows.  The bound is the NORM_K-ulp one of
        the kernel suite plus what R.gn_stats_err derives for the statistics beyond the NORM_K unit those terms
        already give them; the worst ratio against the former alone is kept in `unit_worst`."""
        cpg = C // groups
        parts = [(b, p0, p1) for b in range(B) for p0, p1 in bands(HW, CHUNK_ELEMS // C)]

        def band(b, p0, p1):
            rws = slice(b * HW + p0, b * HW + p1)
            xb = _d(snap("x")[rws])
            if x2 is not None:
                xb = torch.cat([xb, _d(snap("x2")[rws])], -1)
            return xb.reshape(p1 - p0, groups, cpg)
        ks = torch.stack([band(b, 0, 1)[0, :, 0] for b in range(B)])        # the kernel's shifts [B, groups]
        n_sm = torch.cuda.get_device_properties(ks.device).multi_processor_count if ks.is_cuda else 132
        chunks, ppc, lanes, nparts = R.gn_geometry(B, HW, C, groups, n_sm)
        ctas = [(b, c * ppc, min(HW, (c + 1) * ppc)) for b in range(B) for c in range(chunks)]
        sa, sq = torch.zeros_like(ks), torch.zeros_like(ks)
        run = torch.zeros(B, 2, groups, dtype=torch.float64, device=ks.device)
        totals = [[] for _ in range(B)]

        def pass1():
            for b, p0, p1 in ctas:
                xg = band(b, p0, p1)
                dk = xg - ks[b][:, None]
                sa[b] += dk.abs().sum(dim=(0, 2))
                sq[b] += (dk * dk).sum(dim=(0, 2))
                t, r_ = R.gn_cta_sums(dk.reshape(p1 - p0, C), lanes, groups)
                run[b] += r_
                totals[b].append(t)
                del dk
                yield b, xg
        n, mean, m2 = groupnorm_stats(pass1(), B, groups)
        for b in range(B):
            run[b] += R.gn_cross_cta(torch.stack(totals[b]), nparts)
        nt = torch.tensor(n, dtype=torch.float64, device=m2.device)[:, None]
        var = m2 / nt
        r = (var + a["eps"]).rsqrt()
        d_mean, d_rstd = R.gn_stats_err(run.permute(1, 0, 2), sa, sq, nt, mean - ks, var, a["eps"])
        gs = [_d(snap(f"gamma{i}")) for i in range(len(gl))]
        bs = [_d(snap(f"beta{i}")) for i in range(len(gl))]
        per_net = B // len(gl)
        for b, p0, p1 in parts:
            g, bt = gs[b // per_net], bs[b // per_net]
            y = ((band(b, p0, p1) - mean[b, :, None]) * r[b, :, None]).reshape(p1 - p0, C)
            amu = (mean[b].abs() * r[b]).repeat_interleave(cpg)
            pre = y * g + bt
            terms = (y.abs() + amu + 1.0) * g.abs() + bt.abs()
            ch = lambda t: t[b].repeat_interleave(cpg)
            e = NORM_K * U * terms
            excess = R.gn_stats_excess(y, g, ch(r), ch(d_mean), ch(d_rstd), NORM_K * U)
            del y, terms
            ref = R.silu(pre) if a["silu"] else pre
            gb = got("out")[b * HW + p0:b * HW + p1]
            unit = R.ulp(ref, hdt) + (1.1 * e + R.silu_eval_err(pre) if a["silu"] else e)
            unit_worst[0] = max(unit_worst[0], R.worst_element(gb, ref, unit)[0])
            bound = unit + (1.1 * excess if a["silu"] else excess)
            del pre, e, excess, unit
            yield "out" + _tag(parts, f"image {b} rows {p0}-{p1 - 1}"), gb, ref, bound

    def after(post):
        cnt = post("workspace")[:2 * B]
        if bool(_bits(cnt).ne(0).any()):
            yield "workspace", "arrival counters not zero after the call"
    unit_worst = [0.0]
    spec = Spec("groupnorm", o, check, after)
    spec.unit_worst = unit_worst
    return spec


def h_layernorm(be, a, hdt):
    M, C = a["M"], a["C_"]
    o = [rows("x", a["x"], M, C, a.get("ldx") or C), dense("gamma", a["gamma"], (C,)), dense("beta", a["beta"], (C,)),
         rows("out", a["out"], M, C, a.get("ldo") or C, "w")]

    def check(snap, got):
        g, b = _d(snap("gamma")), _d(snap("beta"))
        parts = bands(M, CHUNK_ELEMS // C)
        for r0, r1 in parts:
            y, terms = R.layernorm(_d(snap("x")[r0:r1]), g, b, a["eps"])
            yield "out" + _tag(parts, f"rows {r0}-{r1 - 1}"), got("out")[r0:r1], y, R.ulp(y, hdt) + NORM_K * U * terms
    return Spec("layernorm", o, check)


def _conv_nhwc_bands(snap, k, s, B, Ho, Wo, Cout, has_bias):
    """R.conv_nhwc(x, w, bias, stride=s) (pad k // 2) in bands of whole output rows of one image, at most CHUNK_ELEMS
    outputs each: yields (label, image, y0, y1, out, sum of |x w| + |bias|)."""
    w = _d(snap("w"))
    bd = _d(snap("bias")) if has_bias else None
    parts = [(b, y0, y1) for b in range(B) for y0, y1 in bands(Ho, CHUNK_ELEMS // max(Wo * Cout, 1))]
    for b, y0, y1 in parts:
        pre, mag = conv_rows(snap("x")[b:b + 1], w, k, s, k // 2, (k // 2, k // 2), y0, y1)
        if bd is not None:
            pre, mag = pre + bd, mag + bd.abs()
        yield _tag(parts, f"image {b} rows {y0}-{y1 - 1}"), b, y0, y1, pre, mag


def h_conv_direct(be, a, hdt):
    B, Hin, Win, Cin, Cout, k, s = a["B"], a["Hin"], a["Win"], a["Cin"], a["Cout"], a["ksize"], a["stride"]
    Ho, Wo = -(-Hin // s), -(-Win // s)
    out, add = a["out"], a.get("add")
    ldo = a.get("ldo") or Cout
    o = [dense("x", a["x"], (B, Hin, Win, Cin)), dense("w", a["w"], (k, k, Cin, Cout))]
    if a.get("bias") is not None:
        o.append(dense("bias", a["bias"], (Cout,)))
    if add is not None:
        o.append(dense("add", add, (B, Ho, Wo, Cout)))
    o.append(Operand("out", out, (B, Ho, Wo, Cout), (Ho * Wo * ldo, Wo * ldo, ldo, 1), out.storage_offset(), "w"))

    def check(snap, got):
        for tag, b, y0, y1, pre, mag in _conv_nhwc_bands(snap, k, s, B, Ho, Wo, Cout, a.get("bias") is not None):
            e = (k * k * Cin + 1) * U * mag
            y = pre
            if a["silu"]:
                y, e = R.silu(pre), 1.1 * e + R.silu_eval_err(pre)
            ad = _d(snap("add")[b:b + 1, y0:y1]) if add is not None else torch.zeros_like(y)
            ref = y + ad
            yield "out" + tag, got("out")[b:b + 1, y0:y1], ref, R.ulp(ref, hdt) + e + 2 * U * (y.abs() + ad.abs())
    return Spec("conv_direct", o, check)


def h_conv_in(be, a, hdt):
    B, H, W_, Cin, Cout = a["B"], a["H"], a["W"], a["Cin"], a["Cout"]
    out, out2, add = a["out"], a.get("out2"), a.get("add")
    px = (H * W_, W_, 1)

    def nhwc(name, t, ld, role):
        return Operand(name, t, (B, H, W_, Cout), (px[0] * ld, px[1] * ld, ld, 1), t.storage_offset(), role)
    o = [dense("x", a["x"], (B, H, W_, Cin)), dense("w", a["w"], (3, 3, Cin, Cout))]
    if a.get("bias") is not None:
        o.append(dense("bias", a["bias"], (Cout,)))
    if add is not None:
        o.append(dense("add", add, (B, H, W_, Cout)))
    o.append(nhwc("out", out, a.get("ldo") or Cout, "w"))
    if out2 is not None:
        o.append(nhwc("out2", out2, a.get("ldo2") or Cout, "w"))

    def check(snap, got):
        for tag, b, y0, y1, ref, mag in _conv_nhwc_bands(snap, 3, 1, B, H, W_, Cout, a.get("bias") is not None):
            ad = _d(snap("add")[b:b + 1, y0:y1]) if add is not None else torch.zeros_like(ref)
            ref = ref + ad
            g = got("out")[b:b + 1, y0:y1]
            yield "out" + tag, g, ref, R.ulp(ref, hdt) + (9 * Cin + 2) * U * (mag + ad.abs())
            if out2 is not None:
                yield "out2" + tag, got("out2")[b:b + 1, y0:y1], g, None
    return Spec("conv_in", o, check)


def h_upsample2x(be, a, hdt):
    B, H, W_, C = a["B"], a["H"], a["W"], a["C_"]
    o = [dense("x", a["x"], (B, H, W_, C)), dense("out", a["out"], (B, 2 * H, 2 * W_, C), "w")]

    def check(snap, got):
        parts = [(b, y0, y1) for b in range(B) for y0, y1 in bands(H, CHUNK_ELEMS // (4 * W_ * C))]
        for b, y0, y1 in parts:
            yield ("out" + _tag(parts, f"image {b} rows {2 * y0}-{2 * y1 - 1}"), got("out")[b:b + 1, 2 * y0:2 * y1],
                   R.upsample2x(_d(snap("x")[b:b + 1, y0:y1])), None)
    return Spec("upsample2x", o, check)


def h_small_linear(be, a, hdt):
    M, N, K = a["M"], a["N"], a["K"]
    o = [dense("x", a["x"], (M, K)), dense("w", a["w"], (N, K))]
    if a.get("bias") is not None:
        o.append(dense("bias", a["bias"], (N,)))
    o.append(dense("y", a["y"], (M, N), "w"))

    def check(snap, got):
        snap = _whole(snap)
        x, w = snap("x"), snap("w")
        ref, pre, mag = R.small_linear(x, w, snap("bias") if a.get("bias") is not None else None, a["silu_in"],
                                       a["silu_out"])
        e = (K + 1) * U * mag
        if a["silu_in"]:
            e = e + R.silu_eval_err(x) @ w.abs().T
        if a["silu_out"]:
            e = 1.1 * e + R.silu_eval_err(pre)
        yield "y", got("y"), ref, e
    return Spec("small_linear", o, check)


def h_timestep_embedding(be, a, hdt):
    B, dim = a["B"], a["dim"]
    o = [dense("t", a["t"], (B,)), dense("out", a["out"], (B, dim), "w")]

    def check(snap, got):
        snap = _whole(snap)
        ref, arg, xf = R.timestep_embedding(snap("t"), dim)
        arg_err = (3 * xf[None].abs() + 4) * U * arg.abs()
        yield "out", got("out"), ref, torch.cat([arg_err, arg_err], dim=-1) + 4 * U
    return Spec("timestep_embedding", o, check)


def _h_out(copies):
    def handler(be, a, hdt):
        N, H, W_, C = a["Nimg"], a["H"], a["W"], a["C_"]
        px = (N, H, W_)
        lat, hist, noise = a.get("latents"), a.get("hist"), a.get("noise")
        vpred = a.get("prediction", "epsilon") == "v_prediction"
        o = [dense("xn", a["xn"], (copies * N, H, W_, C)), dense("w", a["w"], (4, 3, 3, C)), dense("bias", a["bias"], (4,))]
        opt = {"eps_out": ((copies * N, H, W_, 4), "w"), "latents": (px + (4,), "rw"), "known": (px + (4,), "r"),
               "noise": (px + (4,), "r"), "mask": (px, "r"), "lat_half_out": ((copies * N, H, W_, 4), "w"),
               "step_counter": ((1,), "rw"), "hist": ((3,) + px + (4,), "rw")}
        for name, (shape, role) in opt.items():
            if a.get(name) is not None and (lat is not None or name in ("eps_out", "step_counter")):
                o.append(dense(name, a[name], shape, role))
        if lat is not None:
            o.append(dense("coef", a["coef"], (16 if hist is not None else 7 if noise is not None else 4,)))

        def check(snap, got):
            snap = _whole(snap)
            eps, mag = R.out_conv(snap("xn"), snap("w"), snap("bias"))
            eb = (9 * C + 1) * U * mag
            if a.get("eps_out") is not None:
                yield "eps_out", got("eps_out"), eps, eb
            if a.get("step_counter") is not None:
                yield "step_counter", got("step_counter"), snap("step_counter") + 1, None
            if lat is None:
                return
            cf = [float(v) for v in snap("coef")]
            x = snap("latents")
            z = torch.zeros_like(x)
            if copies == 2:
                g = float(a["guidance"])
                eu, ec, bu, bc = eps[:N], eps[N:], eb[:N], eb[N:]
                m = R.cfg(eu, ec, g)
                m_err = abs(1 - g) * bu + abs(g) * bc + 3 * U * (eu.abs() + abs(g) * (ec.abs() + eu.abs()))
            else:
                m, m_err = eps, eb
            if vpred:
                x0 = R.ErrLin.lin([(cf[0], x, z), (-cf[1], m, m_err)])
                e = R.ErrLin.lin([(cf[0], m, m_err), (cf[1], x, z)])
            else:
                x0 = R.ErrLin.lin([(1.0 / cf[0], x, z), (-cf[1] / cf[0], m, m_err)])
                e = (m, m_err)
            if hist is not None and cf[7] != 0.0:
                hs = snap("hist")
                m1, m2, last = (hs[0], z), (hs[1], z), (hs[2], z)
                xc = R.ErrLin.lin([(cf[8], x, z), (cf[9], *last), (cf[10], *m1), (cf[11], *m2), (cf[12], *x0)])
                xp = R.ErrLin.lin([(cf[13], *xc), (cf[14], *x0), (cf[15], *m1)])
                hg = got("hist")
                yield "hist[m1]", hg[0], x0[0], x0[1]
                yield "hist[m2]", hg[1], hs[0], None
                yield "hist[last]", hg[2], xc[0], xc[1]
            else:
                xp = R.ErrLin.lin([(cf[2], *x0), (cf[3], *e)])
                if hist is not None:
                    yield "hist", got("hist"), snap("hist"), None
            if a.get("known") is not None:
                xp = R.blend_err(xp, snap("known"), snap("noise") if noise is not None else None, snap("mask"), cf)
            yield "latents", got("latents"), xp[0], xp[1]
            if a.get("lat_half_out") is not None:
                lh = got("lat_half_out")
                for c in range(copies):
                    yield f"lat_half_out[{c}]", lh[c * N:(c + 1) * N], xp[0], xp[1] + R.ulp(xp[0], hdt)
                if copies == 2:
                    yield "lat_half_out[1]", lh[N:], lh[:N], None
        return Spec("out_cfg_ddim" if copies == 2 else "out_ddim", o, check)
    return handler


def h_step_gather(be, a, hdt):
    n_rows = a["n_rows"]
    o = [dense("step_counter", a["step_counter"], (1,))]
    for i, (t, d) in enumerate(zip(a["tables"], a["dsts"])):
        o += [dense(f"table{i}", t, (n_rows, d.numel())), dense(f"dst{i}", d, (d.numel(),), "w")]

    def check(snap, got):
        snap = _whole(snap)
        r = max(0, min(int(snap("step_counter")[0]), n_rows - 1))
        for i in range(len(a["tables"])):
            yield f"dst{i}", got(f"dst{i}"), snap(f"table{i}")[r], None
    return Spec("step_gather", o, check)


def h_sam_relpos(be, a, hdt):
    B, heads, S, d = a["B"], a["heads"], a["S"], a["d"]
    q = a["q"]
    o = [Operand("q", q, (B, S * S, heads * d), (a["q_bs"], a["q_ns"], 1), q.storage_offset(), "r"),
         dense("Rh", a["Rh"], (S, S, d)), dense("Rw", a["Rw"], (S, S, d)),
         dense("rel_h", a["rel_h"], (B * heads, S * S, S), "w"), dense("rel_w", a["rel_w"], (B * heads, S * S, S), "w")]

    def check(snap, got):
        snap = _whole(snap)
        rh, rw, mh, mw = R.sam_relpos(snap("q").reshape(B, S * S, heads, d), snap("Rh"), snap("Rw"))
        yield "rel_h", got("rel_h"), rh, (d + 1) * U * mh
        yield "rel_w", got("rel_w"), rw, (d + 1) * U * mw
    return Spec("sam_relpos", o, check)


def _n_win(H, W_, ws):
    return -(-H // ws) * -(-W_ // ws)


def h_window_partition(be, a, hdt):
    B, H, W_, C, ws = a["B"], a["H"], a["W"], a["C_"], a["ws"]
    o = [dense("x", a["x"], (B, H, W_, C)), dense("out", a["out"], (B * _n_win(H, W_, ws), ws, ws, C), "w")]
    return Spec("window_partition", o,
                lambda snap, got: iter([("out", got("out"), R.window_partition(_d(snap("x")), ws), None)]))


def h_window_unpartition(be, a, hdt):
    B, H, W_, C, ws = a["B"], a["H"], a["W"], a["C_"], a["ws"]
    res = a.get("residual")
    o = [dense("xw", a["xw"], (B * _n_win(H, W_, ws), ws, ws, C))]
    if res is not None:
        o.append(dense("residual", res, (B, H, W_, C)))
    o.append(dense("out", a["out"], (B, H, W_, C), "w"))

    def check(snap, got):
        snap = _whole(snap)
        ref = R.window_unpartition(snap("xw"), B, H, W_, ws)
        if res is None:
            yield "out", got("out"), ref, None
        else:
            ref = ref + snap("residual")
            yield "out", got("out"), ref, 0.5 * R.ulp(ref, hdt) + U * ref.abs()
    return Spec("window_unpartition", o, check)


def h_sam_patchify(be, a, hdt):
    B, Cin, H, W_, ps = a["B"], a["Cin"], a["H"], a["W"], a["ps"]
    o = [dense("img", a["img"], (B, Cin, H, W_)),
         dense("out", a["out"], (B * (H // ps) * (W_ // ps), Cin * ps * ps), "w")]
    return Spec("sam_patchify", o,
                lambda snap, got: iter([("out", got("out"), R.sam_patchify(_d(snap("img")), ps), None)]))


def h_nhwc_to_nchw_f32(be, a, hdt):
    B, HW, C = a["B"], a["HW"], a["C_"]
    o = [dense("x", a["x"], (B, HW, C)), dense("out", a["out"], (B, C, HW), "w")]

    def check(snap, got):
        parts = [(b, p0, p1) for b in range(B) for p0, p1 in bands(HW, CHUNK_ELEMS // C)]
        for b, p0, p1 in parts:
            yield ("out" + _tag(parts, f"image {b} pixels {p0}-{p1 - 1}"), got("out")[b:b + 1, :, p0:p1],
                   R.nhwc_to_nchw(_d(snap("x")[b:b + 1, p0:p1])), None)
    return Spec("nhwc_to_nchw_f32", o, check)


def h_softmax_rows(be, a, hdt):
    r, c = a["rows"], a["cols"]
    o = [rows("s", a["s"], r, c, a.get("lds") or c), rows("p", a["p"], r, c, a.get("ldp") or c, "w")]

    def check(snap, got):
        parts = bands(r, CHUNK_ELEMS // c)
        for r0, r1 in parts:
            ref = R.softmax_rows(_d(snap("s")[r0:r1]))
            yield "p" + _tag(parts, f"rows {r0}-{r1 - 1}"), got("p")[r0:r1], ref, R.ulp(ref, hdt) + 1e-5 * ref.abs()
    return Spec("softmax_rows", o, check)


def h_image_out(be, a, hdt):
    B, HW, C, ldx = a["B"], a["HW"], a["C_"], a["ldx"]
    o = [Operand("x", a["x"], (B, HW, C), (HW * ldx, ldx, 1), a["x"].storage_offset(), "r"),
         dense("out", a["out"], (B, C, HW), "w")]
    sc = (a["scale"], a["shift"], a["lo"], a["hi"])

    def check(snap, got):
        parts = [(b, p0, p1) for b in range(B) for p0, p1 in bands(HW, CHUNK_ELEMS // C)]
        for b, p0, p1 in parts:
            yield ("out" + _tag(parts, f"image {b} pixels {p0}-{p1 - 1}"), got("out")[b:b + 1, :, p0:p1],
                   R.image_out(_d(snap("x")[b:b + 1, p0:p1]), C, *sc), None)
    return Spec("image_out", o, check)


HANDLERS = {"gemm": h_gemm, "gemm_grouped": h_gemm_grouped, "attention": h_attention, "groupnorm": h_groupnorm,
            "layernorm": h_layernorm, "conv_direct": h_conv_direct, "conv_in": h_conv_in, "upsample2x": h_upsample2x,
            "small_linear": h_small_linear, "timestep_embedding": h_timestep_embedding,
            "out_cfg_ddim": _h_out(2), "out_ddim": _h_out(1), "step_gather": h_step_gather,
            "sam_relpos": h_sam_relpos, "window_partition": h_window_partition,
            "window_unpartition": h_window_unpartition, "sam_patchify": h_sam_patchify,
            "nhwc_to_nchw_f32": h_nhwc_to_nchw_f32, "softmax_rows": h_softmax_rows, "image_out": h_image_out}


# ================================================ the auditor ===================================================
def _tensors(obj):
    if torch.is_tensor(obj):
        yield obj
    elif isinstance(obj, (list, tuple)):
        for x in obj:
            yield from _tensors(x)
    elif isinstance(obj, dict):
        for x in obj.values():
            yield from _tensors(x)


def _remap(obj, new):
    if torch.is_tensor(obj):
        flat, shift = new[_key(obj)]
        return torch.as_strided(flat, obj.shape, obj.stride(), obj.storage_offset() + shift)
    if isinstance(obj, list):
        return [_remap(x, new) for x in obj]
    if isinstance(obj, tuple):
        return tuple(_remap(x, new) for x in obj)
    if isinstance(obj, dict):
        return {k: _remap(x, new) for k, x in obj.items()}
    return obj


def _call_site():
    """file:line of the innermost product frame that called the operator table."""
    for fr in reversed(traceback.extract_stack()):
        f = fr.filename.replace(os.sep, "/")
        if "/editanything_b200/" in f and not f.endswith("/ops.py"):
            return f"{f.rsplit('/', 1)[-1]}:{fr.lineno}"
    return "test"


class Snapshot:
    """The pre-call state a call is judged against: every storage the call writes, whole (the out-of-extent check
    needs all of it), and only the declared extents of the operands on storages it merely reads."""

    def __init__(self, spec, storages, written):
        self.whole = {k: _flat(storages[k]).clone() for k in written}
        self.part = {o.name: o.view(_flat(o.t)).clone() for o in spec.operands if _key(o.t) not in written}

    def pre(self, o):
        k = _key(o.t)
        return o.view(self.whole[k]) if k in self.whole else self.part[o.name]


# the argument an operator returns (the ops.* functions return their destination; None where there is none)
RETURNS = {"small_linear": "y", "softmax_rows": "p", "out_cfg_ddim": None, "out_ddim": None, "step_gather": None,
           "sam_relpos": None}


class Auditor:
    """Operator table wrapper (see the module docstring).  case: a name for failure messages; skip_production: run
    only the fenced copy and write its outputs back (a store past a storage then lands in an allocated margin)."""

    def __init__(self, backend, case="", skip_production=False, fence=True):
        self.be, self.case, self.skip_production, self.fence = backend, case, skip_production, fence
        self.calls = 0          # audited launches
        self.other = 0          # calls of operator-table entries that launch nothing
        self.enabled = True     # False: forward launches unchecked (auditing chosen layers of a large network)
        self.unaudited = 0
        self.worst = {}
        self.worst_unit = {}    # GroupNorm: worst error / the bound without the derived statistics term
        self.counts = {}
        # CUDA only: the device's peak allocation over the audited calls (the auditor resets the peak statistics at
        # every call, so a caller reads max(this, torch.cuda.max_memory_allocated())), and the largest growth during
        # one call over what was allocated when it started: the auditor's own snapshots, copies and references
        self.peak_bytes = 0
        self.own_peak_bytes = 0

    def __getattr__(self, name):
        fn = getattr(self.be, name)
        if not callable(fn) or isinstance(fn, type):
            return fn
        if name in PASSTHROUGH:
            def other(*args, **kw):
                self.other += 1
                return fn(*args, **kw)
            return other
        handler = HANDLERS.get(name)
        if handler is None:
            raise AuditError(f"{self.case}: ops.{name} has no audit handler")

        def call(*args, **kw):
            if not self.enabled:            # a stretch the caller chose not to audit
                self.unaudited += 1
                return fn(*args, **kw)
            sig = inspect.signature(fn)
            bound = sig.bind(*args, **kw)
            bound.apply_defaults()
            a = dict(bound.arguments)
            for n, p in sig.parameters.items():      # a wrapper's **kwargs: its keywords as they were passed
                if p.kind == p.VAR_KEYWORD:
                    a.update(a.pop(n, {}))
                    for k, q in inspect.signature(getattr(cpu_ops, name)).parameters.items():
                        if q.default is not q.empty:
                            a.setdefault(k, q.default)
            return self._audit(name, fn, handler, a)
        return call

    # -------------------------------------------------------------------------------------------------------
    def _fail(self, where, operand, msg):
        raise AuditError(f"{self.case}: call {where[2]} ops.{where[0]} at {where[1]}, operand {operand}: {msg}")

    def _audit(self, name, fn, handler, a):
        dev = next(iter(_tensors(a))).device
        if dev.type != "cuda":
            return self._audit_call(name, fn, handler, a)
        self.peak_bytes = max(self.peak_bytes, torch.cuda.max_memory_allocated(dev))
        torch.cuda.reset_peak_memory_stats(dev)
        base = torch.cuda.memory_allocated(dev)
        r = self._audit_call(name, fn, handler, a)
        peak = torch.cuda.max_memory_allocated(dev)
        self.peak_bytes = max(self.peak_bytes, peak)
        self.own_peak_bytes = max(self.own_peak_bytes, peak - base)
        return r

    def _audit_call(self, name, fn, handler, a):
        hdt = self.be.half_dtype()
        spec = handler(self.be, a, hdt)            # may fill in an output the operator would allocate itself
        self.calls += 1
        where = (name, _call_site(), self.calls + self.other + self.unaudited)    # position in the operator trace
        tens = list(_tensors(a))
        dev = tens[0].device
        storages = {}
        for t in tens:
            storages.setdefault(_key(t), t)
        for o in spec.operands:
            storages.setdefault(_key(o.t), o.t)
        written = {}
        for o in spec.operands:
            if o.writes:
                k = _key(o.t)
                if k not in written:
                    written[k] = torch.zeros(_flat(o.t).numel(), dtype=torch.bool, device=dev)
                o.view(written[k]).fill_(True)
        _sync(dev)
        # the snapshot: whole storages of written operands, the declared extents of read-only ones
        snap = Snapshot(spec, storages, written)
        gws = self.be.gemm_workspace(dev) if name.startswith("gemm") and hasattr(self.be, "gemm_workspace") else None

        if not self.skip_production:
            fn(**a)
            _sync(dev)
            for k, m in written.items():               # writes stay inside the declared extents
                bad = (_bits(_flat(storages[k])) != _bits(snap.whole[k])) & ~m
                if bool(bad.any()):
                    i = int(torch.nonzero(bad)[0])
                    names = [o.name for o in spec.operands if _key(o.t) == k]
                    self._fail(where, "/".join(names), f"wrote element {i} of its storage outside the declared "
                                                       f"extent ({int(bad.sum())} elements)")
            self._side_checks(spec, lambda o: o.view(_flat(storages[_key(o.t)])), gws, where, "")
        if self.fence or self.skip_production:
            fenced = self._fenced(fn, a, spec, storages, snap, written, where, gws)
            if self.skip_production:
                for k, (flat, shift) in fenced.items():     # hand the results to the engine as production would
                    if k in written:
                        m = written[k]
                        dst = _flat(storages[k])
                        dst[m] = flat[shift:shift + dst.numel()][m]
                _sync(dev)
            else:
                for k, (flat, shift) in fenced.items():
                    if k in written:
                        prod = _flat(storages[k])
                        m = written[k]
                        d = _bits(flat[shift:shift + prod.numel()][m]) != _bits(prod[m])
                        if bool(d.any()):
                            names = [o.name for o in spec.operands if _key(o.t) == k and o.writes]
                            self._fail(where, "/".join(names), f"the fenced re-run differs from the production run "
                                                               f"in {int(d.sum())} elements: a read outside the "
                                                               f"declared operands reaches the result"
                                                               + self._culprit(fn, a, spec, storages, snap, written))
            del fenced
        del written
        self._check(spec, snap, storages, where)
        key = where[:2]
        if hasattr(spec, "unit_worst"):
            self.worst_unit[key] = max(self.worst_unit.get(key, 0.0), spec.unit_worst[0])
        self.counts[key] = self.counts.get(key, 0) + 1
        if name == "gemm":
            return a["out"] if a.get("out") is not None else a["out_f32"]
        if name == "gemm_grouped":
            return [c[2] if c[2] is not None else c[3]["out_f32"] for c in a["calls"]]
        return a.get(RETURNS.get(name, "out"))       # what the operator returns: its destination argument

    def _side_checks(self, spec, view, gws, where, which):
        if gws is not None and bool(gws[:GEMM_WS_COUNTER_BYTES].ne(0).any()):
            self._fail(where, "gemm workspace", f"split-K counters not zero after the {which}call")
        if spec.after is not None:
            by_name = {o.name: o for o in spec.operands}
            for operand, msg in spec.after(lambda n: view(by_name[n])):
                self._fail(where, operand, f"{msg} ({which or 'production '}run)")

    def _check(self, spec, snap, storages, where):
        ops_ = {o.name: o for o in spec.operands}
        key = where[:2]

        def s(n):
            return snap.pre(ops_[n])

        def g(n):
            o = ops_[n]
            return o.view(_flat(storages[_key(o.t)]))
        for operand, got, ref, bound in spec.check(s, g):
            if bound is None:
                want = ref.to(got.dtype)
                same = _bits(got) == _bits(want) if got.is_floating_point() else got == want
                if not bool(same.all()):
                    i = int(torch.nonzero(~same.reshape(-1))[0])
                    ix = tuple(int(v) for v in np.unravel_index(i, tuple(got.shape)))
                    self._fail(where, operand, f"{int((~same).sum())} of {got.numel()} elements not bit-exact; first "
                                               f"at {ix}: got {float(got.reshape(-1)[i])!r}, ref "
                                               f"{float(want.reshape(-1)[i])!r}")
                self.worst.setdefault(key, 0.0)
                continue
            worst, i, n_bad = R.worst_element(got, ref, bound)
            self.worst[key] = max(self.worst.get(key, 0.0), worst)
            if not worst <= 1.0:
                ix = tuple(int(v) for v in np.unravel_index(i, tuple(ref.shape)))
                self._fail(where, operand, f"{n_bad} of {ref.numel()} elements out of bound; worst at {ix}: got "
                                           f"{float(got.reshape(-1)[i])!r}, ref {float(ref.reshape(-1)[i])!r}, bound "
                                           f"{float(bound.reshape(-1)[i]):.3e} (ratio {worst:.3g})")

    # -------------------------------------------------------------------------------------------------------
    def _relocate(self, spec, storages, snap, fence_keys):
        """Fresh copies of every storage inside 0xFF (NaN) margins: those in fence_keys NaN outside their read
        extents, the others (and integer and scratch storages) with their whole content.  Returns
        {key: (flat, shift in elements)}."""
        new = {}
        for k, t in storages.items():
            es = t.element_size()
            ld = max([o.stride[-2] if len(o.stride) > 1 else 0 for o in spec.operands if _key(o.t) == k] + [0])
            mb = max(MARGIN_BYTES, MARGIN_ROWS * ld * es)
            mb = -(-mb // 4096) * 4096
            n = _flat(t).numel()
            flat = torch.full((2 * mb + n * es,), 0xFF, dtype=torch.uint8, device=t.device).view(t.dtype)
            shift = mb // es
            scratch = any(o.role == "scratch" for o in spec.operands if _key(o.t) == k)
            if k not in fence_keys or not t.is_floating_point() or scratch:
                # a read-only storage is unchanged by a call that passed the checks: its live content is its snapshot
                flat[shift:shift + n].copy_(snap.whole[k] if k in snap.whole else _flat(t))
            else:
                for o in spec.operands:
                    if _key(o.t) == k and o.reads:
                        o.view(flat, shift).copy_(snap.pre(o))
            new[k] = (flat, shift)
        return new

    def _run_relocated(self, fn, a, new, dev):
        kw = _remap(a, new)
        fn(**kw)
        _sync(dev)

    def _fenced(self, fn, a, spec, storages, snap, written, where, gws):
        dev = next(iter(storages.values())).device
        new = self._relocate(spec, storages, snap, set(storages))
        image = {k: flat.clone() for k, (flat, _) in new.items()}
        _sync(dev)
        self._run_relocated(fn, a, new, dev)
        for k, (flat, shift) in new.items():
            n = flat.numel() - 2 * shift
            m = torch.zeros(flat.numel(), dtype=torch.bool, device=dev)
            if k in written:
                m[shift:shift + n] = written[k]
            bad = (_bits(flat) != _bits(image[k])) & ~m
            if bool(bad.any()):
                i = int(torch.nonzero(bad)[0]) - shift
                names = [o.name for o in spec.operands if _key(o.t) == k]
                side = "before its storage" if i < 0 else "past its storage" if i >= n else "inside its storage"
                self._fail(where, "/".join(names), f"the fenced re-run wrote element {i} ({side}) outside the declared "
                                                   f"extent ({int(bad.sum())} elements)")
        del image
        self._side_checks(spec, lambda o: o.view(*new[_key(o.t)]), gws, where, "fenced ")
        return new

    def _culprit(self, fn, a, spec, storages, snap, written):
        """Re-runs with one storage fenced at a time: names the operands whose storage is read outside its extent."""
        dev = next(iter(storages.values())).device
        full = self._relocate(spec, storages, snap, set())
        self._run_relocated(fn, a, full, dev)
        out = []
        for k, t in storages.items():
            if not t.is_floating_point():
                continue
            new = self._relocate(spec, storages, snap, {k})
            self._run_relocated(fn, a, new, dev)
            for kw_, m in written.items():
                (f1, s1), (f0, s0) = new[kw_], full[kw_]
                n = m.numel()
                if bool((_bits(f1[s1:s1 + n][m]) != _bits(f0[s0:s0 + n][m])).any()):
                    out.append("/".join(o.name for o in spec.operands if _key(o.t) == k))
                    break
        return f" (read outside the declared extent of: {', '.join(out)})" if out else ""

    def report(self, title=""):
        lines = [f"worst error / bound per (op, call site){' - ' + title if title else ''}:"]
        for (op, site), v in sorted(self.worst.items()):
            lines.append(f"  {op:20s} {site:18s} {v:.3f}  ({self.counts.get((op, site), 0)} launches)")
        return "\n".join(lines)


# ================================================ engine drivers ================================================
def denoise_engine(name, backend, device):
    """The DenoiseEngine of test_step_trace_cpu.CASES[name] (its EA_* switches already set) on `backend`, and the
    inputs of that case: (engine, x, ctx, hints, scales, guess mode)."""
    from editanything_b200.denoise import DenoiseEngine
    from editanything_b200.unet_spec import TINY21, TINY21_INPAINT, make_state_dict
    from oracle.inputs import make_inputs
    from tests.test_step_trace_cpu import CASES
    cfg, n_cn, _, scales, guess = CASES[name]
    usd = make_state_dict(cfg, "unet", 61)
    csds = [make_state_dict(TINY21 if cfg is TINY21_INPAINT else cfg, "controlnet", 62 + i) for i in range(n_cn)]
    x, ctx, hints = make_inputs(cfg, 2, 8, 7, 5, n_controlnets=2)
    hints = (hints + [hints[0].flip(-1), hints[1].flip(-2)])[:n_cn]
    scales = [torch.rand(8, 8, generator=torch.Generator().manual_seed(9)) if s == "map" else s for s in scales]
    eng = DenoiseEngine(cfg, usd, csds, device, backend=backend)
    return eng, x, ctx, hints, scales, guess


def run_trace_case(eng, x, ctx, hints, scales, guess, unipc_steps=0):
    """The calls of tests/test_step_trace_cpu.record(): prepare, (set_unet_condition), one DDIM step without a graph,
    one eps(); with unipc_steps > 0 that many UniPC steps of a 20-step schedule instead of the DDIM step, so that the
    multistep history is live."""
    from editanything_b200.denoise import ddim_schedule
    ts, a, ap = ddim_schedule(50)
    eng.prepare(ctx, hints, scales, guess_mode=guess)
    if eng.cfg.in_channels == 9:
        eng.set_unet_condition(x[:1, 4:5], x[:1, 5:9])
    eng.begin(x[:1, :4], guidance=7.5, use_graph=False)
    if unipc_steps:
        set_unipc(eng, 20)
        for _ in range(unipc_steps):
            eng.step()
    else:
        eng.step(int(ts[2]), float(a[2]), float(ap[2]))
    eng.eps(x, int(ts[5]))


def set_unipc(eng, n, prediction_type="epsilon"):
    from editanything_b200.pipeline import DDIMScheduler
    from editanything_b200.schedulers import UniPCMultistepScheduler
    sched = UniPCMultistepScheduler.from_config(DDIMScheduler().config, solver_order=2)
    sched.set_timesteps(n)
    ts = sched.timesteps.tolist()
    eng.set_schedule(ts, [float(sched.alphas_cumprod[t]) for t in ts], [1.0] * len(ts),
                     multistep=sched.coefficient_rows(), prediction_type=prediction_type)
