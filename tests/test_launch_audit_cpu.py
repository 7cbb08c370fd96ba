"""The launch auditor (tests/launch_audit.py) itself, on the CPU emulation tests/cpu_ops.py: every operator the engines
call has a handler, every check passes on a correct backend, and each injected fault is reported with its op and
operand."""
import json
import types

import pytest
import torch

from editanything_b200.sam import SAM_TINY, SamEncoderEngine, make_sam_state_dict
from editanything_b200.vae import VAE_TINY, VaeDecoderEngine, VaeEncoderEngine, make_vae_state_dict
from tests import cpu_ops
from tests import launch_audit as LA
from tests import fp64_refs as R
from tests.launch_audit import AuditError, Auditor, _flat, denoise_engine, run_trace_case
from tests.test_step_trace_cpu import CASES, GOLDEN, _set_env

CPU = torch.device("cpu")


@pytest.mark.parametrize("name", list(CASES))
def test_every_call_of_the_step_trace_is_audited(name, monkeypatch):
    _set_env(monkeypatch, name)
    aud = Auditor(cpu_ops, name)
    eng, *inputs = denoise_engine(name, aud, CPU)
    aud.calls = aud.other = 0
    run_trace_case(eng, *inputs)
    with open(GOLDEN) as f:
        want = sum(s["calls"] for s in json.load(f)[name].values())
    assert aud.calls + aud.other == want, (aud.calls, aud.other, want)
    assert aud.calls > 0 and len(aud.worst) > 0


def test_sam_and_vae_are_audited():
    aud = Auditor(cpu_ops, "sam_tiny")
    sd = make_sam_state_dict(SAM_TINY, 5)
    SamEncoderEngine(SAM_TINY, sd, CPU, backend=aud)._encode_eager(torch.randn(2, 3, 256, 256))
    assert aud.calls > 4 * SAM_TINY.depth
    for part, Eng, x in (("decoder", VaeDecoderEngine, torch.randn(3, 4, 6, 6)),
                         ("encoder", VaeEncoderEngine, torch.rand(3, 3, 24, 24) * 2 - 1)):
        aud = Auditor(cpu_ops, f"vae_tiny_{part}")
        eng = Eng(VAE_TINY, make_vae_state_dict(VAE_TINY, 7, part=part), CPU, backend=aud)
        if part == "decoder":
            eng.decode_latents(x, use_graph=False)
        else:
            eng.encode(x, use_graph=False)
        assert aud.calls > 10


def test_unknown_operator_fails():
    be = types.SimpleNamespace(half_dtype=cpu_ops.half_dtype, new_kernel=lambda x: x)
    with pytest.raises(AuditError, match="new_kernel has no audit handler"):
        Auditor(be, "t").new_kernel(1)


# ---- injected faults ------------------------------------------------------------------------------------------
def _backend(**over):
    """cpu_ops with some entries replaced."""
    ns = types.SimpleNamespace(**{k: getattr(cpu_ops, k) for k in dir(cpu_ops) if not k.startswith("__")})
    for k, v in over.items():
        setattr(ns, k, v)
    return ns


def _linear_case(M=40, N=32, K=64, seed=0):
    g = torch.Generator().manual_seed(seed)
    a = torch.randn(M, K, generator=g)
    w = torch.randn(N, K, generator=g) / 8
    bias = torch.randn(N, generator=g)
    return a, w, bias


def _expect(be, fn, op, operand):
    with pytest.raises(AuditError) as exc:
        fn(Auditor(be, "fault"))
    msg = str(exc.value)
    named = msg.split("operand ", 1)[1].split(":", 1)[0].split(" [", 1)[0]      # without the band
    assert f"ops.{op} " in msg and operand in named.split("/"), msg
    return msg


def test_fault_write_one_row_past_out():
    a, w, bias = _linear_case()
    M, N = 40, 32

    def gemm(a, w, out=None, **kw):
        r = cpu_ops.gemm(a, w, out, **kw)
        _flat(out)[out.storage_offset() + M * out.stride(0)] = 1.0
        return r
    buf = torch.zeros(M + 4, N)
    msg = _expect(_backend(gemm=gemm), lambda o: o.gemm(a, w, buf[:M], bias=bias), "gemm", "out")
    assert "outside the declared extent" in msg


def test_fault_store_past_the_storage_lands_in_the_fence():
    """A store one row past an output allocated with exactly M rows: only the fenced re-run's margin can see it, so
    the production run is skipped and every stray store lands in memory the auditor allocated."""
    a, w, bias = _linear_case()
    M = a.shape[0]

    def gemm(a, w, out=None, **kw):
        r = cpu_ops.gemm(a, w, out, **kw)
        _flat(out)[out.storage_offset() + M * out.stride(0)] = 1.0
        return r
    with pytest.raises(AuditError) as exc:
        Auditor(_backend(gemm=gemm), "fence", skip_production=True).gemm(a, w, bias=bias)
    msg = str(exc.value)
    assert "operand out:" in msg and "past its storage" in msg, msg


def test_fault_ldo2_ignored():
    a, w, bias = _linear_case()
    M, N = 40, 32

    def gemm(a, w, out=None, out2=None, ldo=None, ldo2=None, **kw):
        r = cpu_ops.gemm(a, w, out, ldo=ldo, **kw)
        torch.as_strided(out2, (M, N), (ldo or out.stride(0), 1)).copy_(out)      # out2 stored at ldo
        return r
    cat = torch.zeros(M, 3 * N)
    o2 = torch.zeros(2 * M, 2 * N)          # room below the slot for the misplaced rows
    msg = _expect(_backend(gemm=gemm),
                  lambda o: o.gemm(a, w, cat[:, N:2 * N], bias=bias, out2=o2[:M, :N], ldo=3 * N, ldo2=2 * N),
                  "gemm", "out2")
    assert "out2" in msg


def test_fault_last_row_reads_next_rowvec():
    B, H, W_, cin, cout = 3, 4, 4, 64, 32
    g = torch.Generator().manual_seed(1)
    x = torch.randn(B, H, W_, cin, generator=g)
    w = torch.randn(cout, 9 * cin, generator=g) / 24
    table = torch.randn(B + 1, 3 * cout, generator=g)
    rv = table[:B, cout:2 * cout]

    def gemm(a, w, out=None, rowvec=None, **kw):
        r = cpu_ops.gemm(a, w, out, rowvec=rowvec, **kw)
        nxt = torch.as_strided(rowvec, (cout,), (1,), rowvec.storage_offset() + B * rowvec.stride(0))
        out[-1] += nxt - rowvec[B - 1]              # the last row took rowvec[b + 1]
        return r
    out = torch.zeros(B * H * W_, cout)
    msg = _expect(_backend(gemm=gemm), lambda o: o.gemm(x, w, out, mode=1, conv=(B, H, W_, cin), rowvec=rv),
                  "gemm", "out")
    assert "rowvec" in msg


def test_fault_one_element_twice_its_bound():
    a, w, bias = _linear_case()
    K = a.shape[1]
    ad, wd = a.double(), w.double()
    ref = ad @ wd.T + bias.double()
    bound = (K + 2) * R.U32 * (ad.abs() @ wd.abs().T + bias.double().abs()) + R.ulp(ref, torch.float32)

    def gemm(a, w, out=None, **kw):
        r = cpu_ops.gemm(a, w, out, **kw)
        out[7, 5] = float(ref[7, 5] + 2 * bound[7, 5])
        return r
    out = torch.zeros(40, 32)
    msg = _expect(_backend(gemm=gemm), lambda o: o.gemm(a, w, out, bias=bias), "gemm", "out")
    assert "worst at (7, 5)" in msg and 1.9 < float(msg.rsplit("ratio ", 1)[1].rstrip(")")) < 2.1, msg


def test_fault_groupnorm_reads_x2_at_ldx():
    B, HW, C1, C2 = 2, 16, 64, 64
    g = torch.Generator().manual_seed(2)
    b1 = torch.randn(B * HW, C1 + 32, generator=g)
    b2 = torch.randn(B * HW, C2 + 96, generator=g)
    gam, bet = torch.randn(C1 + C2, generator=g), torch.randn(C1 + C2, generator=g)

    def groupnorm(x, gamma, beta, out, *, x2=None, ldx=None, ldx2=None, **kw):
        x2 = torch.as_strided(x2, (B * HW, C2), (ldx, 1), x2.storage_offset())
        return cpu_ops.groupnorm(x, gamma, beta, out, x2=x2, ldx=ldx, ldx2=ldx2, **kw)
    out = torch.zeros(B * HW, C1 + C2)
    msg = _expect(_backend(groupnorm=groupnorm),
                  lambda o: o.groupnorm(b1[:, :C1], gam, bet, out, B=B, HW=HW, C_=C1 + C2, x2=b2[:, :C2], C1=C1,
                                        ldx=C1 + 32, ldx2=C2 + 96, workspace=cpu_ops.gn_workspace(B, CPU)),
                  "groupnorm", "out")
    assert "x2" in msg


def test_correct_backend_passes_the_fault_setups():
    """The same calls on the unmodified emulation pass every check."""
    a, w, bias = _linear_case()
    aud = Auditor(cpu_ops, "clean")
    aud.gemm(a, w, torch.zeros(44, 32)[:40], bias=bias)
    cat, o2 = torch.zeros(40, 96), torch.zeros(40, 64)
    aud.gemm(a, w, cat[:, 32:64], bias=bias, out2=o2[:, :32], ldo=96, ldo2=64)
    B, HW = 2, 16
    g = torch.Generator().manual_seed(2)
    b1, b2 = torch.randn(B * HW, 96, generator=g), torch.randn(B * HW, 160, generator=g)
    aud.groupnorm(b1[:, :64], torch.ones(128), torch.zeros(128), torch.zeros(B * HW, 128), B=B, HW=HW, C_=128,
                  x2=b2[:, :64], C1=64, ldx=96, ldx2=160, workspace=cpu_ops.gn_workspace(B, CPU))
    assert aud.calls == 3


def test_skip_production_hands_back_results_and_destinations():
    """With the production run skipped, the fenced run's outputs land in the caller's tensors and every operator
    returns what it returns unaudited (its destination)."""
    g = torch.Generator().manual_seed(3)
    x = torch.randn(8, 64, generator=g)
    gam, bet = torch.rand(64, generator=g) + 0.5, torch.randn(64, generator=g)
    out = torch.zeros(8, 64)
    aud = Auditor(cpu_ops, "skip", skip_production=True)
    r = aud.layernorm(x, gam, bet, out, M=8, C_=64)
    assert r is out and torch.equal(out, cpu_ops.layernorm(x, gam, bet, torch.zeros(8, 64), M=8, C_=64))
    y = aud.gemm(x, torch.randn(32, 64, generator=g) / 8)
    assert y.shape == (8, 32) and torch.isfinite(y).all()


# ---- bounded-memory references: the banded float64 side equals the whole-operand one ----------------------------
BIG = 1 << 40          # CHUNK_ELEMS at which every reference is built in one band


def _yields(monkeypatch, chunk, name, **a):
    """(operand, ref, bound) the check of ops.<name>(**a) yields with CHUNK_ELEMS = chunk, judged against the
    operands as they are (the call itself is not run)."""
    monkeypatch.setattr(LA, "CHUNK_ELEMS", chunk)
    spec = LA.HANDLERS[name](cpu_ops, a, cpu_ops.half_dtype())
    ops_ = {o.name: o for o in spec.operands}
    view = lambda n: ops_[n].view(_flat(ops_[n].t))
    return [(op, ref, bound) for op, _, ref, bound in spec.check(view, view)]


def _cat(ys, width):
    return (torch.cat([r.reshape(-1, width) for _, r, _ in ys]),
            torch.cat([b.reshape(-1, width) for _, _, b in ys]))


def _same(got, want, scale):
    """Equal to within 1e-12 of `scale` (the magnitude the value is a rounded sum of) per element."""
    assert got.shape == want.shape
    assert bool(((got - want).abs() <= 1e-12 * scale).all()), float(((got - want).abs() / scale).max())


MODES = {"s1": LA.CONV_S1, "s2": LA.CONV_S2, "s2a": LA.CONV_S2A}


def _conv_case(md, extra, B=2, H=7, W_=5, cin=16, cout=8, seed=4):
    g = torch.Generator().manual_seed(seed)
    s = 1 if md == "s1" else 2
    x = torch.randn(B, s * H, s * W_, cin, generator=g)
    ce = 12 if extra else 0
    w = torch.randn(cout, 9 * cin + ce, generator=g) / 12
    xe = torch.randn(B, H, W_, ce, generator=g) if extra else None
    return x, w, xe


@pytest.mark.parametrize("md", list(MODES))
@pytest.mark.parametrize("extra", [False, True])
@pytest.mark.parametrize("per", [1, 2, 3, 7])
def test_conv_band_equals_whole_image_rows(md, extra, per):
    """conv_gemm_rows on output rows [y0, y1) = R.conv_gemm of the whole image on those rows, H = 7 not a multiple
    of the band."""
    x, w, xe = _conv_case(md, extra)
    wd = w.double()
    ref, mag = R.conv_gemm(x.double(), wd, md, xe.double() if extra else None)
    for y0, y1 in LA.bands(7, per):
        pre, m = LA.conv_gemm_rows(x, wd, MODES[md], y0, y1, xe)
        _same(pre, ref[:, y0:y1], mag[:, y0:y1])
        _same(m, mag[:, y0:y1], mag[:, y0:y1])


@pytest.mark.parametrize("md", list(MODES))
@pytest.mark.parametrize("extra", [False, True])
def test_banded_conv_gemm_check_matches_unbanded(md, extra, monkeypatch):
    """The gemm handler's reference and bound with one output row per band against the whole-image float64 path
    (R.conv_gemm, the activation, the epilogue) - bias, SiLU, and a residual where there is no folded skip."""
    B, H, W_, cout = 2, 7, 5, 8
    x, w, xe = _conv_case(md, extra)
    g = torch.Generator().manual_seed(5)
    bias = torch.randn(cout, generator=g)
    res = None if extra else torch.randn(B * H * W_, cout, generator=g)
    kw = dict(mode=MODES[md], conv=(B, H, W_, x.shape[-1]), bias=bias, act=1)
    if extra:
        kw.update(a_extra=xe, ld_extra=xe.shape[-1])
    else:
        kw["residual"] = res
    out = torch.zeros(B * H * W_, cout)
    banded = _yields(monkeypatch, 1, "gemm", a=x, w=w, out=out, **kw)
    assert len(banded) == B * H and banded[H][0] == "out [image 1 rows 0-0]"
    ref, bound = _cat(banded, cout)
    one = _yields(monkeypatch, BIG, "gemm", a=x, w=w, out=out, **kw)
    assert [op for op, _, _ in one] == ["out [image 0 rows 0-6]", "out [image 1 rows 0-6]"]     # one band per image
    pre, mag = R.conv_gemm(x.double(), w.double(), md, xe.double() if extra else None)
    pre, mag = pre.reshape(-1, cout) + bias.double(), mag.reshape(-1, cout) + bias.double().abs()
    y, err = R.gemm_act("silu", pre, (9 * x.shape[-1] + (12 if extra else 0) + 2) * R.U32 * mag)
    want, want_b = R.gemm_out(y, err, 1.0, [] if extra else [res.double()], cpu_ops.half_dtype(), 0)
    for r, b in ((ref, bound), _cat(one, cout)):
        _same(r, want, mag)
        _same(b, want_b, want_b)


def _gn_case(B, HW, C, C1, seed=6):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B * HW, (C1 or C) + 8, generator=g) * 2 + 3          # an offset mean: the merge must carry it
    x2 = torch.randn(B * HW, C - C1 + 16, generator=g) if C1 else None
    return x, x2, g


def _gn_stats_excess(x, gam, groups, eps):
    """R.gn_stats_excess on the whole tensor x [B, HW, C] (132 SMs, as the auditor assumes off the GPU)."""
    B, HW, C = x.shape
    cpg = C // groups
    d_mean, d_rstd, r = R.gn_stats_bound(x, groups, eps, 132)
    xg = x.reshape(B, HW, groups, cpg)
    yn = ((xg - xg.mean(dim=(1, 3), keepdim=True)) * r[:, None, :, None]).reshape(B, HW, C)
    g = torch.stack([t.double() for t in gam]).repeat_interleave(B // len(gam), dim=0)[:, None, :]
    ch = lambda t: t.repeat_interleave(cpg, dim=1)[:, None, :]
    return R.gn_stats_excess(yn, g, ch(r), ch(d_mean), ch(d_rstd), LA.NORM_K * R.U32)


def _kernel_walk(x, groups, n_sm):
    """ea_groupnorm's statistics summed in fp32 exactly as ea_pointwise.cu's loops do, written from the kernel's
    index arithmetic (not from R.gn_geometry): per image, CTA blockIdx.x covers pixels [x ppc, (x + 1) ppc); thread
    (pl, v) adds d = x - k of pixels p0 + pl, p0 + pl + lanes, ...; thread (g, which) adds part[l][g cpg + j] for
    l < lanes, j < cpg; thread pidx < parts adds the CTA slots pidx, pidx + parts, ...; thread i adds the parts.
    Also counts the longest chain of additions.  Returns (S1, S2 [B, groups] float32, chain length)."""
    B, HW, C = x.shape
    cpg = C // groups
    chunks = min(n_sm // B, HW)
    ppc = (HW + chunks - 1) // chunks
    chunks = (HW + ppc - 1) // ppc
    nvec = C // 8
    threads = min(512, ((512 // nvec) * nvec + 31) // 32 * 32)
    lanes = threads // nvec
    g2 = 2 * groups
    parts = max(1, min(threads // g2, ((lanes * 2 * C * 4 + 15) & ~15) // (g2 * 4)))
    xf = x.float()
    k = xf[:, 0, ::cpg].repeat_interleave(cpg, dim=1)                      # [B, C]
    out = torch.zeros(B, 2, groups)
    longest = 0
    for b in range(B):
        slots = torch.zeros(chunks, 2, groups)
        for blk in range(chunks):
            p0, p1 = blk * ppc, min(HW, (blk + 1) * ppc)
            cs = torch.zeros(lanes, C)
            cq = torch.zeros(lanes, C)
            n_thread = 0
            for t in range(0, p1 - p0, lanes):                              # every lane's next pixel
                rows = torch.arange(t, min(t + lanes, p1 - p0))
                d = xf[b, p0 + rows] - k[b]
                cs[rows - t] = cs[rows - t] + d
                cq[rows - t] = cq[rows - t] + d * d
                n_thread += 1
            acc = torch.zeros(2, groups)
            for l in range(lanes):
                for j in range(cpg):
                    acc[0] = acc[0] + cs[l, j::cpg]
                    acc[1] = acc[1] + cq[l, j::cpg]
            slots[blk] = acc
            longest = max(longest, n_thread + lanes * cpg)
        pacc = torch.zeros(parts, 2, groups)
        for pidx in range(parts):
            for cidx in range(pidx, chunks, parts):
                pacc[pidx] = pacc[pidx] + slots[cidx]
        tot = torch.zeros(2, groups)
        for q in range(parts):
            tot = tot + pacc[q]
        out[b] = tot
    return out[:, 0], out[:, 1], longest + -(-chunks // parts) + parts


@pytest.mark.parametrize("B,HW,C", [(1, 3000, 256), (1, 1700, 128), (4, 1500, 320), (2, 700, 64)])
def test_groupnorm_statistics_bound_holds_for_the_kernel_order(B, HW, C):
    """The running bound R.gn_stats_err on ea_groupnorm's statistics holds for the sums done in fp32 in the kernel's
    order (_kernel_walk, an independent walk of its loops), at B = 1 and B = 4 lockstep geometries, on data whose
    groups sit well off their shift so that the rounding is large; R.gn_geometry matches the walk's geometry."""
    groups, eps, n_sm = 32, 1e-6, 132
    g = torch.Generator().manual_seed(B * HW + C)
    x = (torch.randn(B, HW, C, generator=g) * 0.5 + 3 + torch.randn(B, 1, C, generator=g)).half().double()
    s1, s2, chain = _kernel_walk(x, groups, n_sm)
    chunks, ppc, lanes, parts = R.gn_geometry(B, HW, C, groups, n_sm)
    assert chain == -(-ppc // lanes) + lanes * (C // groups) + -(-chunks // parts) + parts
    cpg = C // groups
    n = HW * cpg
    xg = x.reshape(B, HW, groups, cpg)
    k = xg[:, 0, :, 0]
    dk = xg - k[:, None, :, None]
    md, q = dk.mean(dim=(1, 3)), (dk * dk).mean(dim=(1, 3))
    var = xg.var(dim=(1, 3), correction=0)
    # the kernel's mean and rstd from its fp32 sums (ea_pointwise.cu: dm = s inv_n, rstd = rsqrt(q inv_n - dm^2 + eps))
    inv_n = torch.tensor(1.0, dtype=torch.float32) / (torch.tensor(float(HW)) * torch.tensor(float(cpg)))
    dm = s1 * inv_n
    r_k = torch.rsqrt(torch.clamp(s2 * inv_n - dm * dm, min=0.0) + eps).double()
    d_mean, d_rstd, r = R.gn_stats_bound(x, groups, eps, n_sm)
    err_mean = (dm.double() - md).abs()
    err_r = ((r_k - r) / r).abs()
    assert bool((err_mean <= d_mean).all()), float((err_mean / d_mean).max())
    assert bool((err_r <= d_rstd + 2 * R.U32).all()), float((err_r / d_rstd).max())       # + the rsqrt's rounding
    assert float((err_mean / d_mean).max()) > 1e-3          # not vacuous: within three orders of the rounding seen


@pytest.mark.parametrize("n_nets", [1, 2, 3])
@pytest.mark.parametrize("concat", [False, True])
@pytest.mark.parametrize("silu", [False, True])
def test_banded_groupnorm_matches_unbanded(n_nets, concat, silu, monkeypatch):
    """Two passes over bands of 3 pixel rows (HW = 10, not a multiple) against R.groupnorm on the whole tensor: the
    x | x2 concatenation, one gamma / beta per stacked network, SiLU on and off."""
    B, HW, C, groups = 6, 10, 64, 8
    C1 = 24 if concat else 0
    x, x2, g = _gn_case(B, HW, C, C1)
    gam = [torch.rand(C, generator=g) + 0.5 for _ in range(n_nets)]
    bet = [torch.randn(C, generator=g) for _ in range(n_nets)]
    a = dict(x=x[:, :C1 or C], gamma=gam if n_nets > 1 else gam[0], beta=bet if n_nets > 1 else bet[0],
             out=torch.zeros(B * HW, C), B=B, HW=HW, C_=C, groups=groups, eps=1e-5, silu=silu,
             workspace=cpu_ops.gn_workspace(B, CPU, groups), ldx=C1 + 8 if concat else C + 8)
    if concat:
        a.update(x2=x2[:, :C - C1], C1=C1, ldx2=C - C1 + 16)
    banded = _yields(monkeypatch, 3 * C, "groupnorm", **a)
    assert len(banded) == B * 4 and banded[5][0] == "out [image 1 rows 3-5]"
    xs = x[:, :C1 or C].double()
    if concat:
        xs = torch.cat([xs, x2[:, :C - C1].double()], -1)
    y, pre, terms = R.groupnorm(xs.reshape(B, HW, C), [t.double() for t in gam], [t.double() for t in bet], groups,
                                1e-5, silu)
    e = LA.NORM_K * R.U32 * terms + _gn_stats_excess(xs.reshape(B, HW, C), gam, groups, 1e-5)
    bound = R.ulp(y, cpu_ops.half_dtype()) + (1.1 * e + R.silu_eval_err(pre) if silu else e)
    for r, b in (_cat(banded, C), _cat(_yields(monkeypatch, BIG, "groupnorm", **a), C)):
        _same(r, y.reshape(-1, C), terms.reshape(-1, C))
        _same(b, bound.reshape(-1, C), bound.reshape(-1, C))


def test_groupnorm_statistics_merge_is_exact_enough():
    """Chan's merge over 1-row bands of a large-offset signal equals the two-pass statistics."""
    g = torch.Generator().manual_seed(7)
    x = (torch.randn(2, 300, 4, 16, generator=g) * 1e-3 + 1e3).double()
    n, mean, m2 = LA.groupnorm_stats(((b, x[b, i:i + 1]) for b in range(2) for i in range(300)), 2, 4)
    assert n == [300 * 16.0] * 2
    _same(mean, x.mean(dim=(1, 3)), x.abs().mean(dim=(1, 3)))
    var = x.var(dim=(1, 3), correction=0)
    assert bool(((m2 / n[0] - var).abs() <= 1e-9 * var).all())


@pytest.mark.parametrize("k,s", [(1, 1), (3, 1), (3, 2)])
def test_banded_direct_convolutions_match_unbanded(k, s, monkeypatch):
    """conv_direct (and conv_in, k = 3, s = 1) in bands of one output row against R.conv_nhwc of the whole image,
    odd sizes."""
    B, Hin, Win, cin, cout = 2, 9, 7, 3, 16
    g = torch.Generator().manual_seed(8)
    x = torch.randn(B, Hin, Win, cin, generator=g)
    w = torch.randn(k, k, cin, cout, generator=g)
    bias = torch.randn(cout, generator=g)
    Ho, Wo = -(-Hin // s), -(-Win // s)
    out = torch.zeros(B * Ho * Wo, 64)[:, :cout]
    ref, mag = R.conv_nhwc(x.double(), w.double(), bias.double(), stride=s)
    a = dict(x=x, w=w, bias=bias, out=out, B=B, Hin=Hin, Win=Win, Cin=cin, Cout=cout, ksize=k, stride=s, silu=False,
             ldo=64)
    ys = _yields(monkeypatch, 1, "conv_direct", **a)
    assert len(ys) == B * Ho
    got, _ = _cat(ys, cout)
    _same(got, ref.reshape(-1, cout), mag.reshape(-1, cout))
    if (k, s) == (3, 1):
        a = dict(x=x, w=w, bias=bias, out=torch.zeros(B, Hin, Win, cout), B=B, H=Hin, W=Win, Cin=cin, Cout=cout)
        got, _ = _cat(_yields(monkeypatch, 1, "conv_in", **a), cout)
        _same(got, ref.reshape(-1, cout), mag.reshape(-1, cout))


def test_layout_and_small_kernels_pass_banded(monkeypatch):
    """With one row (pixel row, query row) per band every check of the layout kernels, softmax, LayerNorm,
    attention and the direct convolutions still passes on the correct emulation, and covers every output."""
    monkeypatch.setattr(LA, "CHUNK_ELEMS", 1)
    g = torch.Generator().manual_seed(9)
    aud = Auditor(cpu_ops, "banded")
    B, H, W_, C = 2, 5, 3, 8
    x = torch.randn(B, H, W_, C, generator=g)
    aud.upsample2x(x, torch.zeros(B, 2 * H, 2 * W_, C), B=B, H=H, W=W_, C_=C)
    aud.image_out(torch.randn(B * H * W_, 8, generator=g), torch.zeros(B, 3, H * W_), B=B, HW=H * W_, C_=3, ldx=8)
    aud.nhwc_to_nchw_f32(x, torch.zeros(B, C, H * W_), B=B, HW=H * W_, C_=C)
    aud.softmax_rows(torch.randn(6, 9, generator=g), torch.zeros(6, 9), rows=6, cols=9)
    aud.layernorm(torch.randn(6, 16, generator=g), torch.rand(16, generator=g), torch.randn(16, generator=g),
                  torch.zeros(6, 16), M=6, C_=16)
    aud.conv_in(torch.randn(B, H, W_, 4, generator=g), torch.randn(3, 3, 4, 16, generator=g),
                torch.randn(16, generator=g), torch.zeros(B, H, W_, 16), B=B, H=H, W=W_, Cin=4, Cout=16,
                out2=torch.zeros(B, H, W_, 16))
    q = torch.randn(2, 7, 2 * 8, generator=g)
    kv = torch.randn(2, 5, 2 * 8, generator=g)
    aud.attention(q, kv, kv, torch.zeros(2, 7, 16), B=2, heads=2, Nq=7, Nkv=5, d=8, q_strides=(7 * 16, 16),
                  k_strides=(5 * 16, 16), v_strides=(5 * 16, 16), o_strides=(7 * 16, 16), scale=0.3)
    assert aud.calls == 7


def test_sam_and_vae_are_audited_in_bands(monkeypatch):
    """The tiny VAE decoder and encoder and a reduced-width denoising step with every reference built a few rows at
    a time."""
    monkeypatch.setattr(LA, "CHUNK_ELEMS", 64)
    for part, Eng, x in (("decoder", VaeDecoderEngine, torch.randn(2, 4, 5, 3)),
                         ("encoder", VaeEncoderEngine, torch.rand(2, 3, 24, 16) * 2 - 1)):
        aud = Auditor(cpu_ops, f"vae_tiny_{part}_banded")
        eng = Eng(VAE_TINY, make_vae_state_dict(VAE_TINY, 7, part=part), CPU, backend=aud)
        if part == "decoder":
            eng.decode_latents(x, use_graph=False)
        else:
            eng.encode(x, use_graph=False)
        assert aud.calls > 10
    _set_env(monkeypatch, "tiny_cn1")
    aud = Auditor(cpu_ops, "tiny_cn1_banded")
    eng, *inputs = denoise_engine("tiny_cn1", aud, CPU)
    run_trace_case(eng, *inputs, unipc_steps=2)
    assert aud.calls > 0


# ---- injected faults at band boundaries -------------------------------------------------------------------------
def _expect_band(be, fn, op, operand, band):
    msg = _expect(be, fn, op, operand)
    assert f"operand {operand} [{band}]:" in msg, msg
    return msg


@pytest.mark.parametrize("row,band", [(2, "image 1 rows 0-2"), (3, "image 1 rows 3-5")])
def test_fault_conv_output_at_a_band_boundary(row, band, monkeypatch):
    """Bands of 3 output rows: a wrong value in the last row of a band, or in the first row after a boundary, of
    image 1 of a 3x3 convolution is reported in that band."""
    B, H, W_, cin, cout = 2, 7, 5, 16, 8
    x, w, _ = _conv_case("s1", False, B, H, W_, cin, cout)
    monkeypatch.setattr(LA, "CHUNK_ELEMS", 3 * W_ * cout)

    def gemm(a, w, out=None, **kw):
        r = cpu_ops.gemm(a, w, out, **kw)
        out[H * W_ + row * W_ + 4, 3] += 0.01
        return r
    _expect_band(_backend(gemm=gemm), lambda o: o.gemm(x, w, torch.zeros(B * H * W_, cout), mode=1,
                                                       conv=(B, H, W_, cin)), "gemm", "out", band)


def _gn_fault(fault, monkeypatch, per=4):
    B, HW, C, groups = 2, 10, 64, 8
    x, _, g = _gn_case(B, HW, C, 0)
    gam, bet = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g)
    monkeypatch.setattr(LA, "CHUNK_ELEMS", per * C)

    def groupnorm(x, gamma, beta, out, **kw):
        r = cpu_ops.groupnorm(x, gamma, beta, out, **kw)
        fault(out, gamma)
        return r
    return lambda band: _expect_band(
        _backend(groupnorm=groupnorm),
        lambda o: o.groupnorm(x[:, :C], gam, bet, torch.zeros(B * HW, C), B=B, HW=HW, C_=C, groups=groups, silu=False,
                              ldx=C + 8, workspace=cpu_ops.gn_workspace(B, CPU, groups)), "groupnorm", "out", band)


@pytest.mark.parametrize("row,band", [(3, "image 1 rows 0-3"), (4, "image 1 rows 4-7")])
def test_fault_groupnorm_output_at_a_band_boundary(row, band, monkeypatch):
    def fault(out, gamma):
        out[10 + row, 37] += 0.01
    _gn_fault(fault, monkeypatch)(band)


def test_fault_groupnorm_statistics_of_one_group(monkeypatch):
    """Image 1's group 5 normalised with its mean off by 2 % of its standard deviation: every band of image 1 fails,
    the first one is reported."""
    def fault(out, gamma):
        out[10:, 40:48] -= 0.02 * gamma[40:48]
    msg = _gn_fault(fault, monkeypatch)("image 1 rows 0-3")
    assert "32 of 256 elements out of bound" in msg, msg
