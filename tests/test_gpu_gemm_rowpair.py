"""-m gpu: two vertically adjacent 128-row tiles per CTA (ea_gemm_args.force_2cta = 1) against a float64 reference and
against the one-tile-per-CTA layout (force_2cta = -1).

Both layouts compute every output element with the same wgmma K order and the same per-row epilogue, so without
split-K they must agree to the last bit.  The float64 check bounds the error by one ulp of the output type plus the
fp32 accumulation (K * 2^-24 * sum |a w|).  Shapes cover an odd number of row tiles (the last CTA has one valid
sub-tile), M not a multiple of 128, a conv sub-tile whose image block lies past the batch, and a time-embedding row
vector whose images change inside a pair."""
import pytest
import torch
import torch.nn.functional as F

from editanything_b200 import _lib as L
from editanything_b200 import ops
from tests import fp64_refs as R

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
MODES = {"s1": L.EA_GEMM_CONV_S1, "s2": L.EA_GEMM_CONV_S2, "s2a": L.EA_GEMM_CONV_S2A}


def _rand(g, *shape, scale=1.0):
    return torch.randn(*shape, device=DEV, generator=g) * scale


def _bn(n):
    """A tile width both layouts use (the planner may choose different widths for them)."""
    return 128 if n % 128 == 0 else 64


def _both(run):
    """run(force_2cta) -> output tensor(s); returns (one tile per CTA, two tiles per CTA)."""
    a = run(-1)
    b = run(1)
    torch.cuda.synchronize()
    return a, b


def _equal(ref, got):
    for x, y in zip(ref if isinstance(ref, tuple) else (ref,), got if isinstance(got, tuple) else (got,)):
        assert torch.equal(x, y), float((x.float() - y.float()).abs().max())


def _check_fp64(got, ref, mag, K, dtype):
    bound = R.ulp(ref, dtype) + (K + 8) * R.U32 * mag
    err = (got.double() - ref).abs()
    assert bool((err <= bound).all()), float((err / bound).max())


def _conv_ref(x, w, cin, mode, bias, xe=None):
    """x NHWC (input size), w [Cout, 9 Cin (+ Cin_extra)] in the library's (kh, kw, c) order -> NHWC out, |.| sums."""
    cout = w.shape[0]
    wt = w[:, :9 * cin].reshape(cout, 3, 3, cin).permute(0, 3, 1, 2)
    xc = x.permute(0, 3, 1, 2)
    if mode == "s2a":
        xc = F.pad(xc, (0, 1, 0, 1))
        conv = lambda a, b: F.conv2d(a, b, stride=2)
    else:
        conv = lambda a, b: F.conv2d(a, b, stride=1 if mode == "s1" else 2, padding=1)
    out, mag = conv(xc, wt), conv(xc.abs(), wt.abs())
    out, mag = out.permute(0, 2, 3, 1), mag.permute(0, 2, 3, 1)
    if xe is not None:
        we = w[:, 9 * cin:]
        out, mag = out + xe @ we.T, mag + xe.abs() @ we.abs().T
    return out + bias, mag + bias.abs()


@pytest.mark.parametrize("M,N,K", [
    (300, 320, 320),        # 3 row tiles: the second CTA's sub-tile 1 is empty; ragged M
    (1024, 640, 640),       # even number of row tiles
    (8192, 320, 1280),      # a bench shape (ff2 at 64x64)
    (128, 1280, 640),       # one row tile
])
@pytest.mark.parametrize("epi", ["plain", "residual", "rowvec", "out2", "f32", "f32_acc", "accumulate", "row_scale"])
def test_linear(M, N, K, epi):
    dt = ops.half_dtype()
    g = torch.Generator(device=DEV).manual_seed(M + N + K + len(epi))
    x = _rand(g, M, K).to(dt)
    w = _rand(g, N, K, scale=K ** -0.5).to(dt)
    b = _rand(g, N)
    res = _rand(g, M, N).to(dt) if epi == "residual" else None
    rpb = 200 if M >= 400 else 100           # images change inside a pair of row tiles
    rv = _rand(g, (M + rpb - 1) // rpb, N) if epi == "rowvec" else None
    rs = torch.rand(M, device=DEV, generator=g) + 0.5 if epi == "row_scale" else None
    old = _rand(g, M, N)
    f32 = epi.startswith("f32")
    acc = epi in ("accumulate", "f32_acc")

    def run(f2):
        out = None if f32 else (old.to(dt) if acc else torch.full((M, N), 7.0, device=DEV, dtype=dt))
        o32 = old.clone() if f32 else None
        out2 = torch.full((M, N), 5.0, device=DEV, dtype=dt) if epi == "out2" else None
        ops.gemm(x, w, out, out_f32=o32, bias=b, residual=res, rowvec=rv, rows_per_batch=rpb if rv is not None else 0,
                 out2=out2, accumulate=acc, row_scale=rs, out_scale=0.75, force_2cta=f2, force_bn=_bn(N))
        return (o32 if f32 else out,) + ((out2,) if out2 is not None else ())
    ref, got = _both(run)
    _equal(ref, got)
    xd, wd = x.double(), w.double()
    exp, t, mag = R.gemm_epilogue(xd, wd, b.double(), 0.75, rs.double() if rs is not None else None)
    if rv is not None:
        rvd = rv.double().repeat_interleave(rpb, dim=0)[:M] * 0.75
        exp, mag = exp + rvd, mag + rvd.abs()
    if res is not None:
        exp, mag = exp + res.double(), mag + res.double().abs()
    if acc:
        o = old.double() if f32 else old.to(dt).double()
        exp, mag = exp + o, mag + o.abs()
    _check_fp64(got[0], exp, mag, K, torch.float32 if f32 else dt)
    if epi == "out2":
        assert torch.equal(got[0], got[1])


@pytest.mark.parametrize("act", [L.EA_ACT_SILU, L.EA_ACT_GELU, L.EA_ACT_GEGLU])
@pytest.mark.parametrize("M", [300, 8192])
def test_linear_activations_match_one_tile_layout(act, M):
    dt = ops.half_dtype()
    N, K = 1280, 320
    g = torch.Generator(device=DEV).manual_seed(M + act)
    x = _rand(g, M, K).to(dt)
    w = _rand(g, N, K, scale=K ** -0.5).to(dt)
    b = _rand(g, N)
    n_out = N // 2 if act == L.EA_ACT_GEGLU else N
    res = _rand(g, M, n_out).to(dt) if act == L.EA_ACT_GELU else None

    def run(f2):
        out = torch.full((M, n_out), 7.0, device=DEV, dtype=dt)
        ops.gemm(x, w, out, bias=b, residual=res, act=act, force_2cta=f2, force_bn=128)
        return out
    _equal(*_both(run))


@pytest.mark.parametrize("M", [300, 4096])
def test_layernorm_fold_both_sides(M):
    """proj_in-like producer writes per-row statistics, a to_q / GEGLU-like consumer folds them in."""
    dt = ops.half_dtype()
    C, N = 320, 1280
    g = torch.Generator(device=DEV).manual_seed(M)
    x = _rand(g, M, C).to(dt)
    w0 = _rand(g, C, C, scale=C ** -0.5).to(dt)
    b0 = _rand(g, C)
    res = _rand(g, M, C).to(dt)
    w1 = _rand(g, N, C, scale=C ** -0.5).to(dt)
    b1 = _rand(g, N)
    lg = _rand(g, N)

    def run(f2):
        h = torch.empty(M, C, device=DEV, dtype=dt)
        st = torch.empty(C // 32, M, 2, device=DEV)
        ops.gemm(x, w0, h, bias=b0, residual=res, rowstats_out=st, force_2cta=f2, force_bn=64)
        outs = [h, st]
        for act in (L.EA_ACT_NONE, L.EA_ACT_GEGLU):
            n_out = N // 2 if act == L.EA_ACT_GEGLU else N
            out = torch.empty(M, n_out, device=DEV, dtype=dt)
            ops.gemm(h, w1, out, bias=b1, act=act, ln=(st, lg, 1e-5), force_2cta=f2, force_bn=128)
            outs.append(out)
        return tuple(outs)
    _equal(*_both(run))


@pytest.mark.parametrize("B,H,W,cin,cout,mode,extra", [
    (2, 64, 64, 320, 320, "s1", 0),
    (5, 8, 8, 128, 320, "s1", 0),          # 3 row tiles of 2 images: the last pair's sub-tile 1 lies past the batch
    (5, 8, 8, 64, 128, "s1", 128),         # fused 1x1 skip as extra K-blocks, odd number of row tiles
    (2, 32, 32, 320, 320, "s2", 0),
    (3, 8, 8, 128, 128, "s2", 0),
    (1, 64, 64, 128, 128, "s2a", 0),
    (3, 16, 16, 64, 64, "s2a", 0),
])
def test_conv(B, H, W, cin, cout, mode, extra):
    dt = ops.half_dtype()
    g = torch.Generator(device=DEV).manual_seed(B * H + cin + extra)
    s = 1 if mode == "s1" else 2
    x = _rand(g, B, H * s, W * s, cin).to(dt)
    w = _rand(g, cout, 9 * cin + extra, scale=(9 * cin) ** -0.5).to(dt)
    b = _rand(g, cout)
    rv = _rand(g, B, cout)
    xe = _rand(g, B, H, W, extra).to(dt) if extra else None
    res = _rand(g, B * H * W, cout).to(dt)

    def run(f2):
        out = torch.full((B * H * W, cout), 7.0, device=DEV, dtype=dt)
        ops.gemm(x, w, out, mode=MODES[mode], conv=(B, H, W, cin), bias=b, rowvec=rv, residual=res, a_extra=xe,
                 ld_extra=extra, force_2cta=f2, force_bn=_bn(cout))
        return out
    ref, got = _both(run)
    _equal(ref, got)
    exp, mag = _conv_ref(x.double(), w.double(), cin, mode, b.double(), xe.double() if xe is not None else None)
    rvd = rv.double()[:, None, None, :]
    exp = (exp + rvd).reshape(B * H * W, cout) + res.double()
    mag = (mag + rvd.abs()).reshape(B * H * W, cout) + res.double().abs()
    _check_fp64(got, exp, mag, 9 * cin + extra, dt)


@pytest.mark.parametrize("ng", [2, 3])
@pytest.mark.parametrize("kind", ["linear", "conv", "geglu"])
def test_grouped(ng, kind):
    dt = ops.half_dtype()
    g = torch.Generator(device=DEV).manual_seed(ng * 10 + len(kind))
    if kind == "conv":
        B, H, W, cin, cout = 3, 16, 16, 128, 320
        M, K = B * H * W, 9 * cin
        xs = [_rand(g, B, H, W, cin).to(dt) for _ in range(ng)]
        kw = dict(mode=L.EA_GEMM_CONV_S1, conv=(B, H, W, cin), rowvec=_rand(g, B, cout))
        n_out = N = cout
    else:
        M, K, N = 1000, 320, 1280 if kind == "geglu" else 640
        xs = [_rand(g, M, K).to(dt) for _ in range(ng)]
        kw = dict(act=L.EA_ACT_GEGLU) if kind == "geglu" else dict(residual=_rand(g, M, N).to(dt))
        n_out = N // 2 if kind == "geglu" else N
    ws = [_rand(g, N, K, scale=K ** -0.5).to(dt) for _ in range(ng)]
    bs = [_rand(g, N) for _ in range(ng)]

    def run(f2):
        outs = [torch.full((M, n_out), 7.0, device=DEV, dtype=dt) for _ in range(ng)]
        ops.gemm_grouped([(xs[i], ws[i], outs[i], dict(kw, bias=bs[i], force_2cta=f2, force_bn=_bn(N)))
                          for i in range(ng)])
        return tuple(outs)
    ref, got = _both(run)
    _equal(ref, got)
    # each group on its own (ea_gemm) gives the same bits
    for i in range(ng):
        one = torch.full((M, n_out), 7.0, device=DEV, dtype=dt)
        ops.gemm(xs[i], ws[i], one, **dict(kw, bias=bs[i], force_2cta=1, force_bn=_bn(N)))
        torch.cuda.synchronize()
        assert torch.equal(one, got[i])


@pytest.mark.parametrize("variant", [1, 2])
@pytest.mark.parametrize("M,N,K,act", [(8192, 2560, 320, L.EA_ACT_GEGLU), (19000, 640, 192, L.EA_ACT_GELU),
                                       (8192, 320, 320, L.EA_ACT_NONE)])
def test_persistent(M, N, K, act, variant):
    dt = ops.half_dtype()
    g = torch.Generator(device=DEV).manual_seed(M + N + act)
    x = _rand(g, M, K).to(dt)
    w = _rand(g, N, K, scale=K ** -0.5).to(dt)
    b = _rand(g, N)
    n_out = N // 2 if act == L.EA_ACT_GEGLU else N
    res = _rand(g, M, n_out).to(dt) if act != L.EA_ACT_GEGLU else None

    def run(f2, persist):
        out = torch.full((M, n_out), 7.0, device=DEV, dtype=dt)
        ops.gemm(x, w, out, bias=b, residual=res, act=act, force_2cta=f2, force_bn=_bn(N),
                 force_persistent=variant if persist else -1)
        return out
    ref = run(-1, False)
    got = run(1, True)
    torch.cuda.synchronize()
    _equal(ref, got)


@pytest.mark.parametrize("M,N,K,splits,epi", [
    (300, 320, 1280, 4, "residual"),       # 3 row tiles -> 2 items x 3 column tiles x 4 splits
    (512, 1280, 2560, 3, "rowvec"),
    (128, 1280, 2880, 5, "f32_acc"),       # one row tile: the pair's sub-tile 1 is empty
    (384, 1280, 640, 2, "geglu"),
])
def test_split_k(M, N, K, splits, epi):
    dt = ops.half_dtype()
    g = torch.Generator(device=DEV).manual_seed(M + N + K)
    x = _rand(g, M, K).to(dt)
    w = _rand(g, N, K, scale=K ** -0.5).to(dt)
    b = _rand(g, N)
    geglu = epi == "geglu"
    n_out = N // 2 if geglu else N
    res = _rand(g, M, N).to(dt) if epi == "residual" else None
    rv = _rand(g, 3, N) if epi == "rowvec" else None
    old = _rand(g, M, N)
    f32 = epi == "f32_acc"

    def run(f2):
        out = None if f32 else torch.full((M, n_out), 7.0, device=DEV, dtype=dt)
        o32 = old.clone() if f32 else None
        ops.gemm(x, w, out, out_f32=o32, bias=b, residual=res, rowvec=rv, rows_per_batch=200 if rv is not None else 0,
                 act=L.EA_ACT_GEGLU if geglu else L.EA_ACT_NONE, accumulate=f32, force_2cta=f2, force_bn=_bn(N),
                 force_splits=splits)
        return o32 if f32 else out
    ref, got = _both(run)
    # the split partial sums are added in the same order in both layouts
    _equal(ref, got)
    if geglu:
        return
    exp, _, mag = R.gemm_epilogue(x.double(), w.double(), b.double())
    if rv is not None:
        rvd = rv.double().repeat_interleave(200, dim=0)[:M]
        exp, mag = exp + rvd, mag + rvd.abs()
    if res is not None:
        exp, mag = exp + res.double(), mag + res.double().abs()
    if f32:
        exp, mag = exp + old.double(), mag + old.double().abs()
    _check_fp64(got, exp, mag, K, torch.float32 if f32 else dt)


def test_bn256_takes_one_row_tile():
    """BN = 256 keeps one row tile per CTA: forcing two is rejected, the planner's choice falls back to one."""
    dt = ops.half_dtype()
    g = torch.Generator(device=DEV).manual_seed(256)
    x = _rand(g, 1024, 256).to(dt)
    w = _rand(g, 512, 256, scale=1 / 16).to(dt)
    with pytest.raises(RuntimeError):
        ops.gemm(x, w, force_bn=256, force_2cta=1)
    got = ops.gemm(x, w, force_bn=256)
    torch.cuda.synchronize()
    exp, _, mag = R.gemm_epilogue(x.double(), w.double())
    _check_fp64(got, exp, mag, 256, dt)
