"""-m gpu: ea_gemm's implicit-GEMM convolutions (CONV_S1 / CONV_S2 / CONV_S2A, the folded 1x1 skip `a_extra`) per
element against float64 (tests/fp64_refs.conv_gemm), at every tile geometry conv_geometry() produces for the
production shapes and under every launch layout.

A 128-row conv tile is a box of bw x bh pixels x bn images (conv_geometry in csrc/ea_gemm.cu, mirrored below).  The
epilogue is the fast one while a tile spans at most two images (bn <= 2) and the general one beyond (bn >= 4); when B is
not a multiple of bn the last image block is partly empty.  CASES holds one shape per geometry class, each at a B that
leaves the last block partial where bn > 1 (tests/test_conv_geometry_cpu.py keeps it that way).

Gate, per element, with u = 2^-24 and K = 9 Cin + Cin_extra: the pre-activation's error e = (K + 2) u (sum |a w| +
|bias| + |rowvec|), through SiLU's slope 1.1 plus fp64_refs.silu_eval_err where SiLU is on, plus one u per add of the
residual or the accumulated value, plus 1 ulp of the output (none for out_f32).  A failure names the worst element as
(image, y, x, channel).

Canaries: every input buffer has one more image slot past B filled with NaN (image slots past B and pixels past H / W
must be TMA zero fill, never loads), the row vector table one more row of NaN (no valid row may take the row vector of
an image past B), and every destination is a channel slot of a wider buffer with guard rows after row M, all holding a
sentinel that must come back untouched."""
import ctypes
import math

import numpy as np
import pytest
import torch

from editanything_b200 import _lib as L
from editanything_b200 import ops
from tests import fp64_refs as R

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
U = R.U32
MODES = {"s1": L.EA_GEMM_CONV_S1, "s2": L.EA_GEMM_CONV_S2, "s2a": L.EA_GEMM_CONV_S2A}
SENTINEL = 1234.0
GUARD_ROWS = 128
SHAPE = -2                   # EA_ERR_SHAPE
WORST = {}                   # "geometry class, epilogue path, layout" -> worst |err| / bound seen in this run


def conv_geometry(H, W):
    """(bw, bh, bn) of csrc/ea_gemm.cu conv_geometry for an H x W output."""
    bw = 1
    while bw * 2 <= W and bw * 2 <= 128 and W % (bw * 2) == 0:
        bw *= 2
    bh = 1
    while bh * 2 <= H and bw * bh * 2 <= 128 and H % (bh * 2) == 0:
        bh *= 2
    return bw, bh, 128 // (bw * bh)


def row_tiles(c):
    bw, bh, bn = conv_geometry(c["H"], c["W"])
    return -(-c["B"] // bn) * (c["H"] // bh) * (c["W"] // bw)


def epilogue_path(c):
    """The epilogue a one-pass launch runs: fast while a tile spans at most two images and the destination is half."""
    return "general" if conv_geometry(c["H"], c["W"])[2] >= 4 or c.get("f32") else "fast"


# B, H x W (output), Cin, Cout, mode; extra = Cin_extra of the folded skip (ld_extra its pixel stride, 0 = Cin_extra);
# lda = pixel stride of the input (0 = Cin; the channels past Cin hold NaN); rowvec / residual / slots (out and out2
# in channel slots of wider buffers) / silu / f32 (out_f32 accumulated into) / pad = real output channels of a
# zero-padded layer (hint stack: the rest must come out exactly 0)
CASES = {
    # 64x2x1: SD1.5 512^2 top level (ResBlock conv2 with the skip folded in from a wider concat buffer), SAM neck
    "sd15_64_skip": dict(B=2, H=64, W=64, cin=128, cout=320, mode="s1", extra=64, ld_extra=128, slots=True),
    # 64x2x1: ControlNet hint stack, stride 2 on 128^2, channels zero-padded to 64 / 128, SiLU
    "hint_64_s2_silu_pad": dict(B=1, H=64, W=64, cin=64, cin_real=32, cout=128, pad=96, mode="s2", silu=True),
    # 32x4x1: SD2.1 768^2 top level
    "sd21_96": dict(B=1, H=96, W=96, cin=64, cout=64, mode="s1", rowvec=True, residual=True),
    # 128x1x1: 1024^2 tile / VAE; VAE conv_out (8 channels); an fp32 destination accumulated into
    "vae_128_conv_out": dict(B=1, H=128, W=128, cin=128, cout=8, mode="s1"),
    "tile_128_f32_acc": dict(B=1, H=128, W=128, cin=64, cout=64, mode="s1", rowvec=True, f32=True),
    # 128x1x1: VAE encoder Downsample 512^2 -> 256^2
    "vae_s2a_256": dict(B=1, H=256, W=256, cin=64, cout=64, mode="s2a", residual=True),
    # 8x8x2 (fast epilogue, partial last block at odd B): SD1.5 / SD2.1 low levels, unguided sampling of 1, 3, 5 images
    "lat8_b1_conv1": dict(B=1, H=8, W=8, cin=1280, cout=1280, mode="s1", rowvec=True),
    "lat8_b1_skip": dict(B=1, H=8, W=8, cin=1280, cout=1280, mode="s1", extra=2560, slots=True),
    "lat8_b3": dict(B=3, H=8, W=8, cin=128, cout=320, mode="s1", extra=64, ld_extra=192, rowvec=True),
    "lat8_b5": dict(B=5, H=8, W=8, cin=64, cout=64, mode="s1", rowvec=True, residual=True, silu=True),
    "lat24_b3": dict(B=3, H=24, W=24, cin=64, cout=320, mode="s1", rowvec=True, residual=True, slots=True),
    # 8x4x4 (general epilogue): 768x512 bottom level
    "portrait_12x8_b2": dict(B=2, H=12, W=8, cin=128, cout=1280, mode="s1", rowvec=True, residual=True),
    # 4x4x8 (general epilogue): SD2.1 768^2 bottom level; Downsample 24^2 -> 12^2
    "sd21_12_b2": dict(B=2, H=12, W=12, cin=64, cout=320, mode="s1", rowvec=True, silu=True, slots=True),
    "sd21_12_b8_s2": dict(B=8, H=12, W=12, cin=64, cout=64, mode="s2", rowvec=True),
    "sd21_12_b3_s2": dict(B=3, H=12, W=12, cin=128, cout=64, mode="s2", residual=True),
    # 2x2x32: VAE at a 1040^2 image / 520^2 encoder input; an input read from a wider buffer (NaN padding channels)
    "vae_130_lda": dict(B=1, H=130, W=130, cin=64, cout=64, mode="s1", lda=128, residual=True),
    # 1x1x128: VAE at 520^2 (Downsample 130^2 -> 65^2), ragged shapes the ABI accepts
    "vae_65_s2a": dict(B=1, H=65, W=65, cin=64, cout=64, mode="s2a", rowvec=True),
    "ragged_7x13_b3": dict(B=3, H=7, W=13, cin=64, cout=64, mode="s1", extra=64, rowvec=True, residual=True,
                           slots=True),
}


def _bn_for(n):
    return 128 if n % 128 == 0 else 64 if n % 64 == 0 else 32


def _layouts(c):
    """one: one row tile per CTA; pair: two per CTA, bit for bit equal to one; bnXX: forced tile width; split: K split
    3 ways (every CTA resident)."""
    out = ["auto", "pair", "bn32", "bn64", "bn128"]
    if row_tiles(c) * -(-c["cout"] // 128) * 3 <= 132:
        out += ["split"]
    return out


CASE_LAYOUTS = [(n, lay) for n, c in CASES.items() for lay in _layouts(c)]


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    _BUILT.clear()
    if WORST:
        print("\nworst error / bound per geometry class (bw x bh x bn), epilogue path and layout:")
        for k in sorted(WORST):
            print(f"  {k:44s} {WORST[k]:.3f}")


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _randn(shape, seed, scale=1.0):
    return torch.randn(shape, generator=_gen(seed), device=DEV) * scale


def _close(key, what, got, ref, bound):
    """|got - ref| <= bound per element of [B, H, W, C] (NaN fails); records the worst ratio under `key`."""
    worst, i, n_bad = R.worst_element(got, ref, bound)
    WORST[key] = max(WORST.get(key, 0.0), worst)
    if not worst <= 1.0:
        b, y, x, ch = (int(v) for v in np.unravel_index(i, tuple(ref.shape)))
        raise AssertionError(f"{what}: {n_bad} of {ref.numel()} elements out of bound; worst at image {b}, y {y}, "
                             f"x {x}, channel {ch}: got {float(got.reshape(-1)[i])!r}, ref {float(ref.reshape(-1)[i])!r}"
                             f", bound {float(bound.reshape(-1)[i]):.3e} (ratio {worst:.3g})")


def _nan_tail(B, H, W, C, ld, seed, cin_real=None, scale=1.0):
    """[B + 1, H, W, ld] half buffer: image slot B and the channels past C are NaN; values in [:B, ..., :C] (channels
    past cin_real zero).  Returns (buffer, the values as float64 [B, H, W, C])."""
    buf = torch.full((B + 1, H, W, ld), float("nan"), device=DEV, dtype=ops.half_dtype())
    v = _randn((B, H, W, C), seed, scale).to(buf.dtype)
    if cin_real is not None:
        v[..., cin_real:] = 0
    buf[:B, ..., :C] = v
    return buf, v.double()


class _Case:
    """Inputs, weights and the float64 product of one CASES entry (built once per module run)."""

    def __init__(self, name, c, seed):
        h = ops.half_dtype()
        self.name, self.c = name, c
        B, H, W, cin, cout, mode = c["B"], c["H"], c["W"], c["cin"], c["cout"], c["mode"]
        s = 1 if mode == "s1" else 2
        self.M = B * H * W
        self.K = 9 * cin + c.get("extra", 0)
        self.lda = c.get("lda", 0)
        self.x, xd = _nan_tail(B, s * H, s * W, cin, self.lda or cin, seed, c.get("cin_real"))
        w = _randn((cout, self.K), seed + 1, self.K ** -0.5)
        self.bias = _randn((cout,), seed + 2)
        if "pad" in c:                                   # padded output channels: zero weights and bias
            w[c["pad"]:] = 0
            self.bias[c["pad"]:] = 0
        self.w = w.to(h)
        self.xe = None
        ed = None
        if c.get("extra"):
            ce = c["extra"]
            self.xe, ed = _nan_tail(B, H, W, ce, c.get("ld_extra") or ce, seed + 3)
        # row vector: a column slice of a wider [B + 1, 3 cout] table whose row B is NaN
        self.rv_table = torch.full((B + 1, 3 * cout), float("nan"), device=DEV)
        self.rv_table[:B] = _randn((B, 3 * cout), seed + 4, 2.0)
        self.rowvec = self.rv_table[:B, cout:2 * cout] if c.get("rowvec") else None
        # residual: a channel slot of a wider buffer
        self.res = None
        if c.get("residual"):
            rb = _randn((self.M, cout + 64), seed + 5).to(h)
            self.res = rb[:, 32:32 + cout]
        self.old = _randn((self.M, cout), seed + 6) if c.get("f32") else None
        pre, mag = R.conv_gemm(xd[..., :cin], self.w.double(), mode, ed)
        pre, mag = pre + self.bias.double(), mag + self.bias.double().abs()
        if self.rowvec is not None:
            rv = self.rowvec.double()[:, None, None, :]
            pre, mag = pre + rv, mag + rv.abs()
        self.pre, self.mag = pre, mag

    def kwargs(self):
        c = self.c
        kw = dict(mode=MODES[c["mode"]], conv=(c["B"], c["H"], c["W"], c["cin"]), bias=self.bias)
        if self.lda:
            kw["lda"] = self.lda
        if self.xe is not None:
            kw.update(a_extra=self.xe[..., :c["extra"]], ld_extra=self.xe.shape[-1])
        if self.rowvec is not None:
            kw["rowvec"] = self.rowvec
        if self.res is not None:
            kw["residual"] = self.res
        if c.get("silu"):
            kw["act"] = L.EA_ACT_SILU
        return kw

    def dests(self):
        """Fresh destinations in sentinel-filled buffers with GUARD_ROWS rows after row M: (out, out2, out_f32 (each
        a view or None), [(buffer, first column of its destination slot)])."""
        cout, M = self.c["cout"], self.M
        if self.c.get("f32"):
            buf = torch.full((M + GUARD_ROWS, cout + 32), SENTINEL, device=DEV)
            buf[:M, :cout] = self.old
            return None, None, buf[:M, :cout], [(buf, 0)]
        h = ops.half_dtype()
        if self.c.get("slots"):
            b1 = torch.full((M + GUARD_ROWS, 2 * cout + 64), SENTINEL, device=DEV, dtype=h)
            b2 = torch.full((M + GUARD_ROWS, cout + 128), SENTINEL, device=DEV, dtype=h)
            return b1[:M, cout:2 * cout], b2[:M, 64:64 + cout], None, [(b1, cout), (b2, 64)]
        b1 = torch.full((M + GUARD_ROWS, cout), SENTINEL, device=DEV, dtype=h)
        return b1[:M], None, None, [(b1, 0)]

    def check(self, key, what, got):
        """got: [M, cout] -> per-element gate against the float64 reference."""
        c = self.c
        B, H, W, cout = c["B"], c["H"], c["W"], c["cout"]
        y, err = R.gemm_act("silu" if c.get("silu") else "none", self.pre, (self.K + 2) * U * self.mag)
        extra = []
        if self.res is not None:
            extra.append(self.res.double().reshape(B, H, W, cout))
        if self.old is not None:
            extra.append(self.old.double().reshape(B, H, W, cout))
        ref, bound = R.gemm_out(y, err, 1.0, extra, None if got.dtype == torch.float32 else got.dtype)
        got = got.reshape(B, H, W, cout)
        _close(key, f"{self.name} {what}", got, ref, bound)
        if "pad" in c:
            assert bool((got[..., c["pad"]:] == 0).all()), f"{self.name} {what}: padded output channels are not 0"


_BUILT = {}


def _case(name):
    if name not in _BUILT:
        _BUILT[name] = _Case(name, CASES[name], 1000 + 17 * list(CASES).index(name))
    return _BUILT[name]


def _layout_kw(c, layout):
    bn = _bn_for(c["cout"])
    return {"auto": {}, "one": dict(force_2cta=-1, force_splits=1, force_bn=bn),
            "pair": dict(force_2cta=1, force_splits=1, force_bn=bn),
            "bn32": dict(force_2cta=-1, force_splits=1, force_bn=32),
            "bn64": dict(force_2cta=-1, force_splits=1, force_bn=64),
            "bn128": dict(force_2cta=-1, force_splits=1, force_bn=128),
            "split": dict(force_2cta=-1, force_splits=3, force_bn=128)}[layout]


def _run(cs, layout):
    """One launch of case `cs` under `layout`; checks the sentinels and returns the output ([M, cout]) and out2."""
    out, out2, o32, bufs = cs.dests()
    saved = [b.clone() for b, _ in bufs]
    kw = dict(cs.kwargs(), **_layout_kw(cs.c, layout))
    ops.gemm(cs.x, cs.w, out, out2=out2, out_f32=o32, accumulate=o32 is not None, **kw)
    torch.cuda.synchronize()
    cout, M = cs.c["cout"], cs.M
    for (b, c0), s in zip(bufs, saved):   # all but the destination slot keeps its sentinel, guard rows included
        b = b.clone()
        b[:M, c0:c0 + cout] = s[:M, c0:c0 + cout]
        assert torch.equal(b, s), f"{cs.name} {layout}: wrote outside its destination"
    return (o32 if o32 is not None else out), out2


@pytest.mark.parametrize("name,layout", CASE_LAYOUTS, ids=[f"{n}-{l}" for n, l in CASE_LAYOUTS])
def test_conv(name, layout):
    cs = _case(name)
    c = cs.c
    bw, bh, bn = conv_geometry(c["H"], c["W"])
    path = "split-K" if layout.startswith("split") else epilogue_path(c)
    key = f"{bw}x{bh}x{bn} {path} {layout}"
    got, out2 = _run(cs, layout)
    cs.check(key, layout, got)
    if out2 is not None:
        assert torch.equal(out2, got), f"{name} {layout}: out2 differs from out"
    if layout == "pair":
        # without split-K the row pair and one tile per CTA run the same K order and epilogue per row
        one, _ = _run(cs, "one")
        assert torch.equal(one, got), f"{name}: two row tiles per CTA differ from one ({row_tiles(c)} row tiles)"


def test_planner_splits_small_m_conv():
    """8x8 at one image, 1280 -> 1280 with the 2560-channel skip folded in (K = 9 * 1280 + 2560): the planner splits K
    (weight-bound layer), and that launch meets the gate of test_conv."""
    cs = _case("lat8_b1_skip")
    plan = (ctypes.c_int * 5)()
    L.check(L.load().ea_gemm_plan(row_tiles(cs.c), cs.c["cout"], cs.K // 64, L.EA_ACT_NONE, ops.GEMM_WS_BYTES,
                                  torch.cuda.get_device_properties(DEV).multi_processor_count, plan), "plan")
    assert plan[2] > 1, f"the planner does not split K for this layer: {list(plan)}"
    got, _ = _run(cs, "auto")
    cs.check("8x8x2 split-K planner", "planner split-K", got)


# ---- grouped launches: the UNet encoder and ControlNets stacked along the batch, one group per network ----------
GROUPED = {"lat8_b3": 3, "sd21_12_b2": 2}


@pytest.mark.parametrize("ng", [2, 3])
@pytest.mark.parametrize("name", list(GROUPED))
def test_grouped(name, ng):
    """Groups see conv[0] = B images each of a stacked [ng * B, ...] activation (BlockRunner.gemm), with their own
    weights, row vector, residual and a_extra.  Without split-K the grouped launch (one and two row tiles per CTA) and
    each group alone agree bit for bit; the planner's launch meets the float64 gate per group."""
    base = CASES[name]
    c = dict(base, B=GROUPED[name], residual=True, rowvec=True, extra=base.get("extra") or 64, slots=False,
             silu=False, ld_extra=0)
    B, H, W, cout = c["B"], c["H"], c["W"], c["cout"]
    cases = [_Case(f"{name} group {g}", dict(c), 5000 + 31 * g + 7 * ng) for g in range(ng)]
    M = cases[0].M
    h = ops.half_dtype()
    s = 1 if c["mode"] == "s1" else 2
    # stacked operands, image slot ng * B is NaN
    xs = torch.full((ng * B + 1, s * H, s * W, c["cin"]), float("nan"), device=DEV, dtype=h)
    es = torch.full((ng * B + 1, H, W, c["extra"]), float("nan"), device=DEV, dtype=h)
    rs = torch.empty(ng * M, cout, device=DEV, dtype=h)
    for g, cs in enumerate(cases):
        xs[g * B:(g + 1) * B] = cs.x[:B]
        es[g * B:(g + 1) * B] = cs.xe[:B]
        rs[g * M:(g + 1) * M] = cs.res
    bw, bh, bn = conv_geometry(H, W)

    def launch(layout):
        out = torch.full((ng * M + GUARD_ROWS, cout), SENTINEL, device=DEV, dtype=h)
        calls = []
        for g, cs in enumerate(cases):
            kw = dict(cs.kwargs(), a_extra=es[g * B:(g + 1) * B], residual=rs[g * M:(g + 1) * M],
                      **_layout_kw(c, layout))
            calls.append((xs[g * B:(g + 1) * B], cs.w, out[g * M:(g + 1) * M], kw))
        ops.gemm_grouped(calls)
        torch.cuda.synchronize()
        assert bool((out[ng * M:] == SENTINEL).all()), f"{name} x{ng}: wrote past the last group"
        return out[:ng * M]

    auto = launch("auto")
    for g, cs in enumerate(cases):
        cs.check(f"{bw}x{bh}x{bn} grouped x{ng} auto", f"x{ng} auto", auto[g * M:(g + 1) * M])
    one, pair = launch("one"), launch("pair")
    assert torch.equal(one, pair), f"{name} x{ng}: grouped row pairs differ from one tile per CTA"
    for g, cs in enumerate(cases):
        cs.check(f"{bw}x{bh}x{bn} grouped x{ng} one", f"x{ng} one", one[g * M:(g + 1) * M])
        alone = torch.full((M, cout), SENTINEL, device=DEV, dtype=h)
        ops.gemm(xs[g * B:(g + 1) * B], cs.w, alone,
                 **dict(cs.kwargs(), a_extra=es[g * B:(g + 1) * B], residual=rs[g * M:(g + 1) * M],
                        **_layout_kw(c, "one")))
        torch.cuda.synchronize()
        assert torch.equal(alone, one[g * M:(g + 1) * M]), f"{name} x{ng}: group {g} alone differs from grouped"


# ---- argument validation -----------------------------------------------------------------------------------------
def _rejects(status, fn):
    n0 = ops.launch_count()
    with pytest.raises(RuntimeError, match=rf"\({status}\)"):
        fn()
    torch.cuda.synchronize()
    assert ops.launch_count() == n0, "a rejected call launched a kernel"


def _raw(a, w, out, set_fields, **kw):
    """ea_gemm with fields of the filled ea_gemm_args overwritten (values ops.gemm derives from the tensors)."""
    g = L.GemmArgs()
    ops._fill_gemm(g, a, w, out, **kw)
    for k, v in set_fields.items():
        setattr(g, k, v)
    L.check(L.lib().ea_gemm(ctypes.byref(g), ops._stream()), "ea_gemm")


def test_rejected_arguments():
    h = ops.half_dtype()
    S1, S2, S2A = MODES["s1"], MODES["s2"], MODES["s2a"]
    B, H, W = 1, 8, 8
    x = torch.zeros(B, H, W, 128, device=DEV, dtype=h)
    x2 = torch.zeros(B, 2 * H, 2 * W, 128, device=DEV, dtype=h)
    w = torch.zeros(64, 9 * 128 + 64, device=DEV, dtype=h)     # with the folded 64-channel skip
    w1 = torch.zeros(64, 9 * 128, device=DEV, dtype=h)
    xe = torch.zeros(B, H, W, 64, device=DEV, dtype=h)
    out = torch.zeros(B * H * W, 64, device=DEV, dtype=h)
    conv = dict(mode=S1, conv=(B, H, W, 128))
    # Cin % 64, M != B H W, a_extra with the stride-2 modes, Cin_extra % 64
    _rejects(SHAPE, lambda: ops.gemm(x, w1, out, mode=S1, conv=(B, H, W, 96)))
    _rejects(SHAPE, lambda: _raw(x, w1, out, dict(M=B * H * W - 8), **conv))
    for mode in (S2, S2A):
        _rejects(SHAPE, lambda: ops.gemm(x2, w, out, mode=mode, conv=(B, H, W, 128), a_extra=xe))
    xe96 = torch.zeros(B, H, W, 96, device=DEV, dtype=h)
    _rejects(SHAPE, lambda: ops.gemm(x, torch.zeros(64, 9 * 128 + 96, device=DEV, dtype=h), out, a_extra=xe96,
                                     **conv))
    # conv lda: narrower than Cin or not a multiple of 8; ld_extra likewise against Cin_extra
    _rejects(SHAPE, lambda: ops.gemm(x, w1, out, lda=64, **conv))
    _rejects(SHAPE, lambda: ops.gemm(x, w1, out, lda=132, **conv))
    _rejects(SHAPE, lambda: ops.gemm(x, w, out, a_extra=xe, ld_extra=32, **conv))
    _rejects(SHAPE, lambda: ops.gemm(x, w, out, a_extra=xe, ld_extra=68, **conv))
    # ldw narrower than the total K (conv with the folded skip, and linear)
    _rejects(SHAPE, lambda: ops.gemm(x, w, out, a_extra=xe, ldw=9 * 128, **conv))
    a = torch.zeros(128, 256, device=DEV, dtype=h)
    wl = torch.zeros(64, 256, device=DEV, dtype=h)
    ol = torch.zeros(128, 64, device=DEV, dtype=h)
    _rejects(SHAPE, lambda: ops.gemm(a, wl, ol, ldw=128))
    # linear lda < K
    _rejects(SHAPE, lambda: ops.gemm(a, wl, ol, lda=128))
    # ldo, ldo2, ldr narrower than the output width (0 would write every row onto row 0)
    for ld in (0, 32):
        _rejects(SHAPE, lambda: ops.gemm(x, w1, out, ldo=ld, **conv))
        _rejects(SHAPE, lambda: ops.gemm(x, w1, out, out2=torch.zeros_like(out), ldo2=ld, **conv))
        _rejects(SHAPE, lambda: ops.gemm(x, w1, out, residual=torch.zeros_like(out), ldr=ld, **conv))
        _rejects(SHAPE, lambda: ops.gemm(a, wl, ol, ldo=ld))
        _rejects(SHAPE, lambda: ops.gemm(a, wl, out_f32=torch.zeros(128, 64, device=DEV), ldo=ld))
    # GEGLU writes N / 2 columns: ldo = N / 2 is a whole row, less is not
    wg = torch.zeros(256, 256, device=DEV, dtype=h)
    og = torch.zeros(128, 128, device=DEV, dtype=h)
    _rejects(SHAPE, lambda: ops.gemm(a, wg, og, act=L.EA_ACT_GEGLU, ldo=120))
    ops.gemm(a, wg, og, act=L.EA_ACT_GEGLU, ldo=128)
    # the widest accepted values of every check still run: whole rows, wider buffers
    ops.gemm(x, w, out, a_extra=xe, ld_extra=64, ldw=9 * 128 + 64, **conv)
    ops.gemm(x, w1, out, lda=128, **conv)
    torch.cuda.synchronize()
