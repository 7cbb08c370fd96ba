"""The case table of tests/test_gpu_conv_fp64.py keeps one shape per conv tile geometry class production reaches, both
epilogue paths, a partly empty last image block wherever a tile holds more than one image, and the operands and
layouts the float64 gate is meant to cover.  conv_geometry there mirrors csrc/ea_gemm.cu; its expected values below are
worked out from the rule (bw: the largest power of two dividing W, at most 128; bh: the largest power of two dividing H
with bw bh <= 128; bn = 128 / (bw bh))."""
from tests.test_gpu_conv_fp64 import CASES, GROUPED, _layouts, conv_geometry, epilogue_path, row_tiles

# (bw, bh, bn) -> where production runs it
CLASSES = {
    (64, 2, 1): "SD1.5 512^2 top level, SAM neck (64 x 64)",
    (32, 4, 1): "SD2.1 768^2 top level (96 x 96)",
    (128, 1, 1): "1024^2 tile, VAE (128 x 128, 256 x 256)",
    (8, 8, 2): "SD1.5 / SD2.1 low levels (8 x 8, 24 x 24)",
    (8, 4, 4): "768 x 512 bottom level (12 x 8)",
    (4, 4, 8): "SD2.1 768^2 bottom level (12 x 12)",
    (2, 2, 32): "VAE at a 1040^2 image (130 x 130)",
    (1, 1, 128): "VAE at 520^2, ragged shapes (65 x 65, 7 x 13)",
}


def test_conv_geometry_mirror():
    want = {(64, 64): (64, 2, 1), (96, 96): (32, 4, 1), (128, 128): (128, 1, 1), (256, 256): (128, 1, 1),
            (8, 8): (8, 8, 2), (24, 24): (8, 8, 2), (12, 8): (8, 4, 4), (12, 12): (4, 4, 8), (130, 130): (2, 2, 32),
            (65, 65): (1, 1, 128), (7, 13): (1, 1, 128), (260, 260): (4, 4, 8)}
    for (H, W), g in want.items():
        assert conv_geometry(H, W) == g, (H, W)


def test_every_geometry_class_with_a_partial_image_block():
    by_class = {}
    for name, c in CASES.items():
        by_class.setdefault(conv_geometry(c["H"], c["W"]), []).append(name)
    for g, where in CLASSES.items():
        assert g in by_class, f"no case for {g}: {where}"
        if g[2] > 1:
            assert any(CASES[n]["B"] % g[2] for n in by_class[g]), f"{g}: no case leaves the last image block partial"
    assert {epilogue_path(c) for c in CASES.values()} == {"fast", "general"}
    # the fast path's second row vector row at odd B (8 x 8 x 2 with B = 1, 3, 5)
    assert {c["B"] for c in CASES.values() if conv_geometry(c["H"], c["W"]) == (8, 8, 2) and c.get("rowvec")} >= {1, 3, 5}
    assert {c["B"] for c in CASES.values() if (c["H"], c["W"]) == (12, 12)} >= {2, 8}


def test_modes_operands_and_layouts():
    cs = list(CASES.values())
    assert {c["mode"] for c in cs} == {"s1", "s2", "s2a"}
    assert {8, 64, 320, 1280} <= {c["cout"] for c in cs}
    assert any(c.get("extra") and c.get("ld_extra", 0) > c["extra"] for c in cs), "a_extra from a wider buffer"
    assert any(c.get("lda", 0) > c["cin"] for c in cs), "input read from a wider buffer"
    assert any(c.get("pad") and c.get("silu") for c in cs), "zero-padded channels through SiLU"
    assert any(c.get("f32") for c in cs) and any(c.get("slots") for c in cs)
    assert any(c.get("rowvec") for c in cs) and any(c.get("residual") for c in cs)
    # the 2-row-tile layout with an odd number of row tiles (the last CTA's second tile is empty), split-K
    assert any(row_tiles(c) % 2 and "pair" in _layouts(c) for c in cs)
    assert any(row_tiles(c) > 1 and "split" in _layouts(c) for c in cs)
    assert {conv_geometry(CASES[n]["H"], CASES[n]["W"])[2] for n in GROUPED} >= {2, 8}
