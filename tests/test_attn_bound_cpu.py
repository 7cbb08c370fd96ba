"""The per-element error bound of tests/attn_ref.py (attention_bound), checked against a float32 / float16 model of
ea_attention's arithmetic on the CPU, and ea_attention's argument validation.

The model (emulate) follows editanything_b200/csrc/ea_attn.cu, not bit for bit: per query row it walks the keys in
sub-tiles of 128 (64 at d > 80), keeps the running max in the log2 domain, computes p = exp2(s scale log2e - m) in
fp32 (with the bias: s scale log2e + (rel_h + rel_w) log2e, then scale 1), masks only the ragged last sub-tile,
rounds p to fp16 for O += P V in fp32, keeps l in fp32 from the unrounded p and rescales O and l when the max rises.

Two properties at the sizes of attn_ref.CASES small enough for the CPU:
  * the correct model stays within the bound for every generator;
  * each planted defect leaves it on a named case that tests/test_gpu_attention.py also runs:
      (a) one key past Nkv admitted (zero K / V row)    flat-offset, 129 keys, scale 0.05
      (b) O not rescaled when the running max rises     rising, 129 keys
      (c) the bias multiplied by scale                  bias generator
      (d) kk / rel_s and kk % rel_s swapped             bias generator
      (e) V read from the neighbouring head             distinct
      (f) the last ragged sub-tile dropped              flat-offset, 192 keys
Not covered: defects within the rounding the bound allows, for example P rounded toward zero instead of to
nearest (at most one fp16 ulp per P, which the P quantisation term admits), or l summed from the rounded P."""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

from editanything_b200 import _lib
from tests import attn_ref

LOG2E32 = torch.tensor(attn_ref.LOG2E, dtype=torch.float32)
CPU_SIZE = 3_000_000        # B heads Nq Nkv of the cases the model runs


def emulate(inp, scale, rel_s=0, defect=None, dtype=torch.float16):
    q, k, v = inp["q"].float(), inp["k"].float(), inp["v"].float()
    B, Nq, heads, d = q.shape
    Nkv = k.shape[1]
    SN = attn_ref.sub_tile(d)
    n_sub = -(-Nkv // SN)
    ragged = Nkv % SN != 0
    pad = n_sub * SN - Nkv
    k = F.pad(k, (0, 0, 0, 0, 0, pad))          # the TMA zero fill of keys past Nkv
    v = F.pad(v, (0, 0, 0, 0, 0, pad))
    sl = torch.tensor(scale, dtype=torch.float32) * LOG2E32       # the host's fp32 scale * log2e
    bias = rel_s > 0
    sc = torch.tensor(1.0) if bias else sl
    if bias:
        kk = torch.arange(n_sub * SN)
        kh, kw = (kk // rel_s).clamp(max=rel_s - 1), kk % rel_s      # kh clamped for the masked keys
        if defect == "d":
            kh, kw = kw, kh
    last = n_sub - 1 if defect == "f" and ragged and n_sub > 1 else n_sub
    out = torch.empty(B, Nq, heads, d, dtype=dtype)
    for b in range(B):
        for h in range(heads):
            Q, K = q[b, :, h], k[b, :, h]
            V = v[b, :, (h + 1) % heads if defect == "e" else h]
            if bias:
                rh = inp["rel_h"][b * heads + h].float() * LOG2E32
                rw = inp["rel_w"][b * heads + h].float() * LOG2E32
            m = torch.full((Nq,), -math.inf)
            l = torch.zeros(Nq)
            O = torch.zeros(Nq, d)
            for t in range(last):
                ks = slice(t * SN, (t + 1) * SN)
                S = Q @ K[ks].T
                if bias:
                    bt = rw[:, kw[ks]] + rh[:, kh[ks]]
                    S = S * sl + (bt * scale if defect == "c" else bt)
                if ragged and t == n_sub - 1:
                    S[:, Nkv - t * SN + (1 if defect == "a" else 0):] = -math.inf
                mn = torch.maximum(m, S.amax(dim=1) * sc)
                a = torch.exp2(m - mn)
                m = mn
                p = torch.exp2(S * sc - mn[:, None])
                l = l * a + p.sum(dim=1)
                if defect != "b":
                    O = O * a[:, None]
                O = O + p.to(dtype).float() @ V[ks]
            out[b, :, h] = (O / l[:, None]).to(dtype)
    return out


def _inputs(name):
    gen, B, heads, Nq, Nkv, d, scale, rel_s, _ = attn_ref.CASES[name]
    scale = d ** -0.5 if scale is None else scale
    inp = attn_ref.make_inputs(gen, B, heads, Nq, Nkv, d, scale, rel_s, seed=len(name))
    o, bound = attn_ref.attention_bound(inp["q"], inp["k"], inp["v"], scale, inp["rel_h"], inp["rel_w"], rel_s)
    return inp, scale, rel_s, o, bound


def _ratio(got, o, bound):
    return float(((got.double() - o).abs() / bound).max())


SMALL = [n for n, c in attn_ref.CASES.items() if c[1] * c[2] * c[3] * c[4] <= CPU_SIZE]


def test_model_stays_within_bound_on_every_generator():
    worst = {}
    for name in SMALL:
        inp, scale, rel_s, o, bound = _inputs(name)
        r = _ratio(emulate(inp, scale, rel_s), o, bound)
        gen = attn_ref.CASES[name][0]
        worst[gen] = max(worst.get(gen, 0.0), r)
        assert r <= 1.0, (name, r)
    print("\nmodel: worst error / bound per generator")
    for gen in sorted(worst):
        print(f"  {gen:12s} {worst[gen]:.3f}")
    assert set(worst) == set(attn_ref.GENERATORS) - {"randn"}


DEFECTS = {
    "a": "flat-offset d64 keys129 scale0.05",
    "b": "rising d64 keys129",
    "c": "bias d64 bias",
    "d": "bias d80 bias",
    "e": "distinct d40",
    "f": "keys192 d64",
}


@pytest.mark.parametrize("defect", sorted(DEFECTS))
def test_bound_catches_planted_defect(defect):
    name = DEFECTS[defect]
    assert name in SMALL
    inp, scale, rel_s, o, bound = _inputs(name)
    r = _ratio(emulate(inp, scale, rel_s, defect=defect), o, bound)
    gen, B, heads, Nq, Nkv, d = attn_ref.CASES[name][:6]
    print(f"\ndefect ({defect}): case '{name}' gen={gen} B={B} heads={heads} Nq={Nq} Nkv={Nkv} d={d} "
          f"error / bound = {r:.3g}")
    assert r > 1.0, (defect, name, r)


# ---- argument validation: every call below is rejected before any CUDA call ----------------------------------------
EA_ERR_ARG, EA_ERR_SHAPE = -1, -2


def _args(**kw):
    a = _lib.AttnArgs()
    a.q, a.k, a.v, a.out = 0x10000, 0x20000, 0x30000, 0x40000      # placeholders, never dereferenced
    a.B, a.heads, a.Nq, a.Nkv, a.d = 2, 2, 128, 196, 64
    a.q_bs = a.k_bs = a.v_bs = a.o_bs = 196 * 128
    a.q_ns = a.k_ns = a.v_ns = a.o_ns = 128
    a.scale = 0.125
    a.rel_h, a.rel_w, a.rel_s = 0x50000, 0x60000, 14
    for key, val in kw.items():
        setattr(a, key, val)
    return a


REJECTED = [
    ("no q", dict(q=None), EA_ERR_ARG),
    ("no out", dict(out=None), EA_ERR_ARG),
    ("d 0", dict(d=0), EA_ERR_SHAPE),
    ("d 4", dict(d=4), EA_ERR_SHAPE),
    ("d 60", dict(d=60), EA_ERR_SHAPE),
    ("d 196", dict(d=196), EA_ERR_SHAPE),
    ("d 200", dict(d=200), EA_ERR_SHAPE),
    ("d -8", dict(d=-8), EA_ERR_SHAPE),
    ("Nq 0", dict(Nq=0), EA_ERR_SHAPE),
    ("Nkv 0", dict(Nkv=0), EA_ERR_SHAPE),
    ("B 0", dict(B=0), EA_ERR_SHAPE),
    ("heads -1", dict(heads=-1), EA_ERR_SHAPE),
    ("scale 0", dict(scale=0.0), EA_ERR_ARG),
    ("scale -1", dict(scale=-1.0), EA_ERR_ARG),
    ("scale nan", dict(scale=math.nan), EA_ERR_ARG),
    ("scale inf", dict(scale=math.inf), EA_ERR_ARG),
    ("scale -inf", dict(scale=-math.inf), EA_ERR_ARG),
    ("rel_h without rel_w", dict(rel_w=None), EA_ERR_ARG),
    ("rel_w without rel_h", dict(rel_h=None), EA_ERR_ARG),
    ("rel_s 0", dict(rel_s=0), EA_ERR_ARG),
    ("rel_s -14", dict(rel_s=-14), EA_ERR_ARG),
    ("Nkv 197 > rel_s^2", dict(Nkv=197), EA_ERR_SHAPE),
    ("Nkv 4097 > 64^2", dict(Nkv=4097, rel_s=64), EA_ERR_SHAPE),
    ("rel_w rows past shared memory", dict(rel_s=1 << 28), EA_ERR_SHAPE),
] + [(f"{s} misaligned", {s: 128 + 4}, EA_ERR_SHAPE)
     for s in ("q_ns", "k_ns", "v_ns", "o_ns", "q_bs", "k_bs", "v_bs", "o_bs")]


@pytest.mark.parametrize("name,kw,status", REJECTED, ids=[r[0] for r in REJECTED])
def test_attention_rejects_before_launch(name, kw, status):
    lib = _lib.load()
    assert lib.ea_attention(C.byref(_args(**kw)), None) == status, name
