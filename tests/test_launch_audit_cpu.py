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
    assert f"ops.{op} " in msg and operand in msg.split("operand ", 1)[1].split(":", 1)[0].split("/"), msg
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
