"""The operator calls of DenoiseEngine on the CPU emulation (tests/cpu_ops.py): every call made by prepare(), one step
(t, a_t, a_prev) without a CUDA graph and one eps(), with each tensor argument's shape, dtype, storage (numbered in
order of first appearance), offset and strides.  tests/golden/step_trace.json keeps, per case and section, the number
of calls and the SHA-256 of the trace.  The ops backend launches one kernel per call on the buffers it is given, so an
equal trace means the GPU runs the same launches on the same buffers: a change to the host-side encoder paths that
keeps this trace leaves the device work unchanged.

    python -m tests.test_step_trace_cpu          # re-record the golden digests from the current code
    python -m tests.test_step_trace_cpu DIR      # write the full traces to DIR/<case>.txt (to diff two commits)
"""
import hashlib
import inspect
import json
import os
import sys

import pytest
import torch

from editanything_b200.denoise import DenoiseEngine, ddim_schedule
from editanything_b200.unet_spec import TINY, TINY21, TINY21_INPAINT, make_state_dict
from oracle.inputs import make_inputs
from tests import cpu_ops

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "step_trace.json")
ENV = ("EA_LOCKSTEP", "EA_LN_FOLD", "EA_CONCURRENT", "EA_HINT_TC")

# name: (config, ControlNets, environment, conditioning scales, guess mode)
CASES = {
    "tiny_cn0": (TINY, 0, {}, [], False),
    "tiny_cn1": (TINY, 1, {}, [0.8], False),
    "tiny_cn2": (TINY, 2, {}, [0.5, 1.0], False),
    "tiny_cn3_sequential": (TINY, 3, {}, [0.5, 1.0, 0.7], False),
    "tiny_cn2_no_lockstep": (TINY, 2, {"EA_LOCKSTEP": "0"}, [0.5, 1.0], False),
    "tiny_cn2_no_ln_fold": (TINY, 2, {"EA_LN_FOLD": "0"}, [0.5, 1.0], False),
    "tiny21_inpaint_cn1": (TINY21_INPAINT, 1, {}, [0.9], False),
    "tiny_cn2_guess_mode": (TINY, 2, {}, [0.7, 1.0], True),
    "tiny_cn2_scale_map": (TINY, 2, {}, ["map", 0.5], False),
}


class Recorder:
    """An ops backend that runs tests/cpu_ops.py and writes one line per call: the operator and its arguments, tensors
    as #storage+offset, dtype (f = float32, h = float16, b = bfloat16, i = int32), [shape], and /strides when they are
    not the contiguous ones."""

    def __init__(self):
        self.lines, self._storages, self._alive = [], {}, []

    def __getattr__(self, name):
        fn = getattr(cpu_ops, name)
        if not callable(fn):
            return fn

        def call(*args, **kw):
            if name == "gemm_grouped":
                text = "; ".join(self._args(cpu_ops.gemm, (a, w, out), k) for a, w, out, k in args[0])
            else:
                text = self._args(fn, args, kw)
            self.lines.append(f"{name}({text})")
            return fn(*args, **kw)
        return call

    def _args(self, fn, args, kw):
        """Required arguments by position, the others as name=value when they differ from the default."""
        sig = inspect.signature(fn)
        bound = sig.bind(*args, **kw)
        bound.apply_defaults()
        out = []
        for n, v in bound.arguments.items():
            p = sig.parameters[n]
            if p.default is inspect.Parameter.empty:
                out.append(self._fmt(v))
            elif self._fmt(v) != self._fmt(p.default):
                out.append(f"{n}={self._fmt(v)}")
        return ",".join(out)

    def _fmt(self, v):
        if torch.is_tensor(v):
            st = v.untyped_storage()
            sid = self._storages.setdefault(st.data_ptr(), len(self._storages))
            self._alive.append(st)           # a freed storage's address must not come back as a "new" buffer
            dt = {torch.float32: "f", torch.float16: "h", torch.bfloat16: "b", torch.int32: "i"}.get(v.dtype, v.dtype)
            shape = ",".join(map(str, v.shape))
            dense = torch.empty(v.shape, device="meta").stride()
            strides = "" if v.stride() == dense else "/" + ",".join(map(str, v.stride()))
            return f"#{sid}+{v.storage_offset()}{dt}[{shape}{strides}]"
        if isinstance(v, (list, tuple)):
            s = ",".join(self._fmt(x) for x in v)
            return f"[{s}]" if isinstance(v, list) else f"({s})"
        if isinstance(v, dict):
            return "{" + ",".join(f"{k}:{self._fmt(x)}" for k, x in v.items()) + "}"
        return repr(v)


def record(name, swap=False):
    """The trace of one case; the EA_* switches must already be set as the case asks.  swap: build the engine on
    cpu_ops and put the recorder in afterwards, the way bench.py swaps in its GEMM probe."""
    cfg, n_cn, _, scales, guess = CASES[name]
    usd = make_state_dict(cfg, "unet", 61)
    csds = [make_state_dict(TINY21 if cfg is TINY21_INPAINT else cfg, "controlnet", 62 + i) for i in range(n_cn)]
    x, ctx, hints = make_inputs(cfg, 2, 8, 7, 5, n_controlnets=2)
    hints = (hints + [hints[0].flip(-1)])[:n_cn]
    scales = [torch.rand(8, 8, generator=torch.Generator().manual_seed(9)) if s == "map" else s for s in scales]
    rec = Recorder()
    eng = DenoiseEngine(cfg, usd, csds, torch.device("cpu"), backend=cpu_ops if swap else rec)
    if swap:
        eng.ops = eng.runner.ops = eng.unet.ops = rec
        for c in eng.cns:
            c.ops = rec
    rec.lines, rec._storages, rec._alive = [], {}, []
    ts, a, ap = ddim_schedule(50)
    rec.lines.append("== prepare")
    eng.prepare(ctx, hints, scales, guess_mode=guess)
    if cfg.in_channels == 9:
        rec.lines.append("== set_unet_condition")
        eng.set_unet_condition(x[:1, 4:5], x[:1, 5:9])
    rec.lines.append("== step")
    eng.begin(x[:1, :4], guidance=7.5, use_graph=False)
    eng.step(int(ts[2]), float(a[2]), float(ap[2]))
    rec.lines.append("== eps")
    eng.eps(x, int(ts[5]))
    return rec.lines


def _set_env(mp, name):
    for k in ENV:
        mp.delenv(k, raising=False)
    for k, v in CASES[name][2].items():
        mp.setenv(k, v)


def digest(lines):
    """Per section of the trace (prepare, set_unet_condition, step, eps): the number of calls and the SHA-256 of
    their lines."""
    sections, name = {}, None
    for line in lines:
        if line.startswith("== "):
            name = line[3:]
            sections[name] = []
        else:
            sections[name].append(line)
    return {k: {"calls": len(v), "sha256": hashlib.sha256("\n".join(v).encode()).hexdigest()}
            for k, v in sections.items()}


def _check(name, got, tmp_path):
    with open(GOLDEN) as f:
        want = json.load(f)[name]
    if digest(got) != want:
        path = tmp_path / f"{name}.txt"
        path.write_text("\n".join(got) + "\n")
        raise AssertionError(f"{name}: trace differs from the golden digest {want}; this trace is in {path}, "
                             f"`python -m tests.test_step_trace_cpu DIR` on the parent commit writes the expected one")


@pytest.mark.parametrize("name", list(CASES))
def test_step_trace_matches_golden(name, monkeypatch, tmp_path):
    _set_env(monkeypatch, name)
    _check(name, record(name), tmp_path)


@pytest.mark.parametrize("name", ["tiny_cn2", "tiny_cn3_sequential"])
def test_operator_table_swapped_after_construction_sees_every_call(name, monkeypatch, tmp_path):
    _set_env(monkeypatch, name)
    _check(name, record(name, swap=True), tmp_path)


if __name__ == "__main__":
    # no argument: re-record the golden digests; DIR: write every case's full trace to DIR/<case>.txt
    out = sys.argv[1] if len(sys.argv) > 1 else None
    digests = {}
    for case in CASES:
        with pytest.MonkeyPatch.context() as mp:
            _set_env(mp, case)
            lines = record(case)
        digests[case] = digest(lines)
        if out:
            os.makedirs(out, exist_ok=True)
            with open(os.path.join(out, case + ".txt"), "w") as f:
                f.write("\n".join(lines) + "\n")
    if not out:
        with open(GOLDEN, "w") as f:
            f.write("{\n" + ",\n".join(f"{json.dumps(k)}: {json.dumps(v)}" for k, v in digests.items()) + "\n}\n")
    print({k: sum(s["calls"] for s in v.values()) for k, v in digests.items()})
