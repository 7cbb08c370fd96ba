"""Build libea_b200.so (sm_90a only) in-tree with nvcc.  Usage: python -m editanything_b200.csrc.build"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
PKG = os.path.dirname(HERE)
LIB = os.path.join(PKG, "lib", "libea_b200.so")
SOURCES = ["ea_api.cu", "ea_gemm.cu", "ea_attn.cu", "ea_pointwise.cu"]
HEADERS = ["ea_common.cuh", "ea_wgmma.cuh", "ea_internal.h", os.path.join("..", "..", "include", "editanything_b200.h")]


def _stale():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    for f in SOURCES + HEADERS + ["build.py"]:
        if os.path.getmtime(os.path.join(HERE, f)) > t:
            return True
    return False


def build(force=False, verbose=False, extra=()):
    """Compile every .cu for sm_90a into editanything_b200/lib/libea_b200.so."""
    if os.environ.get("EA_NVCC_EXTRA"):
        force = True
    if not force and not _stale():
        return LIB
    os.makedirs(os.path.dirname(LIB), exist_ok=True)
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    objs = []
    procs = []
    for src in SOURCES:
        obj = os.path.join(PKG, "lib", src.replace(".cu", ".o"))
        cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
               "-Xcompiler", "-fPIC", "--use_fast_math" if False else "-DEA_PRECISE_MATH",
               "-c", os.path.join(HERE, src), "-o", obj] + list(extra) + os.environ.get("EA_NVCC_EXTRA", "").split()
        if verbose:
            cmd.insert(1, "-Xptxas")
            cmd.insert(2, "-v")
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode != 0:
            sys.stderr.write(out)
        if p.returncode != 0:
            failed = True
    if failed:
        raise RuntimeError("nvcc failed")
    cmd = [nvcc, "-shared", "-o", LIB] + objs + ["-cudart", "static"]
    subprocess.check_call(cmd)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
