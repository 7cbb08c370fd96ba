"""ctypes binding of libea_b200.so — the C ABI declared in include/editanything_b200.h.

The product path has NO fallback: if the CUDA extension is missing or fails to initialise,
`lib()` raises.  (The CPU oracle under oracle/ is test infrastructure only and is never
imported from here.)
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# EA_LIB_PATH: development hook - A/B two builds of the library on the same box (tools/r02/build_variants.sh)
LIB_PATH = os.environ.get("EA_LIB_PATH") or os.path.join(_HERE, "lib", "libea_b200.so")

EA_GEMM_LINEAR, EA_GEMM_CONV_S1, EA_GEMM_CONV_S2, EA_GEMM_CONV_S2A = 0, 1, 2, 3
EA_ACT_NONE, EA_ACT_SILU, EA_ACT_GELU, EA_ACT_GEGLU = 0, 1, 2, 3


class GemmArgs(C.Structure):
    _fields_ = [
        ("mode", C.c_int), ("M", C.c_int), ("N", C.c_int), ("K", C.c_int),
        ("a", C.c_void_p), ("lda", C.c_longlong),
        ("w", C.c_void_p), ("ldw", C.c_longlong),
        ("Bsz", C.c_int), ("H", C.c_int), ("W", C.c_int), ("Cin", C.c_int),
        ("a_extra", C.c_void_p), ("Cin_extra", C.c_int), ("ld_extra", C.c_longlong),
        ("bias", C.c_void_p), ("rowvec", C.c_void_p), ("rowvec_ld", C.c_int),
        ("rows_per_batch", C.c_int),
        ("residual", C.c_void_p), ("ldr", C.c_longlong),
        ("out", C.c_void_p), ("ldo", C.c_longlong),
        ("out2", C.c_void_p), ("ldo2", C.c_longlong),
        ("out_f32", C.c_void_p),
        ("act", C.c_int), ("out_scale", C.c_float), ("accumulate", C.c_int),
        ("force_bn", C.c_int), ("force_splits", C.c_int), ("force_2cta", C.c_int), ("no_spin", C.c_int),
        ("force_persistent", C.c_int),
        ("rowstats_out", C.c_void_p), ("ln_stats", C.c_void_p), ("ln_g", C.c_void_p), ("ln_parts", C.c_int),
        ("ln_eps", C.c_float), ("row_scale", C.c_void_p),
        ("prefetch", C.c_void_p * 3), ("prefetch_bytes", C.c_longlong * 3),
        ("workspace", C.c_void_p), ("workspace_bytes", C.c_longlong),
    ]


class AttnArgs(C.Structure):
    _fields_ = [
        ("q", C.c_void_p), ("k", C.c_void_p), ("v", C.c_void_p), ("out", C.c_void_p),
        ("B", C.c_int), ("heads", C.c_int), ("Nq", C.c_int), ("Nkv", C.c_int), ("d", C.c_int),
        ("q_bs", C.c_longlong), ("q_ns", C.c_longlong), ("k_bs", C.c_longlong), ("k_ns", C.c_longlong),
        ("v_bs", C.c_longlong), ("v_ns", C.c_longlong), ("o_bs", C.c_longlong), ("o_ns", C.c_longlong),
        ("scale", C.c_float),
        ("rel_h", C.c_void_p), ("rel_w", C.c_void_p), ("rel_s", C.c_int),
    ]


class GnArgs(C.Structure):
    _fields_ = [
        ("x", C.c_void_p), ("ldx", C.c_longlong), ("C1", C.c_int),
        ("x2", C.c_void_p), ("ldx2", C.c_longlong),
        ("gamma", C.c_void_p), ("beta", C.c_void_p),
        ("out", C.c_void_p), ("ldo", C.c_longlong),
        ("B", C.c_int), ("HW", C.c_int), ("C", C.c_int), ("groups", C.c_int),
        ("eps", C.c_float), ("silu", C.c_int), ("two_pass", C.c_int),
        ("workspace", C.c_void_p),
        ("n_nets", C.c_int), ("gamma_more", C.c_void_p * 2), ("beta_more", C.c_void_p * 2),
    ]


# every symbol include/editanything_b200.h declares: name -> (restype, argtypes)
_P, _I, _L, _F = C.c_void_p, C.c_int, C.c_longlong, C.c_float
SYMBOLS = {
    "ea_version": (_I, []),
    "ea_dtype_name": (C.c_char_p, []),
    "ea_strerror": (C.c_char_p, [_I]),
    "ea_init": (_I, []),
    "ea_last_error": (C.c_char_p, []),
    "ea_launch_count": (_L, []),
    "ea_reset_launch_count": (None, []),
    "ea_set_pdl": (None, [_I]),
    "ea_gemm": (_I, [C.POINTER(GemmArgs), _P]),
    "ea_gemm_grouped": (_I, [C.POINTER(GemmArgs), _I, _P]),
    "ea_gemm_plan": (_I, [_I, _I, _I, _I, _L, _I, C.POINTER(C.c_int)]),
    "ea_attention": (_I, [C.POINTER(AttnArgs), _P]),
    "ea_groupnorm": (_I, [C.POINTER(GnArgs), _P]),
    "ea_layernorm": (_I, [_P, _L, _P, _P, _P, _L, _I, _I, _F, _P]),
    "ea_conv_direct": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _P, _L, _P]),
    "ea_conv_in": (_I, [_P, _P, _P, _P, _L, _P, _L, _P, _I, _I, _I, _I, _I, _P]),
    "ea_upsample2x": (_I, [_P, _P, _I, _I, _I, _I, _P]),
    "ea_small_linear": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _P]),
    "ea_timestep_embedding": (_I, [_P, _P, _I, _I, _P]),
    "ea_out_cfg_ddim": (_I, [_P, _P, _P, _P, _P, _P, _F, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _P]),
    "ea_out_ddim": (_I, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _P]),
    "ea_out_cfg_vpred": (_I, [_P, _P, _P, _P, _P, _P, _F, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _P]),
    "ea_out_vpred": (_I, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _P]),
    "ea_latent_mix": (_I, [_P, _P, _P, _P, _P, _F, _P, _I, _P, _I, _I, _I, _I, _P]),
    "ea_step_gather": (_I, [_P, _I, _I, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.POINTER(C.c_longlong), _P]),
    "ea_sam_relpos": (_I, [_P, _L, _L, _P, _P, _P, _P, _I, _I, _I, _I, _P]),
    "ea_window_partition": (_I, [_P, _P, _I, _I, _I, _I, _I, _P]),
    "ea_window_unpartition": (_I, [_P, _P, _P, _I, _I, _I, _I, _I, _P]),
    "ea_sam_patchify": (_I, [_P, _P, _I, _I, _I, _I, _I, _P]),
    "ea_nhwc_to_nchw_f32": (_I, [_P, _P, _I, _I, _I, _P]),
    "ea_softmax_rows": (_I, [_P, _L, _P, _L, _I, _I, _P]),
    "ea_image_out": (_I, [_P, _L, _P, _I, _L, _I, _F, _F, _F, _F, _P]),
}

_lib = None
_inited = False


def load():
    """dlopen the library and bind every declared symbol (no GPU needed)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing: build it with `python -m editanything_b200.csrc.build` "
                "(there is no CPU fallback)")
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in SYMBOLS.items():
            fn = getattr(lib, name)  # AttributeError if the .so does not export it
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


def lib():
    """Library handle, initialised for compute (requires an H100)."""
    global _inited
    l = load()
    if not _inited:
        st = l.ea_init()
        if st != 0:
            raise RuntimeError("libea_b200 init failed: " + l.ea_strerror(st).decode())
        _inited = True
    return l


def check(status, what=""):
    if status != 0:
        detail = load().ea_last_error().decode() if status == -4 else ""
        raise RuntimeError(f"libea_b200 {what} failed: {load().ea_strerror(status).decode()} ({status})" +
                           (f" [{detail}]" if detail else ""))
