"""ctypes binding of ``liboobleck_b200.so`` (C ABI declared in include/oobleck_b200.h).

This is the only place the Python host code touches native code.  There is no fallback: if the library is
missing or a call fails, an exception is raised (the reference's own hot path has no CPU mode either --
``torch.device("cuda")`` is hard-coded at oobleck/execution/pipeline.py:446).
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "liboobleck_b200.so")


class OobleckB200Error(RuntimeError):
    pass


class Planes(C.Structure):
    """``oob_planes``: split 16-bit matrix [nplanes][rows][ld]; format 0 = bf16 planes, 1 = fp16 pair."""
    _fields_ = [("base", C.c_void_p), ("rows", C.c_long), ("cols", C.c_long), ("ld", C.c_long),
                ("plane_stride", C.c_long), ("nplanes", C.c_int), ("format", C.c_int)]


class GemmEpilogue(C.Structure):
    """``oob_gemm_epilogue``."""
    _fields_ = [("d", C.c_void_p), ("ldd", C.c_long), ("bias", C.c_void_p), ("resid", C.c_void_p),
                ("ldr", C.c_long), ("accumulate", C.c_int), ("act", C.c_int), ("aux", C.c_void_p),
                ("ldaux", C.c_long), ("planes", C.c_void_p), ("ldp", C.c_long), ("plane_stride", C.c_long),
                ("nplanes_out", C.c_int), ("alpha", C.c_float)]


class OobDims(C.Structure):
    """``oob_dims``."""
    _fields_ = [("batch", C.c_int), ("seq", C.c_int), ("n_embd", C.c_int), ("n_head", C.c_int), ("vocab", C.c_int),
                ("vocab_padded", C.c_int), ("ln_eps", C.c_float), ("nsplit", C.c_int), ("fwd_fp16", C.c_int),
                ("bwd_fp16", C.c_int), ("loss_scale", C.c_float)]


class OobLayerParams(C.Structure):
    """``oob_layer_params``."""
    _fields_ = [("w", C.c_void_p), ("w_planes", C.c_void_p), ("plane_stride", C.c_long), ("g", C.c_void_p)]


class OobBlockCtx(C.Structure):
    """``oob_block_ctx``."""
    _fields_ = [(n, C.c_void_p) for n in ["ln1_planes", "ln1_mean", "ln1_rstd", "qkv_planes", "att", "att_planes", "lse", "x2",
                                          "ln2_planes", "ln2_mean", "ln2_rstd", "fc", "gelu_planes"]]


class OobBwdScratch(C.Structure):
    """``oob_bwd_scratch``."""
    _fields_ = [(n, C.c_void_p) for n in ["dfc", "dfc_planes", "dln", "dx2", "dx2_planes", "datt", "datt_planes", "delta", "dqkv",
                                          "dqkv_planes", "partials", "partials_side"]] + \
               [("defer_join", C.c_int), ("reserved_", C.c_int)]


class OobHeadCtx(C.Structure):
    """``oob_head_ctx``."""
    _fields_ = [(n, C.c_void_p) for n in ["lnf_planes", "mean", "rstd", "logits", "dlogits_planes", "row_loss", "loss"]]


class LayerProfile(C.Structure):           # oob_layer_profile
    _fields_ = [("forward", C.c_double), ("backward", C.c_double), ("mem_params", C.c_longlong),
                ("mem_activations", C.c_longlong)]


ACT_NONE, ACT_GELU, ACT_DGELU = 0, 1, 2

# plane-set codes of the producers' ``nplanes`` arguments besides 1..3 bf16 planes (include/oobleck_b200.h)
PLANES_BF16X3_FP16_PAIR = 5     # OOB_PLANES_BF16X3_FP16_PAIR: bf16 x 3 followed by the fp16 pair
PLANES_FP16_PAIR = 22           # OOB_PLANES_FP16_PAIR: the fp16 pair only, at planes 0, 1


def planes_count(code: int) -> int:
    """Number of planes a buffer written with plane-set ``code`` holds."""
    return 2 if code == PLANES_FP16_PAIR else code

_P, _L, _I, _F = C.c_void_p, C.c_long, C.c_int, C.c_float
_SIGNATURES = {
    "oob_version": (C.c_int, []),
    "oob_last_error": (C.c_char_p, []),
    "oob_launch_count": (C.c_long, []),
    "oob_plan_pipeline_templates": (C.c_int, [C.POINTER(LayerProfile), C.c_int, C.POINTER(C.c_double), C.c_int, C.c_int,
                                              C.c_int, C.c_int, C.POINTER(C.c_int), C.c_int, C.POINTER(C.c_double),
                                              C.POINTER(C.c_int)]),
    "oob_tensor_map_encodes": (C.c_long, []),
    "oob_gemm_timing_begin": (_I, []),
    "oob_gemm_timing_end": (_I, [C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_double),
                                 C.POINTER(C.c_long)]),
    "oob_ln_bwd_partials_floats": (C.c_long, [_I]),
    "oob_colsum_partials_floats": (C.c_long, [_I]),
    "oob_split_planes": (_I, [_P, _P, _L, _L, _I, _P]),
    "oob_gemm": (_I, [C.POINTER(Planes), _I, C.POINTER(Planes), _I, _I, _I, _I, _I, C.POINTER(GemmEpilogue), _P]),
    "oob_layernorm_fwd": (_I, [_P, _P, _P, _P, _P, _L, _I, _P, _P, _I, _I, _F, _P]),
    "oob_layernorm_bwd": (_I, [_P, _P, _P, _P, _P, _P, _P, _P, _L, _I, _P, _P, _P, _I, _I, _F, _P]),
    "oob_colsum_accumulate": (_I, [_P, _L, _I, _I, _P, _P, _F, _P]),
    "oob_attention_fwd": (_I, [_P, _L, _I, _P, _P, _L, _I, _P, _I, _I, _I, _I, _P]),
    "oob_attention_bwd": (_I, [_P, _L, _I, _P, _P, _P, _L, _P, _P, _P, _P, _L, _I, _I, _I, _I, _I, _P]),
    "oob_embedding_fwd": (_I, [_P, _P, _P, _P, _I, _I, _I, _P]),
    "oob_embedding_bwd": (_I, [_P, _P, _P, _P, _I, _I, _I, _F, _P]),
    "oob_cross_entropy": (_I, [_P, _L, _P, _I, _I, _I, _P, _P, _P, _P, _L, _L, _I, _F, _P]),
    "oob_adamw_step": (_I, [_P, _P, _P, _P, _P, _L, _I, _L, _F, _F, _F, _F, _F, _I, _P]),
    "oob_block_forward": (_I, [C.POINTER(OobDims), C.POINTER(OobLayerParams), _P, _P, C.POINTER(OobBlockCtx), _P]),
    "oob_block_backward": (_I, [C.POINTER(OobDims), C.POINTER(OobLayerParams), _P, C.POINTER(OobBlockCtx), _P, _P,
                                C.POINTER(OobBwdScratch), _P, _P, _P]),
    "oob_head_forward": (_I, [C.POINTER(OobDims), C.POINTER(OobLayerParams), _P, _P, C.POINTER(OobHeadCtx), _P, _P]),
    "oob_head_backward": (_I, [C.POINTER(OobDims), C.POINTER(OobLayerParams), _P, C.POINTER(OobHeadCtx),
                               C.POINTER(OobBwdScratch), _P, _P, _P]),
    "oob_head_eval_partials_floats": (C.c_long, [_I, _I]),
    "oob_head_eval": (_I, [C.POINTER(OobDims), C.POINTER(OobLayerParams), _P, _P, _P, _I, _P, _P, _P, _P, _P, _P, _P]),
    "oob_side_join": (_I, [_P]),
    "oob_side_stream_enable": (_I, [_I]),
    "oob_p2p_header_bytes": (C.c_long, []),
    "oob_p2p_alloc": (_I, [_L, C.POINTER(C.c_void_p), _P]),
    "oob_p2p_open": (_I, [_P, C.POINTER(C.c_void_p)]),
    "oob_p2p_close": (_I, [_P]),
    "oob_p2p_free": (_I, [_P]),
    "oob_p2p_abort": (_I, [_P, _P]),
    "oob_p2p_status": (_I, [_P, C.POINTER(C.c_int)]),
    "oob_p2p_send": (_I, [_P, _L, _P, _P, _I, _L, _L, C.c_uint, _I, _I, _P]),
    "oob_p2p_recv": (_I, [_P, _L, _P, _P, _I, _L, _L, C.c_uint, _I, _I, _P]),
}

_lib = None


def exported_symbols() -> list[str]:
    return list(_SIGNATURES)


def load() -> C.CDLL:
    """Load the library (once).  Raises if it has not been built -- run ``python -c 'import __graft_entry__ as g;
    g.build()'`` or ``make -C oobleck_b200/csrc``."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise OobleckB200Error(f"{LIB_PATH} not found: build the CUDA extension first (no CPU fallback exists)")
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(lib, name)  # AttributeError if a declared symbol is not exported
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        msg = load().oob_last_error().decode(errors="replace")
        raise OobleckB200Error(f"{what} failed ({rc}): {msg}")


def call(name: str, *args) -> None:
    check(getattr(load(), name)(*args), name)
