"""ctypes binding of libidiff_b200.so (include/idiff_b200.h).

The library is the product; there is no CPU or torch fallback.  If the shared object is missing
or a CUDA call fails, an exception is raised -- loudly.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libidiff_b200.so")
# The same sources compiled for each 16-bit storage type (include/idiff_b200.h: idiff_storage_dtype)
LIB_PATHS = {"f16": LIB_PATH, "bf16": os.path.join(_HERE, "csrc", "libidiff_b200_bf16.so")}
DTYPE_CODES = {"f16": 0, "bf16": 1}


class IdiffError(RuntimeError):
    pass


class GemmArgs(C.Structure):
    _fields_ = [
        ("a", C.c_void_p), ("w", C.c_void_p), ("out", C.c_void_p), ("bias", C.c_void_p),
        ("rowadd", C.c_void_p), ("residual", C.c_void_p), ("gate", C.c_float),
        ("M", C.c_int), ("N", C.c_int), ("K", C.c_int),
        ("lda", C.c_int), ("ldw", C.c_int), ("ldo", C.c_int), ("ldr", C.c_int), ("ldra", C.c_int),
        ("rows_per_batch", C.c_int), ("flags", C.c_int),
        ("conv_b", C.c_int), ("conv_h", C.c_int), ("conv_w", C.c_int), ("conv_cin", C.c_int),
        ("workspace", C.c_void_p), ("workspace_bytes", C.c_long),
        ("ln_stats_out", C.c_void_p), ("ln_stats_in", C.c_void_p), ("ln_colsum", C.c_void_p),
        ("ln_slots_in", C.c_int), ("ln_eps", C.c_float),
        ("gate_b", C.c_void_p),
    ]


class AttnArgs(C.Structure):
    _fields_ = [
        ("q", C.c_void_p), ("k0", C.c_void_p), ("v0", C.c_void_p), ("k1", C.c_void_p), ("v1", C.c_void_p),
        ("out", C.c_void_p),
        ("q_ld", C.c_int), ("k0_ld", C.c_int), ("v0_ld", C.c_int), ("k1_ld", C.c_int), ("v1_ld", C.c_int),
        ("out_ld", C.c_int),
        ("batch", C.c_int), ("heads", C.c_int), ("head_dim", C.c_int),
        ("nq", C.c_int), ("n0", C.c_int), ("n1", C.c_int), ("kv1_batch", C.c_int),
        ("scale", C.c_float),
        ("mask_q", C.c_void_p), ("mask_k", C.c_void_p),
    ]


EPI_GEGLU = 1
EPI_SILU = 2
OUT_F32_NCHW = 4
EPI_GELU = 8

# name -> (restype, argtypes); the exported surface of include/idiff_b200.h
_vp, _i, _f, _l = C.c_void_p, C.c_int, C.c_float, C.c_long
SIGNATURES = {
    "idiff_last_error": (C.c_char_p, []),
    "idiff_version": (_i, []),
    "idiff_storage_dtype": (_i, []),
    "idiff_set_batch_invariant": (_i, [_i]),
    "idiff_gemm": (_i, [C.POINTER(GemmArgs), _vp]),
    "idiff_gemm_ln_slots": (_i, [C.POINTER(GemmArgs)]),
    "idiff_row_stats": (_i, [_vp, _vp, _i, _i, _vp]),
    "idiff_gemm_workspace_bytes": (_l, []),
    "idiff_set_gemm_workspace": (_i, [_vp, _l]),
    "idiff_set_gemm_trace": (_i, [_vp]),
    "idiff_attention": (_i, [C.POINTER(AttnArgs), _vp]),
    "idiff_groupnorm": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _f, _i, _vp]),
    "idiff_groupnorm_ws_floats": (_l, [_i, _i]),
    "idiff_scaleu_ws_floats": (_l, [_i, _i]),
    "idiff_layernorm": (_i, [_vp, _vp, _vp, _vp, _i, _i, _f, _vp]),
    "idiff_scaleu_concat": (_i, [_vp, _vp, _vp, _vp, _f, _vp, _i, _i, _i, _i, _i, _vp]),
    "idiff_nchw_f32_to_nhwc_f16": (_i, [_vp, _vp, _i, _i, _i, _i, _vp]),
    "idiff_nhwc_f16_to_nchw_f32": (_i, [_vp, _vp, _i, _i, _i, _vp]),
    "idiff_upsample_nearest2x": (_i, [_vp, _vp, _i, _i, _i, _i, _vp]),
    "idiff_im2col_s2": (_i, [_vp, _vp, _i, _i, _i, _i, _vp]),
    "idiff_im2col_s2_pad01": (_i, [_vp, _vp, _i, _i, _i, _i, _vp]),
    "idiff_fourier_embed": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp]),
    "idiff_plms_update": (_i, [_vp, _vp, _vp, _f, _vp, _vp, _vp, _f, _f, _f, _f, _f, _f, _f, _vp, _vp, _l, _vp]),
    "idiff_ddim_update": (_i, [_vp, _vp, _vp, _f, _f, _f, _f, C.c_uint64, _i, _vp, _vp, _l, _vp]),
    "idiff_dpmpp2m_update": (_i, [_vp, _vp, _vp, _f, _vp, _f, _f, _f, _f, _f, _f, _vp, _vp, _l, _vp]),
    "idiff_noise_latent": (_i, [_vp, _l, _f, _f, C.c_uint64, _vp, _l, _vp]),
    "idiff_inpaint_blend": (_i, [_vp, _vp, _i, _vp, _vp, _i, _i, _i, _i, _l, _f, _f, C.c_uint64, _i, _vp]),
    "idiff_latent_mean": (_i, [_vp, _i, _vp, _l, _vp]),
    "idiff_conv_in_select": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "idiff_encode_image_in": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "idiff_timestep_embedding": (_i, [_vp, _vp, _i, _i, _vp]),
    "idiff_silu_f16": (_i, [_vp, _vp, _l, _vp]),
    "idiff_segs_inconv": (_i, [_vp, C.POINTER(C.c_long), _vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "idiff_patchify": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _vp]),
    "idiff_dwconv7x7": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "idiff_seg_tokens": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "idiff_boxes_to_attmask": (_i, [_vp, _vp, _vp, _i, _i, _i, _vp]),
    "idiff_attmask_words": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "idiff_vae_latent_in": (_i, [_vp, _vp, _vp, _f, _vp, _i, _i, _i, _vp]),
    "idiff_softmax_rows": (_i, [_vp, _i, _i, _l, _vp]),
    "idiff_decode_to_image": (_i, [_vp, _i, _vp, _i, _l, _vp]),
    "idiff_encode_posterior": (_i, [_vp, _vp, _vp, _f, _vp, _vp, _vp, _i, _l, _vp]),
    "idiff_embed_tokens": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "idiff_causal_attention_small": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _f, _vp]),
}

_libs = {}
_storage = "f16"  # which build load() returns; switched by ops.set_storage_dtype
_batch_invariant = False  # idiff_set_batch_invariant of every loaded build; switched by ops.set_batch_invariant


def set_batch_invariant(on: bool) -> None:
    """Set the mode in every build loaded so far; load() sets it in builds loaded later."""
    global _batch_invariant
    _batch_invariant = bool(on)
    for lib in _libs.values():
        lib.idiff_set_batch_invariant(int(_batch_invariant))


def set_storage(kind: str) -> None:
    global _storage
    if kind not in LIB_PATHS:
        raise IdiffError(f"unknown storage type {kind!r} (have {sorted(LIB_PATHS)})")
    _storage = kind


def storage() -> str:
    return _storage


def load(kind: str | None = None) -> C.CDLL:
    """Load the shared library of the current (or the named) storage type; raises if it has not been built."""
    kind = kind or _storage
    lib = _libs.get(kind)
    if lib is not None:
        return lib
    path = LIB_PATHS[kind]
    if not os.path.exists(path):
        raise IdiffError(
            f"{path} not found: the sm_90a CUDA library is required (no fallback). "
            "Build it with `python -m instancediffusion_b200.build` or __graft_entry__.build()."
        )
    lib = C.CDLL(path)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is missing
        fn.restype = res
        fn.argtypes = args
    if lib.idiff_storage_dtype() != DTYPE_CODES[kind]:
        raise IdiffError(f"{path} was not built for {kind} storage")
    lib.idiff_set_batch_invariant(int(_batch_invariant))
    _libs[kind] = lib
    return lib


def check(rc: int, what: str) -> None:
    if rc != 0:
        msg = load().idiff_last_error().decode("utf-8", "replace")
        raise IdiffError(f"{what} failed (rc={rc}): {msg}")
