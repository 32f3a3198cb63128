"""ctypes binding of libprisma_b200.so -- the only door to the CUDA path.

Mirrors include/prisma_b200.h structure-for-structure.  There is deliberately no alternative
implementation behind these functions: if the shared library is missing or no GPU is visible,
calls raise ``PrismaB200Error`` -- nothing silently runs on the CPU or through ATen.
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

PKG_ROOT = Path(__file__).resolve().parents[2]          # .../vit-prisma_b200
LIB_PATH = Path(os.environ.get("PRISMA_B200_LIB", PKG_ROOT / "lib" / "libprisma_b200.so"))

PB_OK, PB_EINVAL, PB_ECUDA, PB_EUNSUPPORTED, PB_ENODEVICE = 0, -1, -2, -3, -4
PB_F32, PB_BF16 = 0, 1
ACT = {None: 0, "none": 0, "relu": 1, "gelu": 2, "silu": 3, "gelu_new": 4, "gelu_fast": 5,
       "quick_gelu": 6, "tanh-relu": 7, "exp": 8}
GEMM_AUTO, GEMM_SIMT, GEMM_TC = 0, 1, 2

vp, i32, i64, f32 = C.c_void_p, C.c_int32, C.c_int64, C.c_float


class PrismaB200Error(RuntimeError):
    pass


class PbGemm(C.Structure):
    _fields_ = [
        ("M", i32), ("N", i32), ("K", i32), ("dtype", i32), ("act", i32), ("impl", i32),
        ("A", vp), ("lda", i64), ("B", vp), ("ldb", i64), ("A_lo", vp), ("B_lo", vp),
        ("bias", vp), ("residual", vp), ("ldr", i64),
        ("out0", vp), ("ld0", i64), ("out1", vp), ("ld1", i64), ("out1_lo", vp),
        ("n_split", i32), ("split_n", i32), ("out_split", vp * 4),
    ]


class PbLayerNorm(C.Structure):
    _fields_ = [
        ("rows", i64), ("cols", i32), ("dtype_in", i32), ("dtype_out", i32), ("eps", f32),
        ("x", vp), ("w", vp), ("b", vp), ("scale", vp), ("norm_f32", vp), ("out", vp), ("out_lo", vp),
        ("scale_in", vp),
    ]


class PbAttention(C.Structure):
    _fields_ = [
        ("B", i32), ("T", i32), ("H", i32), ("dh", i32), ("dtype", i32), ("attn_scale", f32),
        ("q", vp), ("k", vp), ("v", vp), ("scores", vp), ("pattern", vp), ("z", vp),
        ("causal", i32),
    ]


class PbVitLayerW(C.Structure):
    _fields_ = [(n, vp) for n in (
        "ln1_w", "ln1_b", "wqkv", "wqkv_lo", "bqkv", "wo", "wo_lo", "bo",
        "ln2_w", "ln2_b", "win", "win_lo", "bin", "wout", "wout_lo", "bout")]


class PbVitLayerSpill(C.Structure):
    _fields_ = [(n, vp) for n in (
        "ln1_scale", "ln1_norm_f32", "ln1_out", "q", "k", "v", "scores", "pattern", "z",
        "attn_out", "resid_mid", "ln2_scale", "ln2_norm_f32", "ln2_out", "pre", "post",
        "mlp_out", "resid_post")]


class PbVitForward(C.Structure):
    _fields_ = (
        [(n, i32) for n in (
            "batch", "n_channels", "image_size", "patch_size", "n_patches", "n_tokens",
            "d_model", "n_heads", "d_head", "d_mlp", "n_classes", "n_layers_run", "run_head",
            "use_cls", "layer_norm_pre", "normalize_output", "head_proj", "pool_gaap",
            "act", "dtype", "gemm_impl")]
        + [("eps", f32), ("attn_scale", f32)]
        + [(n, vp) for n in (
            "images", "patch_w", "patch_w_lo", "patch_b", "cls", "pos",
            "lnpre_w", "lnpre_b", "lnf_w", "lnf_b", "head_w", "head_w_lo", "head_b")]
        + [("layers_host", C.POINTER(PbVitLayerW))]
        + [(n, vp) for n in (
            "patches", "embed", "full_embed", "lnpre_scale", "lnpre_norm_f32", "lnpre_out")]
        + [("spills_host", C.POINTER(PbVitLayerSpill))]
        + [(n, vp) for n in (
            "lnf_scale", "lnf_norm_f32", "lnf_out", "pooled", "pre_normalize", "out", "lo_scratch")]
        + [("n_frames", i32), ("tubelet_depth", i32)]
    )


class PbTextForward(C.Structure):
    _fields_ = (
        [(n, i32) for n in (
            "batch", "n_tokens", "vocab", "d_model", "n_heads", "d_head", "d_mlp", "n_classes", "n_layers",
            "causal", "normalize_output", "head_proj", "act", "dtype", "gemm_impl")]
        + [("eps", f32), ("attn_scale", f32), ("ids", vp)]
        + [(n, vp) for n in ("token_w", "pos", "lnf_w", "lnf_b", "head_w", "head_w_lo", "head_b")]
        + [("layers_host", C.POINTER(PbVitLayerW)), ("embed", vp), ("full_embed", vp),
           ("spills_host", C.POINTER(PbVitLayerSpill))]
        + [(n, vp) for n in ("lnf_scale", "lnf_norm_f32", "lnf_out", "pooled", "pre_normalize", "out", "lo_scratch")]
    )


# index == argument of pb_abi_sizeof(); the layout test walks this list
ABI_STRUCTS = [PbGemm, PbLayerNorm, PbAttention, PbVitLayerW, PbVitLayerSpill, PbVitForward]
# indices past the SAE / peer-memory structs that sae_engine.py and p2p.py append (6-9)
ABI_TEXT_FORWARD = 10

# name -> (restype, argtypes); also the list the "exports every declared symbol" test walks
SIGNATURES = {
    "pb_version": (i32, []),
    "pb_last_error": (C.c_char_p, []),
    "pb_device_info": (i32, [C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "pb_abi_sizeof": (i32, [i32]),
    "pb_launch_count": (C.c_ulonglong, []),
    "pb_gemm": (i32, [C.POINTER(PbGemm), vp]),
    "pb_split_tf32": (i32, [vp, vp, i64, vp]),
    "pb_layernorm": (i32, [C.POINTER(PbLayerNorm), vp]),
    "pb_attention": (i32, [C.POINTER(PbAttention), vp]),
    "pb_attn_scores": (i32, [C.POINTER(PbAttention), vp]),
    "pb_softmax_rows": (i32, [vp, vp, i64, i32, i32, vp]),
    "pb_attn_pv": (i32, [C.POINTER(PbAttention), vp]),
    "pb_add": (i32, [vp, vp, vp, i64, i32, vp]),
    "pb_mul": (i32, [vp, vp, vp, i64, i32, vp]),
    "pb_activation": (i32, [vp, vp, i64, i32, i32, vp]),
    "pb_l2_normalize_rows": (i32, [vp, vp, i64, i32, f32, i32, vp]),
    "pb_mean_tokens": (i32, [vp, vp, i32, i32, i32, i32, vp]),
    "pb_im2col_patches": (i32, [vp, vp, i32, i32, i32, i32, i32, vp]),
    "pb_im2col_tubelets": (i32, [vp, vp, i32, i32, i32, i32, i32, i32, i32, vp]),
    "pb_embed_assemble": (i32, [vp, vp, vp, vp, i32, i32, i32, i32, i32, vp]),
    "pb_cast": (i32, [vp, i32, vp, i32, i64, vp]),
    "pb_embed_tokens": (i32, [vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, vp]),
    "pb_gather_argmax_rows": (i32, [vp, vp, vp, i32, i32, i32, i32, vp]),
    "pb_vit_forward": (i32, [C.POINTER(PbVitForward), vp]),
    "pb_text_forward": (i32, [C.POINTER(PbTextForward), vp]),
}

_lib = None


def register_signatures(extra: dict) -> None:
    """Other binding modules (sae, p2p) add their entry points here before first use."""
    SIGNATURES.update(extra)
    if _lib is not None:
        _bind(_lib, extra)


def _bind(lib, table) -> None:
    for name, (restype, argtypes) in table.items():
        fn = getattr(lib, name)          # AttributeError here == header/library mismatch
        fn.restype = restype
        fn.argtypes = argtypes


def get_lib():
    global _lib
    if _lib is None:
        if not LIB_PATH.exists():
            raise PrismaB200Error(
                f"{LIB_PATH} not found. Build it with `python vit-prisma_b200/build.py` "
                "(or __graft_entry__.build()); there is no CPU/ATen fallback for the hot path.")
        lib = C.CDLL(str(LIB_PATH))
        _bind(lib, SIGNATURES)
        _lib = lib
    return _lib


def last_error() -> str:
    msg = get_lib().pb_last_error()
    return msg.decode("utf-8", "replace") if msg else ""


def check(rc: int, what: str = "") -> None:
    if rc != PB_OK:
        kind = {PB_EINVAL: "invalid argument", PB_ECUDA: "CUDA error", PB_EUNSUPPORTED: "unsupported",
                PB_ENODEVICE: "no CUDA device"}.get(rc, f"error {rc}")
        raise PrismaB200Error(f"libprisma_b200 {what}: {kind}: {last_error()}")


def device_info():
    sm, major, minor = C.c_int(0), C.c_int(0), C.c_int(0)
    check(get_lib().pb_device_info(C.byref(sm), C.byref(major), C.byref(minor)), "pb_device_info")
    return sm.value, major.value, minor.value
