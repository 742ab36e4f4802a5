"""ctypes binding of include/bagel_b200.h. There is NO fallback: if the library is missing or a call fails,
this raises. The product path never routes around the CUDA kernels."""
from __future__ import annotations

import ctypes as C
import re
from pathlib import Path

_PKG = Path(__file__).resolve().parent
LIB_PATH = _PKG / "libbagel_b200.so"
HEADER_PATH = _PKG.parent / "include" / "bagel_b200.h"

_lib = None


class BagelB200Error(RuntimeError):
    pass


_vp, _ll, _i, _f = C.c_void_p, C.c_longlong, C.c_int, C.c_float

# name -> (restype, argtypes); must mirror include/bagel_b200.h (tests/test_cabi.py cross-checks the names)
SIGNATURES = {
    "bagel_last_error": (C.c_char_p, []),
    "bagel_abi_version": (_i, []),
    "bagel_launch_count": (_ll, []),
    "bagel_gemm_bf16": (_i, [_vp, _ll, _vp, _ll, _vp, _ll, _i, _i, _i, _vp, _vp, _ll, _vp, _i, _vp]),
    "bagel_quantize_fp8_bf16": (_i, [_vp, _ll, _vp, _ll, _vp, _ll, _i, _i, _i, _vp]),
    "bagel_gemm_fp8": (_i, [_vp, _ll, _vp, _ll, _vp, _ll, _vp, _vp, _ll, _i, _i, _i, _vp, _ll, _i, _vp]),
    "bagel_gemm_qkv_norm_rope": (_i, [_vp, _ll, _vp, _ll, _vp, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _ll,
                                      _vp, _vp, _ll, _vp, _i, _i, _f, _i, _vp]),
    "bagel_attn_varlen_fwd": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _f,
                                   _ll, _ll, _ll, _ll, _vp, _vp]),
    "bagel_decode_prepare": (_i, [_vp, _vp, _vp, _vp, _i, _vp]),
    "bagel_argmax_rows_bf16": (_i, [_vp, _ll, _i, _i, _vp, _vp, _vp]),
    "bagel_decode_advance": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _vp]),
    "bagel_sample_rows_bf16": (_i, [_vp, _ll, _i, _i, _f, _vp, _vp, _vp, _vp, _vp]),
    "bagel_decode_advance_stop": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _ll, _i, _ll, _i, _vp]),
    "bagel_rmsnorm_bf16": (_i, [_vp, _ll, _vp, _vp, _vp, _vp, _ll, _i, _i, _f, _vp]),
    "bagel_layernorm_bf16": (_i, [_vp, _ll, _vp, _vp, _vp, _ll, _i, _i, _f, _vp]),
    "bagel_rope_table": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "bagel_qk_norm_rope": (_i, [_vp, _ll, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _ll, _vp, _vp, _ll, _vp,
                                _i, _i, _i, _i, _f, _i, _vp]),
    "bagel_copy_rows_bf16": (_i, [_vp, _ll, _vp, _vp, _ll, _vp, _i, _i, _vp]),
    "bagel_latent_embed_add": (_i, [_vp, _ll, _vp, _vp, _ll, _vp, _vp, _ll, _vp, _i, _i, _vp]),
    "bagel_cfg_euler_step": (_i, [_vp, _vp, _vp, _ll, _vp, _vp, _vp, _i, _i, _f, _f, _f, _i, _f, _vp, _vp]),
    "bagel_cfg_euler_step_batch": (_i, [_vp, _ll, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                        _vp]),
    "bagel_cast_f32_to_bf16": (_i, [_vp, _vp, _ll, _vp]),
    "bagel_conv2d_nhwc_bf16": (_i, [_vp, _i, _i, _i, _i, _vp, _i, _i, _i, _i, _vp, _vp, _vp, _i, _i, _vp]),
    "bagel_groupnorm_workspace_bytes": (_ll, [_i, _i]),
    "bagel_groupnorm_nhwc_bf16": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _ll, _i, _i, _f, _i, _vp]),
    "bagel_upsample2x_nhwc_bf16": (_i, [_vp, _vp, _i, _i, _i, _i, _vp]),
    "bagel_softmax_rows_f32": (_i, [_vp, _ll, _vp, _ll, _i, _i, _f, _vp]),
    "bagel_transpose_bf16": (_i, [_vp, _ll, _vp, _ll, _i, _i, _vp]),
    "bagel_taylor_update_bf16": (_i, [_vp, _ll, _vp, _ll, _i, _i, _i, _i, _vp]),
    "bagel_taylor_eval_bf16": (_i, [_vp, _ll, _i, _i, _vp, _ll, _i, _i, _vp]),
    "bagel_rmsnorm_f32": (_i, [_vp, _ll, _vp, _vp, _vp, _vp, _ll, _i, _i, _i, _f, _vp]),
    "bagel_latent_embed_add_f32": (_i, [_vp, _ll, _vp, _vp, _ll, _vp, _vp, _ll, _vp, _i, _i, _vp]),
    "bagel_image_resize_bicubic_u8": (_i, [_vp, _i, _i, _vp, _i, _i, _vp, _vp, _vp, _i, _vp, _vp, _i, _vp]),
    "bagel_image_normalize_u8": (_i, [_vp, _i, _i, _f, _f, _f, _f, _f, _f, _vp, _ll, _i, _vp]),
    "bagel_siglip_rope2d_bf16": (_i, [_vp, _ll, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp]),
}


def declared_symbols() -> list[str]:
    """Function names declared in include/bagel_b200.h."""
    text = HEADER_PATH.read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(bagel_[a-z0-9_]+)\s*\(", text)))


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not LIB_PATH.exists():
            raise BagelB200Error(
                f"{LIB_PATH} not found. Build it with `python -m bagel_b200.build` (needs nvcc, sm_90a). "
                "bagel_b200 has no CPU or PyTorch fallback.")
        l = C.CDLL(str(LIB_PATH))
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(l, name)
            fn.restype = res
            fn.argtypes = args
        _lib = l
    return _lib


def check(rc: int, what: str) -> None:
    if rc != 0:
        msg = lib().bagel_last_error()
        raise BagelB200Error(f"{what} failed (rc={rc}): {msg.decode() if msg else ''}")


def launch_count() -> int:
    return int(lib().bagel_launch_count())
