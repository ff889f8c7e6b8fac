"""ctypes binding of the lossless WebP (VP8L) encoder twin in oracle/vp8l_oracle.c (built into oracle/liboracle.so with the rest of
the oracle) -- TEST INFRASTRUCTURE, NOT PRODUCT CODE."""
import ctypes as C

import numpy as np

from .oracle import OracleError, lib

NCACHE = 4          # cache-size candidates: 0, 6, 8, 10 bits


def webp_lossless_stages(rgba, force_mode=-1, force_cache=-1):
    """Scalar lossless WebP (VP8L) encoder.  rgba: uint8 [h, w, 4] (or [h, w, 3], opaque).
    force_mode / force_cache (test hooks): every tile's predictor mode, the cache candidate (0..3 -> 0, 6, 8, 10 bits).
    Returns a dict: file (bytes), modes (uint8 [tiles_y, tiles_x]), hits (uint8 [3, h * w]: cache hit per pixel for 6, 8, 10 bits),
    tokens (uint32 [ntok, 2]: position, copy = (length << 8) | distance code or 0 for a literal), cache_bits."""
    rgba = np.asarray(rgba, dtype=np.uint8)
    if rgba.shape[2] == 3:
        rgba = np.concatenate([rgba, np.full(rgba.shape[:2] + (1,), 255, np.uint8)], axis=2)
    rgba = np.ascontiguousarray(rgba)
    h, w = rgba.shape[:2]
    n = w * h
    tx, ty = (w + 15) // 16, (h + 15) // 16
    cap = 4096 + 8 * n + 4 * tx * ty
    out = np.zeros(cap, np.uint8)
    modes = np.zeros((ty, tx), np.uint8)
    hits = np.zeros((NCACHE - 1, n), np.uint8)
    tok = np.zeros((n, 2), np.uint32)
    ntok, bits = C.c_size_t(), C.c_int()
    f = lib().orc_vp8l_encode
    f.restype = C.c_longlong
    size = f(rgba.ctypes.data_as(C.c_void_p), w, h, int(force_mode), int(force_cache), out.ctypes.data_as(C.c_void_p), C.c_size_t(cap),
             modes.ctypes.data_as(C.c_void_p), hits.ctypes.data_as(C.c_void_p), tok.ctypes.data_as(C.c_void_p), C.byref(ntok), C.byref(bits))
    if size < 0:
        raise OracleError("vp8l encode failed")
    return {"file": out[:size].tobytes(), "modes": modes, "hits": hits, "tokens": tok[:ntok.value].copy(), "cache_bits": bits.value}


def webp_lossless_encode(rgba, force_mode=-1, force_cache=-1):
    """rgba: uint8 [h, w, 4] or [h, w, 3] -> the lossless .webp file the device encoder writes for it."""
    return webp_lossless_stages(rgba, force_mode, force_cache)["file"]
