"""ctypes binding of the lossless WebP (VP8L) palette-variant twin in oracle/vp8l_palette_oracle.c (built into oracle/liboracle.so
with the rest of the oracle) -- TEST INFRASTRUCTURE, NOT PRODUCT CODE."""
import ctypes as C

import numpy as np

from .oracle import OracleError, lib


def webp_palette_stages(rgba):
    """The lossless WebP file the encoder keeps with the palette switch on.  rgba: uint8 [h, w, 4] (or [h, w, 3], opaque).
    Returns a dict: file (bytes), sizes (file sizes without / with the palette; 0 for the latter over 256 colours),
    palette (uint32 ARGB, ascending; None over 256 colours), packed (uint32 [h, w'] packed index image; None over 256 colours),
    palette_file (bytes: the palette variant's file, kept or not; None over 256 colours)."""
    rgba = np.asarray(rgba, dtype=np.uint8)
    if rgba.shape[2] == 3:
        rgba = np.concatenate([rgba, np.full(rgba.shape[:2] + (1,), 255, np.uint8)], axis=2)
    rgba = np.ascontiguousarray(rgba)
    h, w = rgba.shape[:2]
    n = w * h
    cap = 4096 + 8 * n + 4 * ((w + 15) // 16) * ((h + 15) // 16)
    out, alt = np.zeros(cap, np.uint8), np.zeros(cap, np.uint8)
    sizes = (C.c_longlong * 2)()
    pal = np.zeros(256, np.uint32)
    packed = np.zeros(n, np.uint32)
    count, pw = C.c_int(), C.c_int()
    f = lib().orc_vp8l_encode_palette
    f.restype = C.c_longlong
    size = f(rgba.ctypes.data_as(C.c_void_p), w, h, out.ctypes.data_as(C.c_void_p), C.c_size_t(cap), sizes, pal.ctypes.data_as(C.c_void_p),
             C.byref(count), packed.ctypes.data_as(C.c_void_p), C.byref(pw), alt.ctypes.data_as(C.c_void_p))
    if size < 0:
        raise OracleError("vp8l palette encode failed")
    k = count.value
    return {"file": out[:size].tobytes(), "sizes": (sizes[0], sizes[1]), "palette": pal[:k].copy() if k > 0 else None,
            "packed": packed[:pw.value * h].reshape(h, pw.value).copy() if k > 0 else None,
            "palette_file": alt[:sizes[1]].tobytes() if k > 0 else None}


def webp_palette_encode(rgba):
    """rgba: uint8 [h, w, 4] or [h, w, 3] -> the lossless .webp file the device encoder writes for it with the palette switch on."""
    return webp_palette_stages(rgba)["file"]
