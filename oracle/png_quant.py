"""ctypes binding of the lossy PNG quantiser twin in oracle/png_quant_oracle.c (built into oracle/liboracle.so with the rest of the
oracle) -- TEST INFRASTRUCTURE, NOT PRODUCT CODE."""
import ctypes as C

import numpy as np

from .oracle import OracleError, lib


def png_quantize(rgba, quality):
    """rgba: uint8 [h, w, 4] -> (palette uint8 [n, 4] as R, G, B, A; indices uint8 [h, w]).  An image with at most 256 distinct
    values comes back exactly (its distinct values, not opaque first, each group in increasing R | G << 8 | B << 16 | A << 24)."""
    rgba = np.ascontiguousarray(rgba, dtype=np.uint8)
    h, w = rgba.shape[:2]
    pal = np.zeros(256, np.uint32)
    idx = np.zeros((h, w), np.uint8)
    f = lib().orc_png_quantize
    f.restype = C.c_int
    n = f(rgba.ctypes.data_as(C.c_void_p), w, h, int(quality), pal.ctypes.data_as(C.c_void_p), idx.ctypes.data_as(C.c_void_p))
    if n <= 0:
        raise OracleError("png quantize failed")
    return pal[:n].view(np.uint8).reshape(n, 4).copy(), idx
