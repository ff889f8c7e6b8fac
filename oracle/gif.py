"""ctypes binding of the GIF re-encoder twin in oracle/gif_oracle.c (built into oracle/liboracle.so with the rest of the oracle)
-- TEST INFRASTRUCTURE, NOT PRODUCT CODE."""
import ctypes as C

import numpy as np

from .oracle import OracleError, lib


def gif_encode(canvases, delays, loop, quality):
    """canvases: uint8 [n, h, w, 4] composited frames (R, G, B, A; alpha 0 or 255, clear pixels all zero); delays in 1/100 s;
    loop: NETSCAPE2.0 count or -1 -> the whole re-encoded file."""
    cv = np.ascontiguousarray(canvases, dtype=np.uint8)
    n, h, w = cv.shape[:3]
    d = np.ascontiguousarray(delays, dtype=np.int32)
    cap = 1024 + n * (800 + 2 * w * h)
    out = np.zeros(cap, np.uint8)
    f = lib().orc_gif_encode
    f.restype = C.c_longlong
    size = f(cv.ctypes.data_as(C.c_void_p), d.ctypes.data_as(C.c_void_p), int(n), int(w), int(h), int(loop), int(quality),
             out.ctypes.data_as(C.c_void_p), C.c_size_t(cap))
    if size < 0:
        raise OracleError("gif encode failed")
    return out[:size].tobytes()


def gif_lzw(indices, min_code_size):
    """indices: uint8 [n], each below 2^min_code_size -> GIF image data as sub-blocks with the terminator."""
    idx = np.ascontiguousarray(indices, dtype=np.uint8).reshape(-1)
    cap = 64 + 2 * idx.size
    out = np.zeros(cap, np.uint8)
    f = lib().orc_gif_lzw
    f.restype = C.c_longlong
    size = f(idx.ctypes.data_as(C.c_void_p), C.c_size_t(idx.size), int(min_code_size), out.ctypes.data_as(C.c_void_p), C.c_size_t(cap))
    if size < 0:
        raise OracleError("gif lzw failed")
    return out[:size].tobytes()


def gif_quantize(rgba, quality):
    """the palette quantiser without its exact path: rgba uint8 [h, w, 4] -> (palette uint8 [n, 4], indices uint8 [h, w])"""
    rgba = np.ascontiguousarray(rgba, dtype=np.uint8)
    h, w = rgba.shape[:2]
    pal = np.zeros(256, np.uint32)
    idx = np.zeros((h, w), np.uint8)
    f = lib().orc_gif_quantize
    f.restype = C.c_int
    n = f(rgba.ctypes.data_as(C.c_void_p), w, h, int(quality), pal.ctypes.data_as(C.c_void_p), idx.ctypes.data_as(C.c_void_p))
    if n <= 0:
        raise OracleError("gif quantize failed")
    return pal[:n].view(np.uint8).reshape(n, 4).copy(), idx
