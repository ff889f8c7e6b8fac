"""ctypes binding of the animated WebP twin in oracle/webp_anim_oracle.c (built into oracle/liboracle.so with the rest of the
oracle) -- TEST INFRASTRUCTURE, NOT PRODUCT CODE."""
import ctypes as C

import numpy as np

from .oracle import OracleError, lib


def compose(width, height, frames):
    """frames: [(x, y, flags, has_alpha, rgba uint8 [h, w, 4])] decoded frame rectangles -> canvases uint8 [n, H, W, 4]."""
    n = len(frames)
    rects = np.array([[f[0], f[1], f[4].shape[1], f[4].shape[0]] for f in frames], np.int32).reshape(-1)
    flags = np.array([f[2] for f in frames], np.int32)
    alpha = np.array([int(bool(f[3])) for f in frames], np.int32)
    px = np.concatenate([np.ascontiguousarray(f[4], np.uint8).reshape(-1) for f in frames]) if n else np.zeros(4, np.uint8)
    out = np.zeros((n, height, width, 4), np.uint8)
    f = lib().orc_webp_anim_compose
    f.restype = C.c_int
    if f(int(width), int(height), n, rects.ctypes.data_as(C.c_void_p), flags.ctypes.data_as(C.c_void_p), alpha.ctypes.data_as(C.c_void_p),
         px.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p)) != 0:
        raise OracleError("webp anim compose failed")
    return out


def frames(canvases, durations):
    """canvases uint8 [n, H, W, 4], durations in ms -> [(kept canvas index, (x, y, w, h), duration)], the output frames."""
    cv = np.ascontiguousarray(canvases, np.uint8)
    n, h, w = cv.shape[:3]
    du = np.ascontiguousarray(durations, np.uint32)
    kept = np.zeros(max(n, 1), np.int32)
    rects = np.zeros(4 * max(n, 1), np.int32)
    dur = np.zeros(max(n, 1), np.uint32)
    f = lib().orc_webp_anim_frames
    f.restype = C.c_int
    m = f(int(w), int(h), int(n), cv.ctypes.data_as(C.c_void_p), du.ctypes.data_as(C.c_void_p), kept.ctypes.data_as(C.c_void_p),
          rects.ctypes.data_as(C.c_void_p), dur.ctypes.data_as(C.c_void_p))
    return [(int(kept[j]), tuple(int(v) for v in rects[4 * j:4 * j + 4]), int(dur[j])) for j in range(m)]
