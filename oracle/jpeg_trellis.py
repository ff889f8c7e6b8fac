"""ctypes binding of the JPEG trellis quantiser's twin in oracle/jpeg_trellis_oracle.c (built into oracle/liboracle.so with the rest
of the oracle), and the lossy JPEG flows with it in place of plain quantisation -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

The flows are composed from the oracle's own stages exactly as orc_jpeg_lossy and orc_jpeg_lossy_resized compose them (decode to
native planes, [YCbCr -> RGB -> Lanczos3 -> YCbCr,] forward, write with the source's markers); with trellis=False they give those
functions' bytes, which tests/test_jpeg_trellis_host.py checks."""
import ctypes as C

import numpy as np

from . import oracle as O


def quantize_trellis(dct, q, chroma=False):
    """int32 FDCT output [8, 8] (natural order, scaled by 8) -> int16 levels [8, 8]."""
    dct = np.ascontiguousarray(dct, dtype=np.int32).reshape(64)
    q = np.ascontiguousarray(q, dtype=np.uint16).reshape(64)
    out = np.zeros(64, dtype=np.int16)
    O.lib().orc_quantize_trellis(dct.ctypes.data_as(C.c_void_p), q.ctypes.data_as(C.c_void_p), int(bool(chroma)), out.ctypes.data_as(C.c_void_p))
    return out.reshape(8, 8)


def forward(planes, p, trellis=True):
    """planes [ncomp, H, W] uint8 -> Jpeg of quantised coefficients (orc_jpeg_forward_trellis, or orc_jpeg_forward)."""
    if not trellis:
        return O.forward(planes, p)
    planes = np.ascontiguousarray(planes, dtype=np.uint8)
    n, h, w = planes.shape
    ptrs = (C.c_void_p * 4)(*[planes[c].ctypes.data if c < n else None for c in range(4)])
    j = O.Jpeg()
    err = C.create_string_buffer(256)
    f = O.lib().orc_jpeg_forward_trellis
    f.restype = C.c_int
    if f(ptrs, w, h, n, C.byref(p), C.byref(j.s), err):
        raise O.OracleError(err.value.decode())
    j._owned = True
    return j


def jpeg_lossy(data, p, trellis=True):
    """libcaesium jpeg::lossy restated (as orc_jpeg_lossy) with trellis quantisation."""
    src = O.Jpeg(data)
    return O.write(forward(src.decode_native(), p, trellis), p, meta=src)


def jpeg_lossy_resized(data, p, width, height, trellis=True):
    """the resize flow restated (as orc_jpeg_lossy_resized) with trellis quantisation."""
    src = O.Jpeg(data)
    native = src.decode_native()
    nw, nh = O.compute_dimensions(src.s.width, src.s.height, width, height)
    if src.ncomp == 3:
        rgb = O.ycc_to_rgb(native)
        ycc = O.rgb_to_ycc(np.stack([O.resize_plane(rgb[c], nw, nh) for c in range(3)]))
    else:
        ycc = O.resize_plane(native[0], nw, nh)[None]
    return O.write(forward(ycc, p, trellis), p, meta=src)
