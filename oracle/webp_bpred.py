"""ctypes binding of the lossy WebP B_PRED twin in oracle/webp_bpred_oracle.c (built into oracle/liboracle.so with the rest of the
oracle) -- TEST INFRASTRUCTURE, NOT PRODUCT CODE."""
import ctypes as C

import numpy as np

from .oracle import OracleError, _take, lib


def webp_bpred_stages(rgb, quality, allow_overflow=False):
    """rgb: uint8 [3, h, w] planar -> dict: file (bytes), levels int16 [nmb, 25, 16], modes uint8 [nmb, 4] (ymode 4 = B_PRED),
    bmodes uint8 [nmb, 16], the reconstruction a decoder shows, Y (after the loop filter), U, V at macroblock-padded size, and the
    encoder's own luma before the loop filter (Yraw).
    A first partition past 19 bits raises unless allow_overflow (then "overflow" is True and the file is not a valid VP8 file)."""
    rgb = np.ascontiguousarray(rgb, dtype=np.uint8)
    _, h, w = rgb.shape
    mbw, mbh = (w + 15) // 16, (h + 15) // 16
    nmb = mbw * mbh
    levels = np.zeros((nmb, 25, 16), np.int16); modes = np.zeros((nmb, 4), np.uint8); bmodes = np.zeros((nmb, 16), np.uint8)
    Y = np.zeros((mbh * 16, mbw * 16), np.uint8); U = np.zeros((mbh * 8, mbw * 8), np.uint8); V = np.zeros_like(U); Yraw = np.zeros_like(Y)
    outp, outl = C.POINTER(C.c_uint8)(), C.c_size_t()
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    rc = lib().orc_webp_bpred_encode(p(rgb[0]), p(rgb[1]), p(rgb[2]), w, h, int(quality), C.byref(outp), C.byref(outl),
                                     p(levels), p(modes), p(bmodes), p(Y), p(U), p(V), p(Yraw))
    if rc == -1 or (rc == -2 and not allow_overflow):
        if rc == -2:
            _take(outp, outl)
        raise OracleError("webp bpred encode failed (%d)" % rc)
    return {"file": _take(outp, outl), "levels": levels, "modes": modes, "bmodes": bmodes, "Y": Y, "U": U, "V": V, "Yraw": Yraw, "overflow": rc == -2}


def webp_bpred_encode(rgb, quality):
    """rgb: uint8 [3, h, w] planar -> the .webp file the device encoder writes with the B_PRED switch on."""
    return webp_bpred_stages(rgb, quality)["file"]
