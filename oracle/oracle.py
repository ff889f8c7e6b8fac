"""ctypes binding of oracle/liboracle.so -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
legs may import this module (see oracle/jpeg_oracle.h for what the oracle restates:
the codec work below caesium-clt's src/compressor.rs:287-306).
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = os.path.join(_HERE, "liboracle.so")


def build(force=False):
    srcs = [os.path.join(_HERE, f) for f in os.listdir(_HERE) if f.endswith((".c", ".h"))]
    if force or not os.path.exists(_LIB) or any(os.path.getmtime(s) > os.path.getmtime(_LIB) for s in srcs):
        subprocess.check_call(["make", "-C", _HERE, "-s"])
    return _LIB


class OrcJpeg(C.Structure):
    _fields_ = [
        ("width", C.c_int), ("height", C.c_int), ("ncomp", C.c_int), ("progressive", C.c_int),
        ("hs", C.c_int * 4), ("vs", C.c_int * 4), ("tq", C.c_int * 4), ("cid", C.c_int * 4),
        ("hmax", C.c_int), ("vmax", C.c_int), ("mcux", C.c_int), ("mcuy", C.c_int),
        ("bw", C.c_int * 4), ("bh", C.c_int * 4), ("rbw", C.c_int * 4), ("rbh", C.c_int * 4),
        ("cw", C.c_int * 4), ("ch", C.c_int * 4),
        ("qt", (C.c_uint16 * 64) * 4), ("qt_present", C.c_int * 4),
        ("coef", C.POINTER(C.c_int16) * 4),
        ("restart_interval", C.c_int), ("nscans", C.c_int),
        ("scan_script", (C.c_int * 8) * 64),
        ("jfif", C.c_int), ("adobe", C.c_int), ("adobe_transform", C.c_int),
        ("markers", C.POINTER(C.c_uint8)), ("markers_len", C.c_size_t),
        ("icc_markers", C.POINTER(C.c_uint8)), ("icc_len", C.c_size_t),
    ]


class OrcJpegParams(C.Structure):
    _fields_ = [("quality", C.c_int), ("subsampling", C.c_int), ("progressive", C.c_int),
                ("keep_metadata", C.c_int), ("preserve_icc", C.c_int)]


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(_LIB)
        _lib.orc_jpeg_read.restype = C.c_int
        _lib.orc_jpeg_lossy.restype = C.c_int
        _lib.orc_jpeg_lossless.restype = C.c_int
        _lib.orc_jpeg_write.restype = C.c_int
        _lib.orc_jpeg_forward.restype = C.c_int
        _lib.orc_jpeg_decode_native.restype = C.c_int
    return _lib


class OracleError(RuntimeError):
    pass


def _buf(data):
    return (C.c_uint8 * len(data)).from_buffer_copy(data)


def quant_table(quality, which=0):
    out = (C.c_uint16 * 64)()
    lib().orc_quant_table(int(quality), int(which), out)
    return np.frombuffer(out, dtype=np.uint16).copy()


def idct_islow(coef, q):
    coef = np.ascontiguousarray(coef, dtype=np.int16).reshape(64)
    q = np.ascontiguousarray(q, dtype=np.uint16).reshape(64)
    out = np.zeros(64, dtype=np.uint8)
    lib().orc_idct_islow(coef.ctypes.data_as(C.c_void_p), q.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p))
    return out.reshape(8, 8)


def fdct_quant(px, q):
    px = np.ascontiguousarray(px, dtype=np.uint8).reshape(64)
    q = np.ascontiguousarray(q, dtype=np.uint16).reshape(64)
    dct = np.zeros(64, dtype=np.int32)
    out = np.zeros(64, dtype=np.int16)
    lib().orc_fdct_islow(px.ctypes.data_as(C.c_void_p), dct.ctypes.data_as(C.c_void_p))
    lib().orc_quantize(dct.ctypes.data_as(C.c_void_p), q.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p))
    return dct.reshape(8, 8), out.reshape(8, 8)


class Jpeg:
    """Decoded coefficient-domain view of a JPEG file (orc_jpeg_read)."""

    def __init__(self, data=None):
        self.s = OrcJpeg()
        self._owned = False
        if data is not None:
            err = C.create_string_buffer(256)
            if lib().orc_jpeg_read(_buf(data), C.c_size_t(len(data)), C.byref(self.s), err):
                raise OracleError(err.value.decode())
            self._owned = True

    def __del__(self):
        if self._owned:
            lib().orc_jpeg_free(C.byref(self.s))
            self._owned = False

    @property
    def ncomp(self):
        return self.s.ncomp

    def coef(self, c):
        """[bh, bw, 64] int16, natural order, quantised (padded to whole MCUs)."""
        n = self.s.bh[c] * self.s.bw[c] * 64
        a = np.ctypeslib.as_array(self.s.coef[c], shape=(n,)).copy()
        return a.reshape(self.s.bh[c], self.s.bw[c], 64)

    def qtable(self, c):
        return np.frombuffer(self.s.qt[self.s.tq[c]], dtype=np.uint16).copy()

    def scans(self):
        return [tuple(self.s.scan_script[i]) for i in range(self.s.nscans)]

    def component_plane(self, c):
        """dequant + IDCT of every allocated block: (bh*8, bw*8) uint8."""
        out = np.zeros((self.s.bh[c] * 8, self.s.bw[c] * 8), dtype=np.uint8)
        lib().orc_jpeg_idct_component(C.byref(self.s), c, out.ctypes.data_as(C.c_void_p))
        return out

    def decode_native(self):
        """[ncomp, H, W] uint8 in the file's own colour space (fancy upsampling)."""
        out = np.zeros((self.s.ncomp, self.s.height, self.s.width), dtype=np.uint8)
        ptrs = (C.c_void_p * 4)(*[out[c].ctypes.data if c < self.s.ncomp else None for c in range(4)])
        err = C.create_string_buffer(256)
        if lib().orc_jpeg_decode_native(C.byref(self.s), ptrs, err):
            raise OracleError(err.value.decode())
        return out


def params(quality=80, subsampling=0, progressive=True, keep_metadata=False, preserve_icc=True):
    return OrcJpegParams(int(quality), int(subsampling), int(bool(progressive)), int(bool(keep_metadata)), int(bool(preserve_icc)))


def forward(planes, p):
    """planes [ncomp,H,W] uint8 -> Jpeg holding quantised coefficients (orc_jpeg_forward)."""
    planes = np.ascontiguousarray(planes, dtype=np.uint8)
    n, h, w = planes.shape
    ptrs = (C.c_void_p * 4)(*[planes[c].ctypes.data if c < n else None for c in range(4)])
    j = Jpeg()
    err = C.create_string_buffer(256)
    if lib().orc_jpeg_forward(ptrs, w, h, n, C.byref(p), C.byref(j.s), err):
        raise OracleError(err.value.decode())
    j._owned = True
    return j


def _take(outp, outl):
    data = C.string_at(outp, outl.value)
    lib().orc_free(outp)
    return data


def write(j, p, meta=None):
    outp, outl = C.POINTER(C.c_uint8)(), C.c_size_t()
    err = C.create_string_buffer(256)
    if lib().orc_jpeg_write(C.byref(j.s), C.byref(p), C.byref(meta.s) if meta is not None else None, C.byref(outp), C.byref(outl), err):
        raise OracleError(err.value.decode())
    return _take(outp, outl)


def jpeg_lossy(data, p):
    """libcaesium jpeg::lossy restated (compress_in_memory, jpeg.optimize == false)."""
    outp, outl = C.POINTER(C.c_uint8)(), C.c_size_t()
    err = C.create_string_buffer(256)
    if lib().orc_jpeg_lossy(_buf(data), C.c_size_t(len(data)), C.byref(p), C.byref(outp), C.byref(outl), err):
        raise OracleError(err.value.decode())
    return _take(outp, outl)


def jpeg_lossy_resized(data, p, width, height):
    """libcaesium JPEG compress with CSParameters.width/height (decode -> RGB -> Lanczos3 -> YCbCr -> encode)."""
    outp, outl = C.POINTER(C.c_uint8)(), C.c_size_t()
    err = C.create_string_buffer(256)
    lib().orc_jpeg_lossy_resized.restype = C.c_int
    if lib().orc_jpeg_lossy_resized(_buf(data), C.c_size_t(len(data)), C.byref(p), C.c_uint32(width), C.c_uint32(height), C.byref(outp), C.byref(outl), err):
        raise OracleError(err.value.decode())
    return _take(outp, outl)


def compute_dimensions(ow, oh, dw, dh):
    nw, nh = C.c_uint32(), C.c_uint32()
    lib().orc_compute_dimensions(C.c_uint32(ow), C.c_uint32(oh), C.c_uint32(dw), C.c_uint32(dh), C.byref(nw), C.byref(nh))
    return nw.value, nh.value


def resize_plane(plane, nw, nh):
    """One u8 channel through image-crate-style Lanczos3 (vertical pass to f32, then horizontal)."""
    plane = np.ascontiguousarray(plane, dtype=np.uint8)
    h, w = plane.shape
    out = np.zeros((nh, nw), dtype=np.uint8)
    lib().orc_resize_plane_lanczos3.restype = C.c_int
    if lib().orc_resize_plane_lanczos3(plane.ctypes.data_as(C.c_void_p), w, h, w, out.ctypes.data_as(C.c_void_p), nw, nh, nw):
        raise OracleError("resize failed")
    return out


def ycc_to_rgb(ycc):
    ycc = np.ascontiguousarray(ycc, dtype=np.uint8)
    out = np.zeros_like(ycc)
    n = ycc[0].size
    lib().orc_ycc_to_rgb(ycc[0].ctypes.data_as(C.c_void_p), ycc[1].ctypes.data_as(C.c_void_p), ycc[2].ctypes.data_as(C.c_void_p),
                         out[0].ctypes.data_as(C.c_void_p), out[1].ctypes.data_as(C.c_void_p), out[2].ctypes.data_as(C.c_void_p), C.c_size_t(n))
    return out


def rgb_to_ycc(rgb):
    rgb = np.ascontiguousarray(rgb, dtype=np.uint8)
    out = np.zeros_like(rgb)
    n = rgb[0].size
    lib().orc_rgb_to_ycc(rgb[0].ctypes.data_as(C.c_void_p), rgb[1].ctypes.data_as(C.c_void_p), rgb[2].ctypes.data_as(C.c_void_p),
                         out[0].ctypes.data_as(C.c_void_p), out[1].ctypes.data_as(C.c_void_p), out[2].ctypes.data_as(C.c_void_p), C.c_size_t(n))
    return out


def jpeg_lossless(data, p):
    """libcaesium jpeg::lossless restated (jpegtran-style transcode)."""
    outp, outl = C.POINTER(C.c_uint8)(), C.c_size_t()
    err = C.create_string_buffer(256)
    if lib().orc_jpeg_lossless(_buf(data), C.c_size_t(len(data)), C.byref(p), C.byref(outp), C.byref(outl), err):
        raise OracleError(err.value.decode())
    return _take(outp, outl)


# ---- PNG lossless leg (oracle/png_oracle.c) -------------------------------------------------------------------
PNG_STRATEGIES = {"none": 0, "sub": 1, "up": 2, "average": 3, "paeth": 4, "minsum": 5, "entropy": 6, "bigrams": 7, "bigent": 8, "brute": 9}


def png_filter(raw, bpp, strategy):
    """raw: uint8 [h, row_bytes] -> filtered uint8 [h, row_bytes + 1] (filter byte first)."""
    raw = np.ascontiguousarray(raw, dtype=np.uint8)
    h, rb = raw.shape
    out = np.zeros((h, rb + 1), dtype=np.uint8)
    lib().orc_png_filter(raw.ctypes.data_as(C.c_void_p), h, rb, bpp, int(strategy), out.ctypes.data_as(C.c_void_p))
    return out


def png_unfilter(filt, bpp):
    filt = np.ascontiguousarray(filt, dtype=np.uint8)
    h, rb1 = filt.shape
    out = np.zeros((h, rb1 - 1), dtype=np.uint8)
    if lib().orc_png_unfilter(filt.ctypes.data_as(C.c_void_p), h, rb1 - 1, bpp, out.ctypes.data_as(C.c_void_p)):
        raise OracleError("bad filter type")
    return out


def png_lz77(stream, bpp, stride):
    """Filtered byte stream -> (tokens uint32[nt], hist uint32[316])."""
    s = np.ascontiguousarray(stream, dtype=np.uint8).reshape(-1)
    tok = np.zeros(s.size, dtype=np.uint32)
    hist = np.zeros(316, dtype=np.uint32)
    lib().orc_png_lz77.restype = C.c_size_t
    nt = lib().orc_png_lz77(s.ctypes.data_as(C.c_void_p), C.c_size_t(s.size), bpp, stride, tok.ctypes.data_as(C.c_void_p), hist.ctypes.data_as(C.c_void_p))
    return tok[:nt].copy(), hist


# ---- WebP (lossy VP8) leg (oracle/webp_oracle.c) ----------------------------------------------------------------
def vp8_qindex(quality):
    return lib().orc_vp8_qindex(int(quality))


def webp_rgb_to_yuv(rgb):
    """rgb: uint8 [3, h, w] planar -> (Y [mbh*16, mbw*16], U, V [mbh*8, mbw*8]) macroblock-padded."""
    rgb = np.ascontiguousarray(rgb, dtype=np.uint8)
    _, h, w = rgb.shape
    mbw, mbh = (w + 15) // 16, (h + 15) // 16
    Y = np.zeros((mbh * 16, mbw * 16), np.uint8); U = np.zeros((mbh * 8, mbw * 8), np.uint8); V = np.zeros_like(U)
    lib().orc_webp_rgb_to_yuv(rgb[0].ctypes.data_as(C.c_void_p), rgb[1].ctypes.data_as(C.c_void_p), rgb[2].ctypes.data_as(C.c_void_p), w, h,
                              Y.ctypes.data_as(C.c_void_p), U.ctypes.data_as(C.c_void_p), V.ctypes.data_as(C.c_void_p))
    return Y, U, V


def webp_analyze(rgb, quality):
    """Stage view: (levels int16 [nmb, 25, 16] zigzag, modes uint8 [nmb, 4] = ymode, uvmode, skip, 0)."""
    rgb = np.ascontiguousarray(rgb, dtype=np.uint8)
    _, h, w = rgb.shape
    nmb = ((w + 15) // 16) * ((h + 15) // 16)
    levels = np.zeros((nmb, 25, 16), np.int16); modes = np.zeros((nmb, 4), np.uint8)
    rc = lib().orc_webp_analyze(rgb[0].ctypes.data_as(C.c_void_p), rgb[1].ctypes.data_as(C.c_void_p), rgb[2].ctypes.data_as(C.c_void_p), w, h, int(quality),
                                levels.ctypes.data_as(C.c_void_p), modes.ctypes.data_as(C.c_void_p))
    if rc:
        raise OracleError("webp analyze failed (%d)" % rc)
    return levels, modes


def vp8_quant_factors(qindex):
    f = (C.c_int * 6)()
    lib().orc_vp8_quant_factors(int(qindex), f)
    return list(f)


def webp_encode(rgb, quality):
    """rgb: uint8 [3, h, w] planar -> (file bytes, (Y, U, V) reconstruction at macroblock-padded size)."""
    rgb = np.ascontiguousarray(rgb, dtype=np.uint8)
    _, h, w = rgb.shape
    mbw, mbh = (w + 15) // 16, (h + 15) // 16
    Y = np.zeros((mbh * 16, mbw * 16), np.uint8); U = np.zeros((mbh * 8, mbw * 8), np.uint8); V = np.zeros_like(U)
    outp, outl = C.POINTER(C.c_uint8)(), C.c_size_t()
    rc = lib().orc_webp_encode(rgb[0].ctypes.data_as(C.c_void_p), rgb[1].ctypes.data_as(C.c_void_p), rgb[2].ctypes.data_as(C.c_void_p), w, h, int(quality),
                               C.byref(outp), C.byref(outl), Y.ctypes.data_as(C.c_void_p), U.ctypes.data_as(C.c_void_p), V.ctypes.data_as(C.c_void_p))
    if rc:
        raise OracleError("webp encode failed (%d)" % rc)
    return _take(outp, outl), (Y, U, V)


def png_expand(tokens, n):
    tokens = np.ascontiguousarray(tokens, dtype=np.uint32)
    out = np.zeros(n, dtype=np.uint8)
    lib().orc_png_expand.restype = C.c_size_t
    got = lib().orc_png_expand(tokens.ctypes.data_as(C.c_void_p), C.c_size_t(tokens.size), out.ctypes.data_as(C.c_void_p), C.c_size_t(n))
    if got != n:
        raise OracleError("token stream does not expand to %d bytes" % n)
    return out
