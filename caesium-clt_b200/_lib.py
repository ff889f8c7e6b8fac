"""ctypes binding of libb200caesium.so (include/b200_caesium.h).

This is the only way Python code in this repo reaches the product: through the same C-ABI a
Rust maintainer would bind at caesium-clt's src/compressor.rs:287-306.  There is no Python or
CPU fallback -- if the shared library is missing, loading raises; if no H100 is visible, every
codec call returns B200_ERR_NO_DEVICE.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libb200caesium.so")

OK, ERR_INVALID_ARGUMENT, ERR_UNKNOWN_FORMAT, ERR_UNSUPPORTED, ERR_CORRUPT_INPUT = 0, 1, 2, 3, 4
ERR_NO_DEVICE, ERR_CUDA, ERR_OUT_OF_MEMORY, ERR_SAME_FORMAT, ERR_TOO_LARGE = 5, 6, 7, 8, 9
FMT_JPEG, FMT_PNG, FMT_GIF, FMT_WEBP, FMT_TIFF, FMT_UNKNOWN = 0, 1, 2, 3, 4, 5


class Status(C.Structure):
    _fields_ = [("code", C.c_int32), ("message", C.c_void_p)]


class Params(C.Structure):
    """b200_params == caesium::parameters::CSParameters as compressor.rs:411-446 fills it."""
    _fields_ = [
        ("keep_metadata", C.c_uint8), ("jpeg_quality", C.c_uint32), ("jpeg_chroma_subsampling", C.c_uint32),
        ("jpeg_progressive", C.c_uint8), ("jpeg_optimize", C.c_uint8), ("jpeg_preserve_icc", C.c_uint8),
        ("png_quality", C.c_uint32), ("png_optimization_level", C.c_uint32), ("png_force_zopfli", C.c_uint8),
        ("png_optimize", C.c_uint8), ("gif_quality", C.c_uint32), ("webp_quality", C.c_uint32),
        ("webp_lossless", C.c_uint8), ("width", C.c_uint32), ("height", C.c_uint32),
    ]


class JpegLayout(C.Structure):
    _fields_ = [
        ("width", C.c_int32), ("height", C.c_int32), ("ncomp", C.c_int32), ("progressive", C.c_int32),
        ("hs", C.c_int32 * 4), ("vs", C.c_int32 * 4), ("bw", C.c_int32 * 4), ("bh", C.c_int32 * 4),
        ("rbw", C.c_int32 * 4), ("rbh", C.c_int32 * 4), ("comp_offset", C.c_int64 * 4), ("total_coefs", C.c_int64),
        ("qt", (C.c_uint16 * 64) * 4),
    ]


class B200Error(RuntimeError):
    def __init__(self, code, message):
        super().__init__(message)
        self.code = code


def build(force=False):
    """Compile the CUDA + C++ sources in-tree (nvcc -gencode arch=compute_90a,code=sm_90a)."""
    if force:
        subprocess.check_call(["make", "-C", _HERE, "-s", "clean"])
    subprocess.check_call(["make", "-C", _HERE, "-s", "-j8"])
    return LIB_PATH


_lib = None

_SYMBOLS = [
    "b200_params_default", "b200_set_entropy_mode", "b200_init", "b200_init_device", "b200_shutdown", "b200_device_count", "b200_version", "b200_free",
    "b200_compress_in_memory", "b200_convert_in_memory", "b200_compress_to_size_in_memory", "b200_compress_batch",
    "b200_sniff_format", "b200_jpeg_decode_coefficients", "b200_jpeg_output_layout", "b200_jpeg_requantize",
    "b200_jpeg_encode_coefficients", "b200_jpeg_decode_planes", "b200_jpeg_quant_table", "b200_jpeg_encode_coefficients_device",
    "b200_png_decode", "b200_png_decode_reduced", "b200_png_filter", "b200_png_lz77", "b200_png_deflate_tokens", "b200_png_level_strategies",
    "b200_webp_encode_rgb", "b200_webp_write_levels", "b200_webp_qindex",
    "b200_jpeg_pipe_create", "b200_jpeg_pipe_run", "b200_jpeg_pipe_finish", "b200_jpeg_pipe_fetch", "b200_jpeg_pipe_kernel_times", "b200_jpeg_pipe_destroy", "b200_device_jobs", "b200_device_numa_node", "b200_png_device_times", "b200_webp_decode", "b200_webp_alpha_chunk", "b200_webp_wrap_alpha", "b200_webp_decode_rgba", "b200_webp_alpha_filter", "b200_webp_d2h_bytes",
    "b200_set_png_lossy", "b200_png_quantize", "b200_set_jpeg_trellis", "b200_set_gif", "b200_gif_decode", "b200_gif_lzw",
    "b200_set_png_resize", "b200_png_resize_samples", "b200_set_webp_lossless_convert", "b200_set_png_interlaced",
    "b200_set_gif_convert", "b200_gif_first_frame", "b200_set_webp_anim", "b200_webp_anim_decode",
    "b200_set_png_zopfli", "b200_png_lz77_zopfli", "b200_set_webp_palette",
    "b200_set_webp_bpred", "b200_webp_encode_rgb_bpred", "b200_webp_write_levels_bpred",
]


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(f"{LIB_PATH} is missing: run __graft_entry__.build() (there is no Python/CPU fallback)")
        L = C.CDLL(LIB_PATH)
        for name in _SYMBOLS:
            getattr(L, name)  # raises AttributeError if the ABI is incomplete
        for f in ("b200_compress_in_memory", "b200_convert_in_memory", "b200_compress_to_size_in_memory",
                  "b200_jpeg_decode_coefficients", "b200_jpeg_output_layout", "b200_jpeg_requantize",
                  "b200_jpeg_encode_coefficients", "b200_jpeg_decode_planes",
                  "b200_png_decode", "b200_png_decode_reduced", "b200_png_filter", "b200_png_lz77", "b200_png_deflate_tokens",
                  "b200_webp_encode_rgb", "b200_webp_write_levels", "b200_jpeg_encode_coefficients_device",
                  "b200_jpeg_pipe_create", "b200_jpeg_pipe_run", "b200_jpeg_pipe_finish", "b200_jpeg_pipe_fetch", "b200_jpeg_pipe_kernel_times", "b200_png_device_times", "b200_webp_decode", "b200_webp_alpha_chunk", "b200_webp_wrap_alpha", "b200_webp_decode_rgba", "b200_png_quantize",
                  "b200_gif_decode", "b200_gif_lzw", "b200_png_resize_samples", "b200_gif_first_frame", "b200_webp_anim_decode",
                  "b200_png_lz77_zopfli", "b200_webp_encode_rgb_bpred", "b200_webp_write_levels_bpred"):
            getattr(L, f).restype = Status
        L.b200_webp_d2h_bytes.restype = C.c_ulonglong
        L.b200_version.restype = C.c_char_p
        L.b200_sniff_format.restype = C.c_uint32
        L.b200_free.argtypes = [C.c_void_p]
        L.b200_jpeg_pipe_destroy.argtypes = [C.c_void_p]
        L.b200_device_jobs.restype = C.c_longlong
        _lib = L
    return _lib


def _check(st):
    if st.code != 0:
        msg = C.string_at(st.message).decode() if st.message else f"error {st.code}"
        lib().b200_free(st.message)
        raise B200Error(st.code, msg)


def default_params():
    p = Params()
    lib().b200_params_default(C.byref(p))
    return p


def _take(outp, outl):
    data = C.string_at(outp, outl.value)
    lib().b200_free(outp)
    return data


def compress_in_memory(data, params):
    """caesium::compress_in_memory (compressor.rs:305)."""
    outp, outl = C.c_void_p(), C.c_size_t()
    _check(lib().b200_compress_in_memory(data, C.c_size_t(len(data)), C.byref(params), C.byref(outp), C.byref(outl)))
    return _take(outp, outl)


def convert_in_memory(data, params, fmt):
    """caesium::convert_in_memory (compressor.rs:289, :300)."""
    outp, outl = C.c_void_p(), C.c_size_t()
    _check(lib().b200_convert_in_memory(data, C.c_size_t(len(data)), C.byref(params), C.c_uint32(fmt), C.byref(outp), C.byref(outl)))
    return _take(outp, outl)


def compress_to_size_in_memory(data, params, max_size, return_smallest=True):
    """caesium::compress_to_size_in_memory (compressor.rs:295, :298); params.jpeg_quality may be updated."""
    outp, outl = C.c_void_p(), C.c_size_t()
    _check(lib().b200_compress_to_size_in_memory(data, C.c_size_t(len(data)), C.byref(params), C.c_size_t(max_size),
                                                 C.c_uint8(1 if return_smallest else 0), C.byref(outp), C.byref(outl)))
    return _take(outp, outl)


class BatchInputs:
    """Inputs of compress_batch marshalled once (pointer / length arrays), for callers that time the C-ABI call itself."""

    def __init__(self, datas):
        self.n = len(datas)
        self.datas = datas                              # keeps the bytes objects alive
        self.ins = (C.c_char_p * self.n)(*datas)
        self.lens = (C.c_size_t * self.n)(*[len(d) for d in datas])


def compress_batch(datas, params, n_threads=0, copy=True):
    """Batch form of start_compression's par_iter (compressor.rs:74-101): returns [(bytes | None, code, message)].
    copy=False: the library's malloc'ed outputs are inspected in place (length, first two bytes) and freed without being
    duplicated into Python bytes objects -- entries are (length, code, message, head)."""
    bi = datas if isinstance(datas, BatchInputs) else BatchInputs(datas)
    n = bi.n
    outs = (C.c_void_p * n)()
    outl = (C.c_size_t * n)()
    sts = (Status * n)()
    lib().b200_compress_batch(bi.ins, bi.lens, n, C.byref(params), int(n_threads), outs, outl, sts)
    res = []
    for i in range(n):
        if sts[i].code == 0 and not copy:
            res.append((outl[i], 0, "", C.string_at(outs[i], 2)))
            lib().b200_free(outs[i])
        elif sts[i].code == 0:
            res.append((C.string_at(outs[i], outl[i]), 0, ""))
            lib().b200_free(outs[i])
        else:
            msg = C.string_at(sts[i].message).decode() if sts[i].message else ""
            lib().b200_free(sts[i].message)
            res.append((None, sts[i].code, msg))
    return res


def sniff_format(data):
    return lib().b200_sniff_format(data, C.c_size_t(len(data)))


def jpeg_quant_table(quality, which=0):
    out = (C.c_uint16 * 64)()
    lib().b200_jpeg_quant_table(int(quality), int(which), out)
    return np.frombuffer(out, dtype=np.uint16).copy()


def jpeg_decode_coefficients(data):
    """Host entropy decode -> (JpegLayout, int16 array of total_coefs, zigzag order)."""
    lay = JpegLayout()
    ptr = C.c_void_p()
    _check(lib().b200_jpeg_decode_coefficients(data, C.c_size_t(len(data)), C.byref(lay), C.byref(ptr)))
    arr = np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_int16)), shape=(lay.total_coefs,)).copy()
    lib().b200_free(ptr)
    return lay, arr


def jpeg_output_layout(in_layout, params):
    out = JpegLayout()
    _check(lib().b200_jpeg_output_layout(C.byref(in_layout), C.byref(params), C.byref(out)))
    return out


def jpeg_requantize(in_layout, in_coefs, out_layout):
    """Device: dequant -> IDCT -> resample -> FDCT -> quantise -> zigzag (host buffers in/out)."""
    in_coefs = np.ascontiguousarray(in_coefs, dtype=np.int16)
    out = np.zeros(out_layout.total_coefs, dtype=np.int16)
    _check(lib().b200_jpeg_requantize(C.byref(in_layout), in_coefs.ctypes.data_as(C.c_void_p), C.byref(out_layout), out.ctypes.data_as(C.c_void_p)))
    return out


def jpeg_encode_coefficients(layout, coefs, progressive=True):
    coefs = np.ascontiguousarray(coefs, dtype=np.int16)
    outp, outl = C.c_void_p(), C.c_size_t()
    _check(lib().b200_jpeg_encode_coefficients(C.byref(layout), coefs.ctypes.data_as(C.c_void_p), int(bool(progressive)), C.byref(outp), C.byref(outl)))
    return _take(outp, outl)


def jpeg_encode_coefficients_device(layout, coefs, progressive=True):
    """Same encoder on the GPU (block-parallel statistics / tables / bit packing / stuffing); bytes identical."""
    coefs = np.ascontiguousarray(coefs, dtype=np.int16)
    outp, outl = C.c_void_p(), C.c_size_t()
    f = lib().b200_jpeg_encode_coefficients_device
    f.restype = Status
    _check(f(C.byref(layout), coefs.ctypes.data_as(C.c_void_p), int(bool(progressive)), C.byref(outp), C.byref(outl)))
    return _take(outp, outl)


def set_entropy_mode(mode):
    """1 = device entropy encoder (default), 0 = host encoder."""
    return lib().b200_set_entropy_mode(int(mode))


def set_png_lossy(on):
    """b200_set_png_lossy: lossy PNG (png_optimize = 0) on the device quantiser (True) or refused with code 3 (False, the default)."""
    return lib().b200_set_png_lossy(int(bool(on)))


def set_png_resize(on):
    """b200_set_png_resize: PNG -> PNG with width / height resized on the device (True) or refused with code 3 (False, the default)."""
    return lib().b200_set_png_resize(int(bool(on)))


def set_webp_lossless_convert(on):
    """b200_set_webp_lossless_convert: convert_in_memory to WebP with webp_lossless on JPEG and PNG sources runs on the device (1) or
    is refused with code 3 (0, the default).  Any other value is refused with B200_ERR_INVALID_ARGUMENT."""
    return lib().b200_set_webp_lossless_convert(int(on))


def set_png_interlaced(on):
    """b200_set_png_interlaced: Adam7-interlaced PNG sources are accepted by every PNG leg (1) or refused with code 3 (0, the default).
    Any other value is refused with B200_ERR_INVALID_ARGUMENT."""
    return lib().b200_set_png_interlaced(int(on))


def set_jpeg_trellis(on):
    """b200_set_jpeg_trellis: trellis (rate-distortion) quantisation of lossy JPEG output (1) or plain quantisation (0, the default).
    Any other value is refused with B200_ERR_INVALID_ARGUMENT."""
    return lib().b200_set_jpeg_trellis(int(on))


def png_quantize(rgba, quality):
    """b200_png_quantize: rgba uint8 [h, w, 4] -> (palette uint8 [n, 4] as R, G, B, A; indices uint8 [h, w])."""
    rgba = np.ascontiguousarray(rgba, dtype=np.uint8)
    h, w = rgba.shape[:2]
    pal = np.zeros((256, 4), np.uint8)
    idx = np.zeros((h, w), np.uint8)
    n = C.c_int()
    _check(lib().b200_png_quantize(rgba.ctypes.data_as(C.c_void_p), w, h, int(quality), pal.ctypes.data_as(C.c_void_p), C.byref(n),
                                   idx.ctypes.data_as(C.c_void_p)))
    return pal[:n.value].copy(), idx


def set_gif(on):
    """b200_set_gif: GIF sources re-encoded on the device (True) or refused with code 3 (False, the default)."""
    return lib().b200_set_gif(int(bool(on)))


def gif_decode(data):
    """b200_gif_decode (host): -> (canvases uint8 [n, h, w, 4], delays list, loop or None)."""
    w, h, n, loop = C.c_int(), C.c_int(), C.c_int(), C.c_int()
    px, dl = C.POINTER(C.c_uint8)(), C.POINTER(C.c_int)()
    _check(lib().b200_gif_decode(data, C.c_size_t(len(data)), C.byref(w), C.byref(h), C.byref(n), C.byref(loop), C.byref(px), C.byref(dl)))
    size = n.value * h.value * w.value * 4
    canv = np.frombuffer(C.string_at(px, size), np.uint8).reshape(n.value, h.value, w.value, 4).copy()
    delays = list(np.frombuffer(C.string_at(dl, 4 * n.value), np.int32))
    lib().b200_free(px)
    lib().b200_free(dl)
    return canv, [int(x) for x in delays], (None if loop.value < 0 else loop.value)


def set_gif_convert(on):
    """b200_set_gif_convert: convert_in_memory to GIF from JPEG, PNG and WebP, and from GIF to JPEG, PNG and lossy WebP, runs on the
    device (1) or is refused with code 3 (0, the default).  Any other value is refused with B200_ERR_INVALID_ARGUMENT."""
    return lib().b200_set_gif_convert(int(on))


def gif_first_frame(data):
    """b200_gif_first_frame (host): frame 0 as the conversions read it -> uint8 [h, w, 4] (palette RGB with alpha 0 for the
    transparent index, all zero outside the frame's rectangle)."""
    w, h, px = C.c_int(), C.c_int(), C.POINTER(C.c_uint8)()
    _check(lib().b200_gif_first_frame(data, C.c_size_t(len(data)), C.byref(w), C.byref(h), C.byref(px)))
    out = np.frombuffer(C.string_at(px, h.value * w.value * 4), np.uint8).reshape(h.value, w.value, 4).copy()
    lib().b200_free(px)
    return out


def set_webp_anim(on):
    """b200_set_webp_anim: compress_in_memory on animated WebP sources runs on the device (1) or is refused with code 3 (0, the
    default).  Any other value is refused with B200_ERR_INVALID_ARGUMENT."""
    return lib().b200_set_webp_anim(int(on))


def set_png_zopfli(on):
    """b200_set_png_zopfli: png_force_zopfli takes the iterated optimal LZ77 parse on every PNG output (1) or is accepted and
    ignored (0, the default).  Any other value is refused with B200_ERR_INVALID_ARGUMENT."""
    return lib().b200_set_png_zopfli(int(on))


def set_webp_palette(on):
    """b200_set_webp_palette: every lossless WebP output also tries the colour-indexing (palette) transform on images of at most 256
    colours and keeps the smaller file (1), or never does (0, the default).  Any other value is refused with B200_ERR_INVALID_ARGUMENT."""
    return lib().b200_set_webp_palette(int(on))


def set_webp_bpred(on):
    """b200_set_webp_bpred: every lossy WebP output lets macroblocks take 4x4 intra prediction (B_PRED) where it scores lower in
    distortion + lambda * rate (1), or never (0, the default).  Any other value is refused with B200_ERR_INVALID_ARGUMENT."""
    return lib().b200_set_webp_bpred(int(on))


def png_lz77_zopfli(stream, bpp, stride):
    """b200_png_lz77_zopfli: the optimal parse of a filtered stream on the device -> tokens uint32[nt] in png_lz77's format."""
    s = np.ascontiguousarray(stream, dtype=np.uint8).reshape(-1)
    tok, nt = C.POINTER(C.c_uint32)(), C.c_size_t()
    _check(lib().b200_png_lz77_zopfli(s.ctypes.data_as(C.c_void_p), C.c_size_t(s.size), int(bpp), int(stride), C.byref(tok), C.byref(nt)))
    out = np.frombuffer(C.string_at(tok, nt.value * 4), dtype=np.uint32).copy()
    lib().b200_free(tok)
    return out


def webp_anim_decode(data):
    """b200_webp_anim_decode (host): -> (canvases uint8 [n, h, w, 4] as R, G, B, A, durations list in ms, loop, background bytes)."""
    w, h, n, loop = C.c_int(), C.c_int(), C.c_int(), C.c_int()
    bg = (C.c_uint8 * 4)()
    px, du = C.POINTER(C.c_uint8)(), C.POINTER(C.c_int)()
    _check(lib().b200_webp_anim_decode(data, C.c_size_t(len(data)), C.byref(w), C.byref(h), C.byref(n), C.byref(loop), bg, C.byref(px), C.byref(du)))
    size = n.value * h.value * w.value * 4
    canv = np.frombuffer(C.string_at(px, size), np.uint8).reshape(n.value, h.value, w.value, 4).copy()
    durations = [du[i] for i in range(n.value)]
    lib().b200_free(px)
    lib().b200_free(du)
    return canv, durations, loop.value, bytes(bg)


def gif_lzw(indices, min_code_size):
    """b200_gif_lzw (device): indices uint8 [n] -> GIF image data as sub-blocks with the terminator."""
    idx = np.ascontiguousarray(indices, dtype=np.uint8).reshape(-1)
    outp, outl = C.c_void_p(), C.c_size_t()
    _check(lib().b200_gif_lzw(idx.ctypes.data_as(C.c_void_p), C.c_size_t(idx.size), int(min_code_size), C.byref(outp), C.byref(outl)))
    return _take(outp, outl)


def jpeg_decode_planes(in_layout, in_coefs):
    """Device: dequant + IDCT + fancy upsample -> [ncomp, H, W] uint8 in the file's colour space."""
    in_coefs = np.ascontiguousarray(in_coefs, dtype=np.int16)
    out = np.zeros((in_layout.ncomp, in_layout.height, in_layout.width), dtype=np.uint8)
    _check(lib().b200_jpeg_decode_planes(C.byref(in_layout), in_coefs.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p)))
    return out


# ---- PNG stage entry points (lossless path) ----------------------------------------------------------------
class PngInfo(C.Structure):
    _fields_ = [("width", C.c_uint32), ("height", C.c_uint32), ("bit_depth", C.c_int32), ("color_type", C.c_int32),
                ("bpp", C.c_int32), ("row_bytes", C.c_uint64)]


def png_decode(data):
    """Host: parse + inflate + unfilter -> (PngInfo, raw uint8 [height, row_bytes])."""
    info, raw = PngInfo(), C.POINTER(C.c_uint8)()
    buf = (C.c_uint8 * len(data)).from_buffer_copy(data)
    _check(lib().b200_png_decode(buf, C.c_size_t(len(data)), C.byref(info), C.byref(raw)))
    n = info.height * info.row_bytes
    arr = np.frombuffer(C.string_at(raw, n), dtype=np.uint8).reshape(info.height, info.row_bytes).copy()
    lib().b200_free(raw)
    return info, arr


def png_decode_reduced(data):
    """Host: png_decode + the palette reduction of the lossless path -> (PngInfo, raw, palette [n, 4] RGBA or None)."""
    info, raw = PngInfo(), C.POINTER(C.c_uint8)()
    pal, npal = (C.c_uint8 * 1024)(), C.c_int(0)
    buf = (C.c_uint8 * len(data)).from_buffer_copy(data)
    _check(lib().b200_png_decode_reduced(buf, C.c_size_t(len(data)), C.byref(info), C.byref(raw), pal, C.byref(npal)))
    n = info.height * info.row_bytes
    arr = np.frombuffer(C.string_at(raw, n), dtype=np.uint8).reshape(info.height, info.row_bytes).copy()
    lib().b200_free(raw)
    palette = np.frombuffer(bytes(pal), dtype=np.uint8)[:4 * npal.value].reshape(-1, 4).copy() if npal.value else None
    return info, arr, palette


def png_filter(raw, bpp, strategy):
    """Device K6: raw uint8 [h, row_bytes] -> filtered [h, row_bytes + 1]."""
    raw = np.ascontiguousarray(raw, dtype=np.uint8)
    h, rb = raw.shape
    out = np.zeros((h, rb + 1), dtype=np.uint8)
    _check(lib().b200_png_filter(raw.ctypes.data_as(C.c_void_p), h, rb, int(bpp), int(strategy), out.ctypes.data_as(C.c_void_p)))
    return out


def png_lz77(stream, bpp, stride):
    """Device K7: filtered stream -> (tokens uint32[nt], hist uint32[316])."""
    s = np.ascontiguousarray(stream, dtype=np.uint8).reshape(-1)
    tok, nt = C.POINTER(C.c_uint32)(), C.c_size_t()
    hist = np.zeros(316, dtype=np.uint32)
    _check(lib().b200_png_lz77(s.ctypes.data_as(C.c_void_p), C.c_size_t(s.size), int(bpp), int(stride), C.byref(tok), C.byref(nt), hist.ctypes.data_as(C.c_void_p)))
    out = np.frombuffer(C.string_at(tok, nt.value * 4), dtype=np.uint32).copy()
    lib().b200_free(tok)
    return out, hist


def png_deflate_tokens(tokens, adler):
    """Host: dynamic-Huffman DEFLATE + zlib framing of a token stream."""
    tokens = np.ascontiguousarray(tokens, dtype=np.uint32)
    outp, outl = C.POINTER(C.c_uint8)(), C.c_size_t()
    _check(lib().b200_png_deflate_tokens(tokens.ctypes.data_as(C.c_void_p), C.c_size_t(tokens.size), C.c_uint32(adler), C.byref(outp), C.byref(outl)))
    return _take(outp, outl)


def webp_alpha_filter(alpha):
    """Host: (filter id 0..3, residual plane) the alpha plane is coded with."""
    a = np.ascontiguousarray(alpha, dtype=np.uint8)
    out = np.empty_like(a)
    k = lib().b200_webp_alpha_filter(a.ctypes.data_as(C.c_void_p), int(a.shape[1]), int(a.shape[0]), out.ctypes.data_as(C.c_void_p))
    return k, out


def webp_alpha_chunk(tokens, width, height, filter=0):
    """Host: ALPH chunk payload (VP8L-coded alpha plane) from the (filtered) plane's LZ77 tokens."""
    tokens = np.ascontiguousarray(tokens, dtype=np.uint32)
    outp, outl = C.POINTER(C.c_uint8)(), C.c_size_t()
    _check(lib().b200_webp_alpha_chunk(tokens.ctypes.data_as(C.c_void_p), C.c_size_t(tokens.size), int(width), int(height), int(filter), C.byref(outp), C.byref(outl)))
    return _take(outp, outl)


def webp_wrap_alpha(simple_file, alph, width, height):
    """Host: VP8X + ALPH + VP8 container from a simple lossy file and an ALPH payload."""
    outp, outl = C.POINTER(C.c_uint8)(), C.c_size_t()
    _check(lib().b200_webp_wrap_alpha(bytes(simple_file), C.c_size_t(len(simple_file)), bytes(alph), C.c_size_t(len(alph)), int(width), int(height), C.byref(outp), C.byref(outl)))
    return _take(outp, outl)


def png_device_times(data, level=3, iters=2):
    """{kernel: (ms per launch, launches per image)} of the PNG device pipeline on one image (b200_png_device_times)."""
    buf = C.create_string_buffer(1 << 14)
    _check(lib().b200_png_device_times(data, C.c_size_t(len(data)), int(level), int(iters), buf, C.c_size_t(len(buf))))
    out = {}
    for line in buf.value.decode().splitlines():
        name, ms, cnt = line.split()
        out[name] = (float(ms), int(cnt))
    return out


def png_level_strategies(level):
    out = (C.c_int * 10)()
    n = lib().b200_png_level_strategies(int(level), out)
    return list(out[:n])


# ---- WebP stage entry points (lossy VP8) ---------------------------------------------------------------------
def webp_encode_rgb(rgb, quality, want_stage=False):
    """Device K8 + host writer: planar uint8 [3, h, w] -> .webp bytes (and, if asked, (levels [nmb,25,16], modes [nmb,4]))."""
    rgb = np.ascontiguousarray(rgb, dtype=np.uint8)
    _, h, w = rgb.shape
    nmb = ((w + 15) // 16) * ((h + 15) // 16)
    levels = np.zeros((nmb, 25, 16), np.int16) if want_stage else None
    modes = np.zeros((nmb, 4), np.uint8) if want_stage else None
    outp, outl = C.POINTER(C.c_uint8)(), C.c_size_t()
    _check(lib().b200_webp_encode_rgb(rgb.ctypes.data_as(C.c_void_p), w, h, int(quality), C.byref(outp), C.byref(outl),
                                      levels.ctypes.data_as(C.c_void_p) if want_stage else None, modes.ctypes.data_as(C.c_void_p) if want_stage else None))
    data = _take(outp, outl)
    return (data, levels, modes) if want_stage else data


def webp_encode_rgb_bpred(rgb, quality, want_stage=False):
    """The B_PRED encoder whatever the switch says: planar uint8 [3, h, w] -> .webp bytes (and, if asked, (levels [nmb,25,16],
    modes [nmb,4], bmodes [nmb,16]))."""
    rgb = np.ascontiguousarray(rgb, dtype=np.uint8)
    _, h, w = rgb.shape
    nmb = ((w + 15) // 16) * ((h + 15) // 16)
    levels = np.zeros((nmb, 25, 16), np.int16) if want_stage else None
    modes = np.zeros((nmb, 4), np.uint8) if want_stage else None
    bmodes = np.zeros((nmb, 16), np.uint8) if want_stage else None
    p = lambda a: a.ctypes.data_as(C.c_void_p) if a is not None else None
    outp, outl = C.POINTER(C.c_uint8)(), C.c_size_t()
    _check(lib().b200_webp_encode_rgb_bpred(p(rgb), w, h, int(quality), C.byref(outp), C.byref(outl), p(levels), p(modes), p(bmodes)))
    data = _take(outp, outl)
    return (data, levels, modes, bmodes) if want_stage else data


def webp_write_levels_bpred(w, h, quality, levels, modes, bmodes):
    """Host writer with sub-block modes: (levels [nmb,25,16], modes [nmb,4], bmodes [nmb,16]) -> .webp bytes."""
    lv = np.ascontiguousarray(levels, dtype=np.int16); md = np.ascontiguousarray(modes, dtype=np.uint8); bm = np.ascontiguousarray(bmodes, dtype=np.uint8)
    outp, outl = C.POINTER(C.c_uint8)(), C.c_size_t()
    _check(lib().b200_webp_write_levels_bpred(int(w), int(h), int(quality), lv.ctypes.data_as(C.c_void_p), md.ctypes.data_as(C.c_void_p),
                                              bm.ctypes.data_as(C.c_void_p), C.byref(outp), C.byref(outl)))
    return _take(outp, outl)


def webp_decode(data):
    """Host VP8 decoder (bit-exact with libwebp): lossy .webp bytes -> uint8 [h, w, 3]."""
    w, h, ptr = C.c_int(), C.c_int(), C.POINTER(C.c_uint8)()
    _check(lib().b200_webp_decode(data, C.c_size_t(len(data)), C.byref(w), C.byref(h), C.byref(ptr)))
    arr = np.frombuffer(C.string_at(ptr, 3 * w.value * h.value), dtype=np.uint8).reshape(3, h.value, w.value).transpose(1, 2, 0).copy()
    lib().b200_free(ptr)
    return arr


def webp_decode_rgba(data):
    """Host WebP decoder incl. lossless files and alpha planes: bytes -> (uint8 [h, w, 3], uint8 [h, w] or None when opaque)."""
    w, h, ptr, ap = C.c_int(), C.c_int(), C.POINTER(C.c_uint8)(), C.POINTER(C.c_uint8)()
    _check(lib().b200_webp_decode_rgba(data, C.c_size_t(len(data)), C.byref(w), C.byref(h), C.byref(ptr), C.byref(ap)))
    arr = np.frombuffer(C.string_at(ptr, 3 * w.value * h.value), dtype=np.uint8).reshape(3, h.value, w.value).transpose(1, 2, 0).copy()
    lib().b200_free(ptr)
    alpha = None
    if ap:
        alpha = np.frombuffer(C.string_at(ap, w.value * h.value), dtype=np.uint8).reshape(h.value, w.value).copy()
        lib().b200_free(ap)
    return arr, alpha


def webp_write_levels(w, h, quality, levels, modes):
    """Host only: boolean-code a stage view (layout of webp_encode_rgb) into a .webp file."""
    levels = np.ascontiguousarray(levels, dtype=np.int16); modes = np.ascontiguousarray(modes, dtype=np.uint8)
    outp, outl = C.POINTER(C.c_uint8)(), C.c_size_t()
    _check(lib().b200_webp_write_levels(int(w), int(h), int(quality), levels.ctypes.data_as(C.c_void_p), modes.ctypes.data_as(C.c_void_p), C.byref(outp), C.byref(outl)))
    return _take(outp, outl)


def webp_qindex(quality):
    f = (C.c_int * 6)()
    q = lib().b200_webp_qindex(int(quality), f)
    return q, list(f)


def component_view(layout, coefs, c):
    """[bh, bw, 64] view (zigzag order) of component c inside a flat coefficient buffer."""
    o = layout.comp_offset[c]
    n = layout.bw[c] * layout.bh[c] * 64
    return coefs[o:o + n].reshape(layout.bh[c], layout.bw[c], 64)


class JpegPipe:
    """Device-resident FULL re-encode path (bench.py's `value`): n same-shaped baseline JPEGs uploaded once; run() enqueues
    Huffman decode -> transform -> Huffman encode for all of them behind `stream` without a host wait."""

    def __init__(self, datas, params, group=8):
        self.h = C.c_void_p()
        self.n = len(datas)
        self._inputs = BatchInputs(datas)
        _check(lib().b200_jpeg_pipe_create(self._inputs.ins, self._inputs.lens, self.n, C.byref(params), int(group), C.byref(self.h)))

    def run(self, stream=None, which=0):
        n = C.c_int(0)
        _check(lib().b200_jpeg_pipe_run(self.h, C.c_void_p(stream), int(which), C.byref(n)))
        return n.value

    def finish(self):
        """-> (entropy-coded bytes per image, images not settled by the device decoder, encoder retries)"""
        sizes = (C.c_size_t * self.n)()
        bad, retries = C.c_int(0), C.c_int(0)
        _check(lib().b200_jpeg_pipe_finish(self.h, sizes, C.byref(bad), C.byref(retries)))
        return list(sizes), bad.value, retries.value

    def fetch(self, index):
        outp, outl = C.c_void_p(), C.c_size_t()
        _check(lib().b200_jpeg_pipe_fetch(self.h, int(index), C.byref(outp), C.byref(outl)))
        return _take(outp, outl)

    def kernel_times(self, iters=3):
        """{kernel name: (ms per launch, launches per megabatch)} of ONE megabatch run alone with an event after every launch."""
        buf = C.create_string_buffer(1 << 14)
        _check(lib().b200_jpeg_pipe_kernel_times(self.h, int(iters), buf, C.c_size_t(len(buf))))
        out = {}
        for line in buf.value.decode().splitlines():
            name, ms, cnt = line.split()
            out[name] = (float(ms), int(cnt))
        return out

    def close(self):
        if self.h:
            lib().b200_jpeg_pipe_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def png_resize_samples(data, width=0, height=0):
    """b200_png_resize_samples (device): -> (PngInfo of the decoded type at the target size, rows uint8 [height, row_bytes] in PNG
    byte order).  width / height as in Params; both 0 = the expanded image at the source's size."""
    info, raw = PngInfo(), C.POINTER(C.c_uint8)()
    buf = (C.c_uint8 * len(data)).from_buffer_copy(data)
    _check(lib().b200_png_resize_samples(buf, C.c_size_t(len(data)), C.c_uint32(width), C.c_uint32(height), C.byref(info), C.byref(raw)))
    n = info.height * info.row_bytes
    arr = np.frombuffer(C.string_at(raw, n), dtype=np.uint8).reshape(info.height, info.row_bytes).copy()
    lib().b200_free(raw)
    return info, arr
