"""ctypes binding of the PNG resize twin in oracle/png_resize_oracle.c (built into oracle/liboracle.so with the rest of the oracle)
-- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

png_resize: un-filtered PNG rows + IHDR / PLTE / tRNS -> the image crate's decoded type, Lanczos3 to the target size (u8 planes
through orc_resize_plane_lanczos3, u16 planes through orc_resize_plane_lanczos3_u16), packed back into PNG rows."""
import ctypes as C

import numpy as np

from .oracle import OracleError, compute_dimensions, lib, resize_plane
from .png_quant import png_quantize


def decoded_type(color_type, bit_depth, trns=b""):
    """(colour type, channels, depth) of the image crate's buffer for a PNG source."""
    ct, ch, d = C.c_int(), C.c_int(), C.c_int()
    lib().orc_png_decoded_type(int(color_type), int(bit_depth), C.c_size_t(len(trns)), C.byref(ct), C.byref(ch), C.byref(d))
    return ct.value, ch.value, d.value


def expand_planes(raw, width, height, bit_depth, color_type, plte=b"", trns=b""):
    """raw uint8 [height, row_bytes] -> planes [channels, height, width] (uint8 for depth 8, uint16 for depth 16)."""
    raw = np.ascontiguousarray(raw, dtype=np.uint8)
    _, ch, depth = decoded_type(color_type, bit_depth, trns)
    planes = np.zeros((ch, height, width), np.uint16)
    pl, tr = bytes(plte) or b"\0", bytes(trns) or b"\0"
    lib().orc_png_expand_planes.restype = C.c_int
    lib().orc_png_expand_planes(raw.ctypes.data_as(C.c_void_p), C.c_size_t(raw.shape[1]), int(width), int(height), int(color_type), int(bit_depth),
                                pl, C.c_size_t(len(plte)), tr, C.c_size_t(len(trns)), planes.ctypes.data_as(C.c_void_p))
    return planes if depth == 16 else planes.astype(np.uint8)


def resize_plane_u16(plane, nw, nh):
    plane = np.ascontiguousarray(plane, dtype=np.uint16)
    h, w = plane.shape
    out = np.zeros((nh, nw), np.uint16)
    lib().orc_resize_plane_lanczos3_u16.restype = C.c_int
    if lib().orc_resize_plane_lanczos3_u16(plane.ctypes.data_as(C.c_void_p), w, h, w, out.ctypes.data_as(C.c_void_p), nw, nh, nw):
        raise OracleError("resize failed")
    return out


def pack_rows(planes):
    """planes [channels, h, w] uint8 / uint16 -> PNG rows uint8 [h, w * channels * bytes] (16 bits big-endian)."""
    inter = np.moveaxis(planes, 0, -1)
    if planes.dtype == np.uint16:
        inter = inter.astype(">u2")
    return np.ascontiguousarray(inter).view(np.uint8).reshape(planes.shape[1], -1)


def png_resize(raw, width, height, bit_depth, color_type, plte=b"", trns=b"", want_w=0, want_h=0):
    """-> (dict(width, height, bit_depth, color_type, channels, row_bytes), rows uint8 [nh, row_bytes]).  want_w / want_h as in
    CSParameters (compute_dimensions); both 0 = the expanded image at the source's size."""
    nw, nh = compute_dimensions(width, height, want_w, want_h) if (want_w or want_h) else (width, height)
    ct, ch, depth = decoded_type(color_type, bit_depth, trns)
    planes = expand_planes(raw, width, height, bit_depth, color_type, plte, trns)
    one = resize_plane_u16 if depth == 16 else resize_plane
    out = np.stack([one(planes[c], nw, nh) for c in range(ch)])
    rows = pack_rows(out)
    return dict(width=nw, height=nh, bit_depth=depth, color_type=ct, channels=ch, row_bytes=rows.shape[1]), rows


def rows_to_rgba8(info, rows):
    """resized rows -> RGBA8 [h, w, 4] as the lossy leg's quantiser sees them (16 bits: the high byte)."""
    ch = info["channels"]
    px = rows.reshape(info["height"], info["width"], ch, info["bit_depth"] // 8)[..., 0]
    if ch == 1:
        return np.concatenate([np.repeat(px, 3, 2), np.full(px.shape[:2] + (1,), 255, np.uint8)], 2)
    if ch == 2:
        return np.concatenate([np.repeat(px[:, :, :1], 3, 2), px[:, :, 1:]], 2)
    if ch == 3:
        return np.concatenate([px, np.full(px.shape[:2] + (1,), 255, np.uint8)], 2)
    return np.ascontiguousarray(px)


def quantized_rgba(info, rows, quality):
    """the quantiser twin over the resized image: its palette applied to its indices, RGBA8 [h, w, 4]."""
    pal, idx = png_quantize(rows_to_rgba8(info, rows), quality)
    return pal[idx]
