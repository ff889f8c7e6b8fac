"""An Adam7 PNG writer in numpy + zlib for the interlaced-input tests (Pillow reads Adam7 files but cannot write them).

adam7_pair() writes one image twice: as an Adam7 file, whose pass rows take filter types drawn from a seeded RNG (all five appear,
Paeth on 1-byte pixels included), and as its non-interlaced twin -- the same pixels, chunks, PLTE and tRNS, interlace method 0.
Padding bits after a row's last pixel are zero in the twin's rows, so a decoder that de-interlaces correctly gives identical rows."""
import zlib

import numpy as np

from png_webp_cases import CHANNELS, DEPTHS, row_bytes, samples
from pngutil import chunk

# pass p: (x0, y0, dx, dy), PNG 8.2
PASSES = [(0, 0, 8, 8), (4, 0, 8, 8), (0, 4, 4, 8), (2, 0, 4, 4), (0, 2, 2, 4), (1, 0, 2, 2), (0, 1, 1, 2)]
SHAPES = [(1, 1), (1, 9), (9, 1), (2, 2), (3, 5), (5, 3), (7, 7), (8, 8), (9, 9), (33, 17)]     # (w, h): every combination of empty passes


def pairs():
    """every legal (colour type, bit depth)"""
    return [(ct, bd) for ct, depths in DEPTHS.items() for bd in depths]


def layout(w, h, bits):
    """restatement: per pass (w, h, rb, filt_off, raw_off), total inflated and pass-packed bytes"""
    out, fo, ro = [], 0, 0
    for x0, y0, dx, dy in PASSES:
        pw = -(-(w - x0) // dx) if w > x0 else 0
        ph = -(-(h - y0) // dy) if h > y0 else 0
        if not pw or not ph:
            pw = ph = 0
        rb = (pw * bits + 7) // 8
        out.append((pw, ph, rb, fo, ro))
        fo += ph * (rb + 1) if ph else 0
        ro += ph * rb
    return out, fo, ro


def _paeth(a, b, c):
    p = a + b - c
    pa, pb, pc = np.abs(p - a), np.abs(p - b), np.abs(p - c)
    return np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))


def filter_rows(rows, bpp, types):
    """PNG 9.2 filtering of rows uint8 [n, rb] with one filter type per row -> [n, rb + 1] (filter byte first)"""
    n, rb = rows.shape
    out = np.zeros((n, rb + 1), np.uint8)
    r = rows.astype(np.int64)
    for y in range(n):
        x = r[y]
        up = r[y - 1] if y else np.zeros(rb, np.int64)
        left = np.concatenate([np.zeros(min(bpp, rb), np.int64), x[:-bpp]]) if rb > bpp else np.zeros(rb, np.int64)
        ul = np.concatenate([np.zeros(min(bpp, rb), np.int64), up[:-bpp]]) if rb > bpp else np.zeros(rb, np.int64)
        t = int(types[y])
        pred = [np.zeros(rb, np.int64), left, up, (left + up) >> 1, _paeth(left, up, ul)][t]
        out[y, 0] = t
        out[y, 1:] = ((x - pred) & 0xFF).astype(np.uint8)
    return out


def _pack(vals, bd):
    """sample values [n, w] (one channel, bd < 8) -> packed rows [n, ceil(w * bd / 8)], zero padding bits"""
    n, w = vals.shape
    bits = ((vals[..., None] >> np.arange(bd - 1, -1, -1)) & 1).astype(np.uint8).reshape(n, w * bd)
    return np.packbits(bits, axis=1)


def pass_rows(raw, w, h, ct, bd):
    """the seven passes' un-filtered rows (a pass with no pixels: an empty [0, 0] array)"""
    nc = CHANNELS[ct]
    out = []
    if bd < 8:
        vals = samples(raw, w, ct, bd)[..., 0]
    else:
        B = nc * bd // 8
        pix = np.asarray(raw, np.uint8)[:, :w * B].reshape(h, w, B)
    for x0, y0, dx, dy in PASSES:
        if x0 >= w or y0 >= h:
            out.append(np.zeros((0, 0), np.uint8))
        elif bd < 8:
            out.append(_pack(vals[y0::dy, x0::dx], bd))
        else:
            sub = pix[y0::dy, x0::dx]
            out.append(np.ascontiguousarray(sub.reshape(sub.shape[0], -1)))
    return out


def zero_padding(raw, w, ct, bd):
    """raw rows with the bits after each row's last pixel cleared"""
    raw = np.array(raw, np.uint8)
    used = w * CHANNELS[ct] * bd
    if used % 8:
        raw[:, -1] &= (0xFF << (8 - used % 8)) & 0xFF
    return raw


def _file(w, h, ct, bd, interlace, zstream, plte, trns, before, after, split):
    ihdr = w.to_bytes(4, "big") + h.to_bytes(4, "big") + bytes([bd, ct, 0, 0, interlace])
    body = chunk(b"IHDR", ihdr) + before
    if plte:
        body += chunk(b"PLTE", plte)
    if trns:
        body += chunk(b"tRNS", trns)
    step = max(1, -(-len(zstream) // split))
    body += b"".join(chunk(b"IDAT", zstream[i:i + step]) for i in range(0, len(zstream), step))
    return b"\x89PNG\r\n\x1a\n" + body + after + chunk(b"IEND", b"")


def adam7_filtered(raw, w, h, ct, bd, seed=0):
    """the Adam7 file's inflated stream: each non-empty pass's rows, filtered with seeded random filter types"""
    rng = np.random.default_rng(seed)
    bpp = max(1, CHANNELS[ct] * bd // 8)
    parts = []
    for rows in pass_rows(raw, w, h, ct, bd):
        if rows.size:
            parts.append(filter_rows(rows, bpp, rng.integers(0, 5, rows.shape[0])).tobytes())
    return b"".join(parts)


def adam7_pair(raw, w, h, ct, bd, seed=0, plte=b"", trns=b"", before=b"", after=b"", split=1, level=6):
    """(Adam7 file, non-interlaced twin) of the rows raw [h, row_bytes] (padding bits are cleared first)"""
    raw = zero_padding(raw, w, ct, bd)
    bpp = max(1, CHANNELS[ct] * bd // 8)
    inter = zlib.compress(adam7_filtered(raw, w, h, ct, bd, seed), level)
    twin = zlib.compress(filter_rows(raw, bpp, np.random.default_rng(seed + 1).integers(0, 5, h)).tobytes(), level)
    return (_file(w, h, ct, bd, 1, inter, plte, trns, before, after, split),
            _file(w, h, ct, bd, 0, twin, plte, trns, before, after, split))


ANCILLARY_BEFORE = chunk(b"gAMA", (45455).to_bytes(4, "big")) + chunk(b"tEXt", b"Comment\0adam7 test")
ANCILLARY_AFTER = chunk(b"tEXt", b"Author\0nobody")


def adam7_case(w, h, ct, bd, seed=0, trns=None, split=3):
    """(Adam7 file, twin, raw rows, plte, trns) of random samples; trns: None, 'key' (colour types 0 and 2: the first pixel's value)
    or 'partial' (colour type 3: soft alphas on the first entries).  Ancillary chunks before and after IDAT, IDAT in `split` chunks."""
    rng = np.random.default_rng(seed)
    raw = zero_padding(rng.integers(0, 256, (h, row_bytes(w, ct, bd)), dtype=np.uint8), w, ct, bd)
    plte, t = b"", b""
    if ct == 3:
        plte = rng.integers(0, 256, 3 << bd, dtype=np.uint8).tobytes()
        if trns:
            t = bytes([0, 128, 255, 7][:min(4, 1 << bd)])
    elif trns and ct in (0, 2):
        s = samples(raw[:1], 1, ct, bd)[0, 0]
        t = b"".join(int(v).to_bytes(2, "big") for v in s)
    inter, twin = adam7_pair(raw, w, h, ct, bd, seed, plte, t, ANCILLARY_BEFORE, ANCILLARY_AFTER, split)
    return inter, twin, raw, plte, t
