"""Hand-framed PNG sources for the resize tests: every legal colour type x bit depth, with and without tRNS, rows filtered with the
oracle's per-row heuristic (so the un-filter sees every filter type).  Palette sources use an index past PLTE and past tRNS."""
import struct
import zlib

import numpy as np

from pngutil import chunk, frame_png

# (colour type, bit depth, with tRNS)
LEGAL = [(0, d, t) for d in (1, 2, 4, 8, 16) for t in (False, True)] + \
        [(2, d, t) for d in (8, 16) for t in (False, True)] + \
        [(3, d, t) for d in (1, 2, 4, 8) for t in (False, True)] + \
        [(4, d, False) for d in (8, 16)] + [(6, d, False) for d in (8, 16)]
NIN = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}


def case_id(ct, bd, trns):
    return f"ct{ct}_d{bd}{'_trns' if trns else ''}"


def _values(h, w, nin, bd, seed):
    """unscaled samples [h, w, nin]: smooth gradients + noise, spanning the depth's range"""
    top = (1 << bd) - 1
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    out = []
    for c in range(nin):
        base = 0.5 + 0.45 * np.sin(xx / (5.0 + 2 * c) + c) * np.cos(yy / (7.0 + c))
        out.append(np.clip(base + rng.normal(0, 0.04, (h, w)), 0, 1) * top)
    return np.clip(np.rint(np.stack(out, -1)), 0, top).astype(np.int64)


def _pack(v, bd):
    """samples [h, w, nin] -> un-filtered rows uint8 [h, row_bytes]"""
    h, w, nin = v.shape
    flat = v.reshape(h, w * nin)
    if bd == 16:
        return flat.astype(">u2").view(np.uint8).reshape(h, -1)
    if bd == 8:
        return flat.astype(np.uint8)
    per = 8 // bd
    rb = (w * nin * bd + 7) // 8
    rows = np.zeros((h, rb), np.uint8)
    for k in range(w * nin):
        rows[:, k // per] |= (flat[:, k] << (8 - bd - (k % per) * bd)).astype(np.uint8)
    return rows


def make(O, ct, bd, trns, w, h, seed=0):
    """-> dict(png, raw, width, height, bit_depth, color_type, plte, trns, values)"""
    nin = NIN[ct]
    v = _values(h, w, nin, bd, seed)
    plte, tr = b"", b""
    if ct == 3:
        npal = max(1, (1 << bd) - 1 - (1 << bd) // 8)            # some indices lie past PLTE
        v[0, 0, 0] = (1 << bd) - 1                               # at least one of them is used
        rng = np.random.default_rng(seed + 100)
        plte = bytes(rng.integers(0, 256, 3 * npal, dtype=np.uint8))
        if trns:
            tr = bytes(rng.integers(0, 256, max(1, npal // 2), dtype=np.uint8))   # entries past tRNS are opaque
    elif trns:
        key = v[h // 2, w // 3] if h * w > 1 else v[0, 0]
        v[: max(1, h // 4), : max(1, w // 4)] = key                                 # the key covers a block
        tr = b"".join(struct.pack(">H", int(k)) for k in key)
    raw = _pack(v, bd)
    bpp = max(1, nin * bd // 8)
    filt = O.png_filter(raw, bpp, O.PNG_STRATEGIES["minsum"])
    extra = (chunk(b"PLTE", plte) if plte else b"") + (chunk(b"tRNS", tr) if tr else b"")
    png = frame_png(w, h, bd, ct, zlib.compress(filt.tobytes()), extra)
    return dict(png=png, raw=raw, width=w, height=h, bit_depth=bd, color_type=ct, plte=plte, trns=tr, values=v)
