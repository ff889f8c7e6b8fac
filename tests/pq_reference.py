"""Plain reference of the lossy PNG palette quantiser -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Written from the rules in the header comment of caesium-clt_b200/csrc/png_quant_core.h, not from its code, and sharing nothing
with it or with the scalar twin (oracle/png_quant_oracle.c): every quantity is an exact integer (numpy int64 for sums that fit,
Python integers for the products that may not), every rounding is written out as floor(x + 1/2) of a rational, and the nearest-
entry search is exhaustive.  So a rule that is wrong in the shared header shows up as a difference between this module and both
the twin and the device.  Slow by design: meant for images of up to about 10^5 pixels.
"""
from fractions import Fraction

import numpy as np

MAX_COLOURS = 256
REFINE_PASSES = 3
# target mean squared error per quality: 2000 * ((100 - q) / 100)^3, rounded (no value falls on a half)
TARGET_MSE = [int(Fraction(2000 * (100 - q) ** 3, 100 ** 3) + Fraction(1, 2)) for q in range(101)]


def _round_div(num, den):
    """floor(num / den + 1/2) for non-negative integers (scalars or int64 arrays): the rounded quotient, halves up."""
    return (2 * num + den) // (2 * den)


def premultiply(rgba):
    """uint8 [..., 4] -> int64 [..., 4]: round(c * a / 255) for R, G, B (255 is odd, so no value falls on a half) and a itself."""
    v = np.asarray(rgba).astype(np.int64)
    a = v[..., 3:4]
    return np.concatenate([_round_div(v[..., :3] * a, 255), a], -1)


def entry_rgba(s, n):
    """a palette entry from the exact premultiplied sums s[4] of its n pixels: the rounded mean, un-premultiplied (rounded) to RGBA8"""
    m = [_round_div(int(s[c]), int(n)) for c in range(4)]
    a = m[3]
    assert a > 0, "entries are means of pixels that are not fully transparent"
    return tuple(min(255, _round_div(255 * m[c], a)) for c in range(3)) + (a,)


def entry_coords(e):
    """where an entry is compared: its RGBA premultiplied again"""
    return tuple(int(x) for x in premultiply(np.array(e, np.uint8)))


def _packed(rgba):
    v = np.ascontiguousarray(rgba, dtype=np.uint8).reshape(-1, 4).astype(np.uint64)
    return v[:, 0] | v[:, 1] << np.uint64(8) | v[:, 2] << np.uint64(16) | v[:, 3] << np.uint64(24)


def nearest(points, coords):
    """index of the nearest entry (squared distance over four channels; ties to the lower index) of every point, exhaustively"""
    pts = np.asarray(points, np.int64).reshape(-1, 4)
    c = np.asarray(coords, np.int64).reshape(-1, 4)
    out = np.empty(len(pts), np.int64)
    for i in range(0, len(pts), 4096):
        d = ((pts[i:i + 4096, None, :] - c[None, :, :]) ** 2).sum(-1)
        out[i:i + 4096] = d.argmin(1)          # argmin returns the first (lowest) index among equal minima
    return out


def _exact(rgba):
    """the at most 256 distinct values, entries that are not opaque first, each group in increasing R | G<<8 | B<<16 | A<<24"""
    keys = _packed(rgba)
    vals = sorted(set(int(k) for k in keys), key=lambda v: ((v >> 24) == 255, v))
    pal = np.array([[(v >> (8 * c)) & 255 for c in range(4)] for v in vals], np.uint8)
    pos = {v: i for i, v in enumerate(vals)}
    idx = np.array([pos[int(k)] for k in keys], np.uint8).reshape(rgba.shape[:2])
    return pal, idx


class _Cells:
    """the occupied 5-bit-per-channel cells of the pixels that are not fully transparent: coordinates, pixel counts, exact sums and
    representatives (rounded means)"""

    def __init__(self, p):
        p = p[p[:, 3] > 0]
        self.npix = len(p)
        cell = ((p[:, 0] >> 3) << 15) | ((p[:, 1] >> 3) << 10) | ((p[:, 2] >> 3) << 5) | (p[:, 3] >> 3)
        order = np.argsort(cell, kind="stable")
        cell, p = cell[order], p[order]
        starts = np.flatnonzero(np.r_[True, cell[1:] != cell[:-1]]) if len(cell) else np.zeros(0, np.int64)
        self.coord = np.stack([(cell[starts] >> (15 - 5 * c)) & 31 for c in range(4)], 1) if len(cell) else np.zeros((0, 4), np.int64)
        self.count = np.diff(np.r_[starts, len(cell)]).astype(np.int64)
        self.sums = np.add.reduceat(p, starts, axis=0) if len(cell) else np.zeros((0, 4), np.int64)
        self.rep = _round_div(self.sums, self.count[:, None])


def _box_stats(cells, members):
    n = int(cells.count[members].sum())
    w = cells.count[members][:, None]
    v = cells.rep[members]
    s1 = [int(x) for x in (w * v).sum(0)]
    s2 = [int(x) for x in (w * v * v).sum(0)]
    sse = [s2[c] - (s1[c] * s1[c]) // n for c in range(4)]       # per axis: s2 - floor(s1^2 / n)
    return n, sse


def _box_split(cells, members):
    """(axis, t) of a box's split, or None: the axis of largest SSE (ties to the lower axis) among those with two or more occupied
    coordinates; t is the last coordinate that stays, the weighted median (first t with 2 * cum >= n), capped at hi - 1"""
    n, sse = _box_stats(cells, members)
    best = None
    for c in range(4):
        if len(np.unique(cells.coord[members, c])) < 2:
            continue
        if best is None or sse[c] > sse[best]:
            best = c
    if best is None:
        return None
    marg = np.zeros(32, np.int64)
    np.add.at(marg, cells.coord[members, best], cells.count[members])
    occ = np.flatnonzero(marg)
    lo, hi = int(occ[0]), int(occ[-1])
    cum = 0
    t = lo
    for k in range(lo, hi + 1):
        cum += int(marg[k])
        t = k
        if 2 * cum >= n:
            break
    return best, min(t, hi - 1)


def _median_cut(cells, quality, max_boxes):
    q = min(100, max(0, quality))
    limit = TARGET_MSE[q] * cells.npix
    label = np.zeros(len(cells.count), np.int64)
    boxes = [np.arange(len(cells.count))]
    sse = [sum(_box_stats(cells, boxes[0])[1])]
    while len(boxes) < max_boxes and sum(sse) > limit:
        pick = None
        for b in sorted(range(len(boxes)), key=lambda b: (-sse[b], b)):       # largest SSE first, ties to the lower box
            split = _box_split(cells, boxes[b])
            if split is not None:
                pick = b
                break
        if pick is None:
            break
        axis, t = split
        m = boxes[pick]
        up = cells.coord[m, axis] > t
        boxes.append(m[up])
        boxes[pick] = m[~up]
        label[m[up]] = len(boxes) - 1
        sse[pick] = sum(_box_stats(cells, boxes[pick])[1])
        sse.append(sum(_box_stats(cells, boxes[-1])[1]))
    return label, len(boxes)


def _entries(cells, label, k):
    """entries from the pixels of each label 0..k-1; labels without pixels are dropped, the others keep their order"""
    out = []
    for b in range(k):
        m = label == b
        n = int(cells.count[m].sum())
        if n:
            out.append(entry_rgba([int(x) for x in cells.sums[m].sum(0)], n))
    return out


def palette_of(rgba, quality):
    """the quantised palette (RGBA tuples, the reserved (0, 0, 0, 0) first when the source has fully transparent pixels)"""
    p = premultiply(np.asarray(rgba, np.uint8).reshape(-1, 4))
    clear = bool((p[:, 3] == 0).any())
    cells = _Cells(p)
    ent = []
    if cells.npix:
        label, nb = _median_cut(cells, quality, MAX_COLOURS - clear)
        ent = _entries(cells, label, nb)
        for _ in range(REFINE_PASSES):
            ent = _entries(cells, nearest(cells.rep, [entry_coords(e) for e in ent]), len(ent))
    ent = [e for e in ent if e[3] != 255] + [e for e in ent if e[3] == 255]
    return ([(0, 0, 0, 0)] if clear else []) + ent


def dither(rgba, palette):
    """raster Floyd-Steinberg (7, 3, 5, 1 sixteenths) on premultiplied values against the entries after the reserved one: the
    incoming error rounded half away from zero, the target clamped to 0..255; fully transparent pixels take index 0 and neither
    take nor pass error.  Returns (indices uint8 [h, w], targets int64 [h, w, 4]; a transparent pixel's target is -1)."""
    rgba = np.asarray(rgba, np.uint8)
    h, w = rgba.shape[:2]
    p = premultiply(rgba).tolist()
    clear = int((rgba[:, :, 3] == 0).any())
    coords = [entry_coords(e) for e in palette[clear:]]
    carr = np.array(coords, np.int64).reshape(-1, 4)
    idx = np.zeros((h, w), np.uint8)
    tgt = np.full((h, w, 4), -1, np.int64)
    up = [[0] * 4 for _ in range(w + 2)]
    for y in range(h):
        cur = [[0] * 4 for _ in range(w + 2)]            # cur[x + 1]: this row's error at x
        for x in range(w):
            px = p[y][x]
            if px[3] == 0:
                continue
            t = []
            for c in range(4):
                e16 = 7 * cur[x][c] + 3 * up[x + 2][c] + 5 * up[x + 1][c] + up[x][c]
                r = (abs(e16) + 8) // 16                 # |e16| / 16 rounded half up, then the sign back: half away from zero
                t.append(min(255, max(0, px[c] + (r if e16 >= 0 else -r))))
            k = int(((carr - t) ** 2).sum(1).argmin())
            idx[y, x] = clear + k
            tgt[y, x] = t
            cur[x + 1] = [t[c] - coords[k][c] for c in range(4)]
        up = cur
    return idx, tgt


def png_quantize_ref(rgba, quality):
    """rgba uint8 [h, w, 4] -> (palette uint8 [n, 4], indices uint8 [h, w]), as the quantiser's rules define them"""
    rgba = np.ascontiguousarray(rgba, dtype=np.uint8)
    if len(np.unique(_packed(rgba))) <= 256:
        return _exact(rgba)
    pal = palette_of(rgba, quality)
    idx, _ = dither(rgba, pal)
    return np.array(pal, np.uint8).reshape(-1, 4), idx


def check_dither(rgba, palette, indices):
    """Checks a quantiser result against the definition rather than one loop: re-derives every target from the indices alone (the
    error a pixel passes on is its target minus the entry its index names) and confirms that each pixel that is not fully
    transparent holds the exhaustive nearest entry of its target (ties to the lower index, never the reserved entry), and that
    fully transparent pixels hold index 0 of a reserved (0, 0, 0, 0).  A source with at most 256 distinct values must come back
    exactly.  Returns (targets int64 [h, w, 4] with -1 where transparent, pixels whose target the clamp changed) for callers that
    measure what a source exercised (None on the exact path)."""
    rgba = np.asarray(rgba, np.uint8)
    palette = np.asarray(palette, np.uint8).reshape(-1, 4)
    indices = np.asarray(indices)
    h, w = rgba.shape[:2]
    assert indices.shape == (h, w) and len(palette) >= 1 and int(indices.max()) < len(palette)
    if len(np.unique(_packed(rgba))) <= 256:
        assert np.array_equal(palette[indices], rgba), "exact path: the palette applied to the indices is not the source"
        return None
    clear = int((rgba[:, :, 3] == 0).any())
    if clear:
        assert tuple(palette[0]) == (0, 0, 0, 0), f"reserved entry is {tuple(palette[0])}"
    coords = np.array([entry_coords(tuple(int(v) for v in e)) for e in palette], np.int64)
    p = premultiply(rgba).tolist()
    tgt = np.full((h, w, 4), -1, np.int64)
    cl = coords.tolist()
    clamped = 0
    up = [[0] * 4 for _ in range(w + 2)]
    for y in range(h):
        cur = [[0] * 4 for _ in range(w + 2)]
        for x in range(w):
            px = p[y][x]
            if px[3] == 0:
                assert indices[y, x] == 0, f"transparent pixel ({x}, {y}) has index {indices[y, x]}"
                continue
            raw = []
            for c in range(4):
                e16 = 7 * cur[x][c] + 3 * up[x + 2][c] + 5 * up[x + 1][c] + up[x][c]
                r = (2 * abs(e16) + 16) // 32            # floor(|e16| / 16 + 1/2)
                raw.append(px[c] + (r if e16 >= 0 else -r))
            t = [min(255, max(0, v)) for v in raw]
            clamped += t != raw
            tgt[y, x] = t
            k = int(indices[y, x])
            cur[x + 1] = [t[c] - cl[k][c] for c in range(4)]
        up = cur
    live = rgba[:, :, 3] > 0
    want = clear + nearest(tgt[live], coords[clear:])
    got = indices[live].astype(np.int64)
    bad = np.flatnonzero(want != got)
    if len(bad):
        ys, xs = np.nonzero(live)
        i = bad[0]
        raise AssertionError(f"pixel ({xs[i]}, {ys[i]}) target {tuple(tgt[ys[i], xs[i]])}: index {got[i]}, nearest entry {want[i]} "
                             f"({len(bad)} pixels differ)")
    return tgt, clamped


def ties(rgba, palette, targets):
    """pixels whose target has two or more nearest entries (the tie rule decided their index)"""
    rgba = np.asarray(rgba, np.uint8)
    live = rgba[:, :, 3] > 0
    clear = int((rgba[:, :, 3] == 0).any())
    coords = np.array([entry_coords(tuple(int(v) for v in e)) for e in np.asarray(palette)[clear:]], np.int64)
    t = targets[live]
    n = 0
    for i in range(0, len(t), 4096):
        d = ((t[i:i + 4096, None, :] - coords[None]) ** 2).sum(-1)
        n += int(((d == d.min(1, keepdims=True)).sum(1) > 1).sum())
    return n
