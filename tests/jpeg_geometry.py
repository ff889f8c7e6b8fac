"""JPEG files at any per-component sampling geometry, for the geometry tests (not a fixture: imported by the test modules).

Pillow writes only 4:4:4, 4:2:2, 4:2:0 and grey.  make_jpeg() builds the coefficient image by hand -- a tools.synth picture,
box-downsampled per component, FDCT + quantised block by block by the oracle, plus a sparse high-frequency sprinkle -- and
has the oracle's writer code it in the requested geometry.  Every file is pinned to libjpeg-turbo (through Pillow) inside
the helper: at a legal geometry its native YCbCr decode must equal the oracle's, and at an illegal one (more than 10 blocks in
an interleaved MCU, or a sampling factor that does not divide the largest) libjpeg-turbo must refuse it.  So a test that
compares the product with the oracle at some geometry fails where the oracle is wrong, instead of agreeing with it."""
import functools
import io
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

# (Y, Cb, Cr) sampling factors (h, v); 4:4:0 is Y 1x2, which cameras write for rotated 4:2:2
GEOMETRIES = {
    "y12": ((1, 2), (1, 1), (1, 1)),
    "y41": ((4, 1), (1, 1), (1, 1)),
    "y14": ((1, 4), (1, 1), (1, 1)),
    "y42": ((4, 2), (1, 1), (1, 1)),
    "y24": ((2, 4), (1, 1), (1, 1)),
    "y31": ((3, 1), (1, 1), (1, 1)),
    "y13": ((1, 3), (1, 1), (1, 1)),
    "y32": ((3, 2), (1, 1), (1, 1)),
    "cr22": ((2, 2), (1, 1), (2, 2)),
    "c22": ((1, 1), (2, 2), (2, 2)),
    "c21": ((2, 2), (2, 1), (2, 1)),
    "c12": ((2, 2), (1, 2), (1, 2)),
    "grey22": ((2, 2),),
    "s420": ((2, 2), (1, 1), (1, 1)),
}
OVERSIZED = {                       # legal factors, but more than 10 blocks in the interleaved MCU
    "y33_11": ((3, 3), (1, 1), (1, 1)),
    "y42_c21_12": ((4, 2), (2, 1), (2, 1)),
    "y44_18": ((4, 4), (1, 1), (1, 1)),
}
FRACTIONAL = ((3, 1), (2, 1), (1, 1))     # Cb's 2 does not divide hmax = 3: no integral upsampling ratio
SMALL_SIZES = [(1, 1), (2, 3), (17, 9), (67, 45), (130, 61), (513, 33)]


def mcu_blocks(factors):
    return 1 if len(factors) == 1 else sum(h * v for h, v in factors)


def fractional(factors):
    hmax, vmax = max(h for h, _ in factors), max(v for _, v in factors)
    return any(hmax % h or vmax % v for h, v in factors)


def geometry(w, h, factors):
    """Per component (hs, vs, cw, ch, rbw, rbh, bw, bh) as the readers derive it (a grey file is one block per MCU)."""
    fs = [(1, 1)] if len(factors) == 1 else list(factors)
    hmax, vmax = max(f[0] for f in fs), max(f[1] for f in fs)
    mcux, mcuy = -(-w // (8 * hmax)), -(-h // (8 * vmax))
    out = []
    for hs, vs in fs:
        cw, ch = -(-w * hs // hmax), -(-h * vs // vmax)
        out.append((hs, vs, cw, ch, -(-cw // 8), -(-ch // 8), mcux * hs, mcuy * vs))
    return out, (hmax, vmax, mcux, mcuy)


def block_row_widths(factors, n):
    """An odd image width at which component c's real block row is exactly n blocks, for each component c."""
    fs = [(1, 1)] if len(factors) == 1 else list(factors)
    hmax = max(f[0] for f in fs)
    return [(8 * n - 4) * hmax // hs + 1 for hs, _ in fs]


def sizes_for(factors):
    """SMALL_SIZES plus widths that put some component's real block row at 31, 32, 33 (the 32-block warp tile) and 257 (past the
    256-block CTA), the component chosen per n."""
    fs = [(1, 1)] if len(factors) == 1 else list(factors)
    out = list(SMALL_SIZES)
    for i, n in enumerate((31, 32, 33)):
        out.append((block_row_widths(factors, n)[i % len(fs)], 11))
    widest = max(range(len(fs)), key=lambda c: fs[c][0])
    out.append((block_row_widths(factors, 257)[widest], 5))
    return out


def libjpeg_native(data):
    """libjpeg-turbo's decode in the file's own colour space (fancy upsampling), [ncomp, H, W]."""
    from PIL import Image
    im = Image.open(io.BytesIO(data))
    im.draft("YCbCr" if im.mode != "L" else "L", im.size)
    a = np.asarray(im)
    return a[None] if a.ndim == 2 else np.ascontiguousarray(a.transpose(2, 0, 1))


def libjpeg_refuses(data):
    try:
        libjpeg_native(data)
    except (OSError, SyntaxError, ValueError):
        return True
    return False


def _box_down(plane, rx, ry, cw, ch):
    """plane [H, W] -> [ch, cw]: mean of each rx x ry box (edge-replicated), nearest sample where the ratio is not integral."""
    H, W = plane.shape
    if float(rx).is_integer() and float(ry).is_integer():
        rx, ry = int(rx), int(ry)
        p = np.pad(plane.astype(np.int32), ((0, ch * ry - H), (0, cw * rx - W)), mode="edge")
        s = p.reshape(ch, ry, cw, rx).sum(axis=(1, 3))
        return ((s + rx * ry // 2) // (rx * ry)).astype(np.uint8)
    ys = np.minimum((np.arange(ch) * ry).astype(int), H - 1)
    xs = np.minimum((np.arange(cw) * rx).astype(int), W - 1)
    return plane[ys][:, xs]


@functools.lru_cache(maxsize=None)
def _coefficients(w, h, factors, seed, quality):
    from oracle import oracle as O
    from tools.synth import synth_rgb
    rgb = np.ascontiguousarray(synth_rgb(w, h, seed).transpose(2, 0, 1))
    planes = O.rgb_to_ycc(rgb)
    geo, (hmax, vmax, _, _) = geometry(w, h, factors)
    rng = np.random.default_rng(seed * 7919 + w * 31 + h)
    coefs, qts = [], []
    for c, (hs, vs, cw, ch, rbw, rbh, bw, bh) in enumerate(geo):
        q = O.quant_table(quality, 0 if c == 0 else 1)
        ds = _box_down(planes[c], hmax / hs, vmax / vs, cw, ch)
        full = np.pad(ds, ((0, bh * 8 - ch), (0, bw * 8 - cw)), mode="edge")
        co = np.zeros((bh, bw, 64), np.int16)
        for by in range(bh):
            for bx in range(bw):
                co[by, bx] = O.fdct_quant(full[by * 8:by * 8 + 8, bx * 8:bx * 8 + 8], q)[1].reshape(64)
        sprinkle = rng.random((bh, bw)) < 0.08               # a few high-frequency terms the picture alone would quantise away
        pos = rng.integers(36, 64, size=(bh, bw))
        val = rng.choice(np.array([-3, -2, -1, 1, 2, 3], np.int16), size=(bh, bw))
        by, bx = np.nonzero(sprinkle)
        co[by, bx, pos[by, bx]] += val[by, bx]
        coefs.append(co)
        qts.append(q)
    return coefs, qts


@functools.lru_cache(maxsize=None)
def make_jpeg(w, h, factors, progressive=False, seed=0, quality=75):
    """A w x h JPEG with per-component sampling factors `factors` ((h, v) per component, 1 or 3 components, each in 1..4),
    baseline or progressive; checked against libjpeg-turbo before it is returned (see the module docstring)."""
    import ctypes as C
    from oracle import oracle as O
    factors = tuple(tuple(f) for f in factors)
    assert len(factors) in (1, 3) and all(1 <= f <= 4 for hv in factors for f in hv)
    coefs, qts = _coefficients(w, h, factors, seed, quality)
    geo, (hmax, vmax, mcux, mcuy) = geometry(w, h, factors)
    j = O.Jpeg()
    s = j.s
    s.width, s.height, s.ncomp = w, h, len(factors)
    for c, (hs, vs, cw, ch, rbw, rbh, bw, bh) in enumerate(geo):
        s.hs[c], s.vs[c] = factors[c]                      # as written in SOF (a grey 2x2 header stays 2x2 in the file)
        s.tq[c], s.cid[c] = (0 if c == 0 else 1), c + 1
        s.cw[c], s.ch[c], s.rbw[c], s.rbh[c], s.bw[c], s.bh[c] = cw, ch, rbw, rbh, bw, bh
        s.coef[c] = coefs[c].ctypes.data_as(C.POINTER(C.c_int16))
    for t in range(2 if len(factors) == 3 else 1):
        for k in range(64):
            s.qt[t][k] = int(qts[t][k])
        s.qt_present[t] = 1
    s.hmax, s.vmax, s.mcux, s.mcuy = hmax, vmax, mcux, mcuy
    data = O.write(j, O.params(quality, 0, progressive))
    del j                                                   # borrowed coefficient arrays: nothing for the oracle to free
    if mcu_blocks(factors) > 10 or fractional(factors):
        assert libjpeg_refuses(data), f"libjpeg-turbo decoded {factors}, which the tests take as illegal"
    else:
        ref = libjpeg_native(data)
        got = O.Jpeg(data).decode_native()
        assert ref.shape == got.shape and np.array_equal(ref, got), f"oracle decode differs from libjpeg-turbo at {factors} {w}x{h} prog={progressive}"
    return data
