"""Every device leg at its format's dimension limit, and the Lanczos3 resampler (K3) at extreme ratios, run with -m gpu on an H100.

- JPEG sides of exactly 65500 (libjpeg's JPEG_MAX_DIMENSION) through the lossy, lossless, trellis and megabatch legs: the oracle's
  bytes, decoded by libjpeg-turbo (Pillow) to the oracle's decode.  JPEG targets over 65500 answer 1; PNG targets keep 65535.
- WebP frames 16383 wide or tall (VP8's 14-bit size fields) through K8 and the lossless leg, against the twins and libwebp.
- K3 against a float64 Lanczos3 written here in numpy / scipy (no code shared with the twin), with an a-priori bound on the f32
  error of the device's two passes, at 65500 taps in one window, 1-pixel sources stretched across a whole axis, near-unit
  ratios, one axis kept, and widths around the kernels' 128 / 256-thread launch tiles.
All fixtures are made here."""
import functools
import io
import zlib

import numpy as np
import pytest
import scipy.sparse as sp
from PIL import Image, ImageFile

import jpeg_geometry as G
from oracle import jpeg_trellis as T
from oracle import png_resize as R
from pngutil import frame_png, pil_png, synth
from webputil import pil_decode

pytestmark = pytest.mark.gpu

JPEG_MAX, PNG_MAX, WEBP_MAX = 65500, 65535, 16383
FMT_JPEG, FMT_PNG, FMT_WEBP = 0, 1, 3
LIBJPEG_TOO_BIG = "Maximum supported image dimension is 65500 pixels"


def planar(img):
    return np.ascontiguousarray(np.asarray(img).transpose(2, 0, 1))


def _params(L, q=80, ss=420, prog=True, w=0, h=0, **kw):
    p = L.default_params()
    p.jpeg_quality, p.jpeg_chroma_subsampling, p.jpeg_progressive, p.width, p.height = q, ss, int(prog), w, h
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def _refused(L, call):
    with pytest.raises(L.B200Error) as e:
        call()
    return e.value.code, str(e.value)


# ---- JPEG sources at 65500 -------------------------------------------------------------------------------------------------
SUBSAMPLING = {"420": 2, "422": 1, "444": 0, "grey": None}         # Pillow's subsampling argument; None = one grey component
LONG_SHAPES = [(JPEG_MAX, 1), (JPEG_MAX, 8), (JPEG_MAX, 17), (1, JPEG_MAX), (8, JPEG_MAX), (17, JPEG_MAX)]


@functools.lru_cache(maxsize=None)
def jpeg_source(w, h, geo, progressive, seed=0):
    """a libjpeg-turbo (Pillow) file of w x h: smooth colour ramps with noise, so that every block carries AC coefficients"""
    rng = np.random.default_rng(seed * 1000 + w + 3 * h + 7 * progressive)
    pos = np.add.outer(np.arange(h), np.arange(w)).astype(np.float64)
    img = np.stack([128 + 90 * np.sin(pos / (29.0 + 11 * c) + seed) for c in range(3)], -1) + rng.normal(0, 12, (h, w, 3))
    img = np.clip(np.rint(img), 0, 255).astype(np.uint8)
    b = io.BytesIO()
    block = ImageFile.MAXBLOCK          # Pillow writes a progressive file into one buffer of about w * h bytes: too few for 1 x 65500
    ImageFile.MAXBLOCK = max(block, 8 * w * h)
    try:
        if SUBSAMPLING[geo] is None:
            Image.fromarray(img[:, :, 1]).save(b, "JPEG", quality=90, progressive=progressive)
        else:
            Image.fromarray(img).save(b, "JPEG", quality=90, subsampling=SUBSAMPLING[geo], progressive=progressive)
    finally:
        ImageFile.MAXBLOCK = block
    return b.getvalue()


def patch_sof(data, w=None, h=None):
    """the same file with its frame header's width and / or height rewritten"""
    d, i = bytearray(data), 2
    while i + 4 <= len(d):
        m, n = d[i + 1], d[i + 2] << 8 | d[i + 3]
        if m in (0xC0, 0xC1, 0xC2):
            if h is not None:
                d[i + 5:i + 7] = h.to_bytes(2, "big")
            if w is not None:
                d[i + 7:i + 9] = w.to_bytes(2, "big")
            return bytes(d)
        i += 2 + n
    raise AssertionError("no SOF")


def decodes_to_the_oracle(O, out):
    """libjpeg-turbo reads the file, and its decode is the oracle's"""
    assert np.array_equal(G.libjpeg_native(out), O.Jpeg(out).decode_native())


@pytest.mark.parametrize("geo", list(SUBSAMPLING))
@pytest.mark.parametrize("w,h", LONG_SHAPES, ids=[f"{w}x{h}" for w, h in LONG_SHAPES])
def test_jpeg_at_the_limit_matches_the_oracle(L, O, w, h, geo):
    for prog in (False, True):
        data = jpeg_source(w, h, geo, prog)
        for q, ss, oprog in ((80, 420, True), (60, 444, False)):
            out = L.compress_in_memory(data, _params(L, q, ss, oprog))
            assert out == O.jpeg_lossy(data, O.params(q, ss, oprog)), (prog, q, ss, oprog)
            decodes_to_the_oracle(O, out)
        out = L.compress_in_memory(data, _params(L, 80, 0, True, jpeg_optimize=1))
        assert out == O.jpeg_lossless(data, O.params(80, 0, True)), prog
        decodes_to_the_oracle(O, out)


@pytest.mark.parametrize("geo", ["420", "grey"])
def test_jpeg_trellis_at_the_limit(L, O, geo):
    assert L.set_jpeg_trellis(1) == 0
    try:
        for w, h in ((JPEG_MAX, 17), (17, JPEG_MAX), (JPEG_MAX, 1)):
            data = jpeg_source(w, h, geo, False)
            out = L.compress_in_memory(data, _params(L, 80, 420, True))
            assert out == T.jpeg_lossy(data, O.params(80, 420, True)), (w, h)
            decodes_to_the_oracle(O, out)
    finally:
        assert L.set_jpeg_trellis(0) == 0


@pytest.mark.parametrize("geo", list(SUBSAMPLING))
def test_jpeg_megabatch_at_the_limit(L, O, geo):
    """same-shaped baseline files form one megabatch on the device decoder; each answer is the oracle's single-file answer"""
    for w, h in ((JPEG_MAX, 8), (8, JPEG_MAX), (JPEG_MAX, 17)):
        datas = [jpeg_source(w, h, geo, False, seed=s) for s in range(3)]
        for q, ss, prog, opt in ((80, 420, True, 0), (60, 444, False, 0), (80, 0, True, 1)):
            want = O.jpeg_lossless if opt else O.jpeg_lossy
            res = L.compress_batch(datas, _params(L, q, ss, prog, jpeg_optimize=opt), n_threads=3)
            for i, (d, (out, code, msg)) in enumerate(zip(datas, res)):
                assert code == 0, msg
                assert out == want(d, O.params(q, ss, prog)), (w, h, i, q, ss, prog, opt)


def test_jpeg_sources_over_the_limit_everywhere(L, O):
    """the refusal reaches the device entry points too: single calls, conversions, the megabatch and the resident pipe"""
    good = jpeg_source(JPEG_MAX, 8, "420", False)
    for side in (JPEG_MAX + 1, PNG_MAX):
        for bad in (patch_sof(good, w=side), patch_sof(jpeg_source(8, JPEG_MAX, "grey", False), h=side)):
            calls = [lambda: L.compress_in_memory(bad, _params(L)), lambda: L.compress_in_memory(bad, _params(L, jpeg_optimize=1)),
                     lambda: L.compress_in_memory(bad, _params(L, w=100)), lambda: L.convert_in_memory(bad, _params(L, png_optimize=1), FMT_PNG),
                     lambda: L.convert_in_memory(bad, _params(L), FMT_WEBP), lambda: L.compress_to_size_in_memory(bad, _params(L), 4000)]
            for call in calls:
                code, msg = _refused(L, call)
                assert code == L.ERR_CORRUPT_INPUT and LIBJPEG_TOO_BIG in msg, msg
            with pytest.raises(L.B200Error, match=LIBJPEG_TOO_BIG):
                L.JpegPipe([bad, bad], _params(L))
    bad = patch_sof(good, w=JPEG_MAX + 1)
    datas = [good, bad, jpeg_source(JPEG_MAX, 8, "420", False, seed=1), bad, good]
    for p in (_params(L), _params(L, jpeg_optimize=1)):
        singles = {id(d): L.compress_in_memory(d, p) for d in (datas[0], datas[2])}
        for d, (out, code, msg) in zip(datas, L.compress_batch(datas, p, n_threads=2)):
            if d is bad:
                assert code == L.ERR_CORRUPT_INPUT and LIBJPEG_TOO_BIG in msg, msg
            else:
                assert code == 0 and out == singles[id(d)], msg


# ---- JPEG targets at the limit ---------------------------------------------------------------------------------------------
def test_jpeg_resize_target_at_the_limit(L, O):
    for geo in ("420", "grey"):
        small = jpeg_source(40, 8, geo, False)
        for tw, th in ((JPEG_MAX, 8), (8, JPEG_MAX)):
            for q, ss, prog in ((80, 420, True), (60, 444, False)):
                out = L.compress_in_memory(small, _params(L, q, ss, prog, tw, th))
                assert out == O.jpeg_lossy_resized(small, O.params(q, ss, prog), tw, th), (geo, tw, th, q)
                decodes_to_the_oracle(O, out)
        for tw, th in ((JPEG_MAX + 1, 8), (8, JPEG_MAX + 1), (PNG_MAX, 8)):
            for call in (lambda: L.compress_in_memory(small, _params(L, 80, 420, True, tw, th)),
                         lambda: L.compress_to_size_in_memory(small, _params(L, 80, 420, True, tw, th), len(small) - 1)):
                code, msg = _refused(L, call)
                assert code == L.ERR_INVALID_ARGUMENT and "invalid target dimensions" in msg, (tw, th, msg)
            with pytest.raises(O.OracleError, match="invalid target dimensions"):
                O.jpeg_lossy_resized(small, O.params(80, 420, True), tw, th)


def test_png_and_webp_to_jpeg_at_the_limit(L, O):
    op = O.params(80, 420, True)
    for w, h in ((JPEG_MAX, 8), (3, JPEG_MAX)):
        rgb = synth(h, w, 3, seed=w)
        out = L.convert_in_memory(pil_png(rgb, compress_level=1), _params(L), FMT_JPEG)
        assert out == O.write(O.forward(O.rgb_to_ycc(planar(rgb)), op), op), (w, h)
        decodes_to_the_oracle(O, out)
    grey = synth(JPEG_MAX + 1, 2, 1, seed=2)
    for src in (pil_png(synth(8, JPEG_MAX + 1, 3, seed=1), compress_level=1), pil_png(grey, compress_level=1)):
        code, msg = _refused(L, lambda: L.convert_in_memory(src, _params(L), FMT_JPEG))
        assert code == L.ERR_INVALID_ARGUMENT and "invalid target dimensions" in msg, msg
    small_png = pil_png(synth(8, 40, 3, seed=3))
    b = io.BytesIO()
    Image.fromarray(synth(8, 40, 3, seed=4)).save(b, "WEBP", quality=90)
    for src in (small_png, b.getvalue()):
        out = L.convert_in_memory(src, _params(L, w=JPEG_MAX, h=8), FMT_JPEG)
        assert Image.open(io.BytesIO(out)).size == (JPEG_MAX, 8)
        decodes_to_the_oracle(O, out)
        code, msg = _refused(L, lambda: L.convert_in_memory(src, _params(L, w=JPEG_MAX + 1, h=8), FMT_JPEG))
        assert code == L.ERR_INVALID_ARGUMENT and "invalid target dimensions" in msg, msg


def test_png_targets_keep_65535(L, O):
    assert L.set_png_resize(True) == 0
    try:
        rgb = synth(3, 40, 3, seed=5)
        raw = rgb.reshape(3, -1)
        src = pil_png(rgb)
        for tw, th in ((PNG_MAX, 3), (40, PNG_MAX)):
            info, rows = L.png_resize_samples(src, tw, th)
            want, wrows = R.png_resize(raw, 40, 3, 8, 2, b"", b"", tw, th)
            assert (info.width, info.height) == (want["width"], want["height"]) == (tw, th)
            assert np.array_equal(rows, wrows)
            out = L.compress_in_memory(src, _params(L, w=tw, h=th, png_optimize=1, png_optimization_level=1))
            got = np.asarray(Image.open(io.BytesIO(out)).convert("RGB"))
            assert np.array_equal(got.reshape(th, -1), wrows)
        code, msg = _refused(L, lambda: L.compress_in_memory(src, _params(L, w=PNG_MAX + 1, h=3, png_optimize=1)))
        assert code == L.ERR_INVALID_ARGUMENT, msg
    finally:
        L.set_png_resize(False)


def test_batch_neighbours_of_refused_targets(L, O):
    """a batch with a 65500-wide target: the JPEGs are resized, a source over the limit answers 4; at 65501 every JPEG answers 1"""
    small = [jpeg_source(40, 8, "420", False, seed=s) for s in range(2)] + [jpeg_source(40, 8, "grey", False)]
    bad = patch_sof(jpeg_source(JPEG_MAX, 8, "420", False), w=JPEG_MAX + 1)
    datas = [small[0], bad, small[1], small[2], bad]
    p = _params(L, 80, 420, True, JPEG_MAX, 8)
    singles = [L.compress_in_memory(d, p) if d is not bad else None for d in datas]
    for d, single, (out, code, msg) in zip(datas, singles, L.compress_batch(datas, p, n_threads=3)):
        if d is bad:
            assert code == L.ERR_CORRUPT_INPUT, msg
        else:
            assert code == 0 and out == single == O.jpeg_lossy_resized(d, O.params(80, 420, True), JPEG_MAX, 8), msg
    p = _params(L, 80, 420, True, JPEG_MAX + 1, 8)
    for d, (out, code, msg) in zip(datas, L.compress_batch(datas, p, n_threads=3)):
        assert code == (L.ERR_CORRUPT_INPUT if d is bad else L.ERR_INVALID_ARGUMENT), msg


# ---- WebP at 16383 ---------------------------------------------------------------------------------------------------------
WEBP_SHAPES = [(WEBP_MAX, 1), (1, WEBP_MAX), (WEBP_MAX, 16), (16, WEBP_MAX), (WEBP_MAX, 17)]


@pytest.mark.parametrize("w,h", WEBP_SHAPES, ids=[f"{w}x{h}" for w, h in WEBP_SHAPES])
def test_k8_at_the_limit(L, O, w, h):
    img = planar(synth(h, w, 3, seed=w + h, kind="photo"))
    data, levels, modes = L.webp_encode_rgb(img, 80, want_stage=True)
    wl, wm = O.webp_analyze(img, 80)
    assert np.array_equal(levels, wl) and np.array_equal(modes, wm)
    assert data == O.webp_encode(img, 80)[0]
    dec = pil_decode(data)
    assert dec.shape == (h, w, 3)
    assert np.abs(dec.astype(int) - img.transpose(1, 2, 0).astype(int)).mean() < 4.0        # test_k8_many_rows_wavefront's bound


def test_jpeg_to_webp_target_at_the_limit(L, O):
    small = jpeg_source(40, 8, "420", False)
    ycc = O.Jpeg(small).decode_native()
    rgb = O.ycc_to_rgb(ycc)
    for tw, th in ((WEBP_MAX, 8), (8, WEBP_MAX)):
        out = L.convert_in_memory(small, _params(L, w=tw, h=th), FMT_WEBP)
        rz = np.stack([O.resize_plane(rgb[c], tw, th) for c in range(3)])
        assert out == O.webp_encode(rz, L.default_params().webp_quality)[0]
        assert pil_decode(out).shape == (th, tw, 3)
        code, msg = _refused(L, lambda: L.convert_in_memory(small, _params(L, w=tw + (tw == WEBP_MAX), h=th + (th == WEBP_MAX)), FMT_WEBP))
        assert code == L.ERR_INVALID_ARGUMENT and "invalid target dimensions" in msg, msg


def test_lossless_webp_at_the_limit(L):
    from oracle import vp8l
    for h, kind in ((4, "photo"), (3, "flat")):
        b = io.BytesIO()
        Image.fromarray(synth(h, WEBP_MAX, 3, seed=h, kind=kind)).save(b, "WEBP", lossless=True, method=0)
        rgb, a = L.webp_decode_rgba(b.getvalue())
        px = np.ascontiguousarray(np.concatenate([rgb, np.full(rgb.shape[:2] + (1,), 255, np.uint8) if a is None else a[:, :, None]], 2))
        out = L.compress_in_memory(b.getvalue(), _params(L, webp_lossless=1))
        assert out == vp8l.webp_lossless_encode(px)
        assert np.array_equal(np.asarray(Image.open(io.BytesIO(out)).convert("RGBA")), px)


# ---- K3 against float64 ----------------------------------------------------------------------------------------------------
U = 2.0 ** -24                  # unit roundoff of f32


def gamma(n):
    return n * U / (1 - n * U)


@functools.lru_cache(maxsize=None)
def axis_matrix(n_in, n_out):
    """one axis of image 0.25.9's Lanczos3 (imageops/sample.rs) as a sparse [n_out, n_in] matrix.  The crate places the window and
    the tap positions in f32 (left = floor(c - 3s), right = ceil(c + 3s), both clamped; s = max(ratio, 1)): so does this, since
    those positions are part of the algorithm.  The weights sinc(x) sinc(x / 3) and their normalisation are float64.
    -> (weights, the same pattern with ones, taps per output)"""
    f = np.float32
    ratio = f(n_in) / f(n_out)
    sratio = max(ratio, f(1))
    support = f(3) * sratio
    c = (np.arange(n_out, dtype=np.float32) + f(0.5)) * ratio
    left = np.clip(np.floor(c - support).astype(np.int64), 0, n_in - 1)
    right = np.minimum(np.maximum(np.ceil(c + support).astype(np.int64), left + 1), n_in)
    taps = right - left
    rows = np.repeat(np.arange(n_out), taps)
    cols = left[rows] + np.arange(rows.size) - np.repeat(np.cumsum(taps) - taps, taps)
    x = (cols.astype(np.float32) - (c - f(0.5))[rows]).astype(np.float64) / float(sratio)
    k = np.where(np.abs(x) < 3, np.sinc(x) * np.sinc(x / 3), 0.0)
    vals = k / np.bincount(rows, weights=k, minlength=n_out)[rows]
    W = sp.csr_matrix((vals, (rows, cols)), shape=(n_out, n_in))
    ones = sp.csr_matrix((np.ones_like(vals), (rows, cols)), shape=(n_out, n_in))
    return W, ones, taps


def pass_bound(W, ones, taps, a, prev):
    """a-priori bound on |f32 pass - exact pass| for every output of one pass over inputs of magnitude <= a that are themselves
    within prev of their exact values.  Recursive summation of the n products: gamma_n * sum|w x|; the f32 weights were divided
    by an f32 sum of n terms: another gamma_n * sum|w x|; each f32 kernel value (sinf, products, quotient) is off by at most
    8u * max|w|; the inputs' own error goes through sum|w|."""
    Wa = abs(W)
    mx = Wa.max(axis=1).toarray().ravel()
    g = gamma(taps)[:, None]
    return 2 * g * (Wa @ a) + 8 * U * mx[:, None] * (ones @ a) + (Wa @ prev if prev is not None else 0)


def lanczos_f64(plane, nw, nh):
    """-> (exact value t, bound b, most taps in a window) of every output sample: vertical pass, then horizontal"""
    h, w = plane.shape
    X = plane.astype(np.float64)
    Wv, Pv, nv = axis_matrix(h, nh)
    Wh, Ph, nh_taps = axis_matrix(w, nw)
    t1 = Wv @ X
    b1 = pass_bound(Wv, Pv, nv, np.abs(X), None)
    t = (Wh @ t1.T).T
    b = pass_bound(Wh, Ph, nh_taps, (np.abs(t1) + b1).T, b1.T).T
    return t, b, max(nv.max(), nh_taps.max())


def round_half_away(v):
    return np.floor(v + 0.5)            # v >= 0 here: clamped first


def check_against_f64(got, plane, nw, nh, top, what):
    t, b, taps = lanczos_f64(plane, nw, nh)
    lo = round_half_away(np.clip(t - b, 0, top))
    hi = round_half_away(np.clip(t + b, 0, top))
    g = got.astype(np.float64)
    bad = (g < lo) | (g > hi)
    assert not bad.any(), (what, int(bad.sum()), float(np.abs(g - t)[bad].max()), float(b[bad].max()))
    if taps <= 64:                      # a bias inside the bound still moves the rounding of many samples
        exact = (g == round_half_away(np.clip(t, 0, top))).mean()
        assert exact >= 0.99, (what, exact)


def k3_plane(h, w, top, seed):
    """full-range noise with columns and rows pinned at 0 and the maximum: the lobes overshoot both ends of the range"""
    rng = np.random.default_rng(seed)
    p = rng.integers(0, top + 1, (h, w)).astype(np.int64)
    p[:, 1::5] = top
    p[:, 3::5] = 0
    if h > 4:
        p[2::7] = top
    return p


# (source w, h) -> (target w, h)
K3_SHAPES = [((JPEG_MAX, 2), (1, 1)), ((2, JPEG_MAX), (1, 1)), ((1, 1), (JPEG_MAX, 1)), ((1, 1), (1, JPEG_MAX)),
             ((WEBP_MAX, 5), (3, 2)), ((1000, 40), (999, 39)), ((999, 39), (1000, 40)), ((300, 40), (300, 17)), ((300, 40), (123, 40)),
             ((127, 9), (257, 5)), ((128, 9), (129, 5)), ((129, 9), (128, 5)), ((255, 9), (256, 5)), ((256, 9), (255, 5)), ((257, 9), (127, 5))]
K3_IDS = [f"{a}x{b}_to_{c}x{d}" for (a, b), (c, d) in K3_SHAPES]


def _png_rgb(planes, depth):
    inter = np.moveaxis(planes, 0, -1)
    inter = inter.astype(">u2" if depth == 16 else np.uint8)
    h, w = planes.shape[1:]
    raw = np.ascontiguousarray(inter).view(np.uint8).reshape(h, -1)
    z = zlib.compress(np.concatenate([np.zeros((h, 1), np.uint8), raw], 1).tobytes(), 1)
    return frame_png(w, h, depth, 2, z), raw


@pytest.mark.parametrize("depth", [8, 16])
@pytest.mark.parametrize("src,dst", K3_SHAPES, ids=K3_IDS)
def test_k3_png_samples_against_float64(L, O, src, dst, depth):
    (w, h), (nw, nh) = src, dst
    top = 65535 if depth == 16 else 255
    planes = np.stack([k3_plane(h, w, top, seed=w * 3 + h + c) for c in range(3)])
    png, raw = _png_rgb(planes, depth)
    info, rows = L.png_resize_samples(png, nw, nh)
    assert (info.width, info.height, info.bit_depth) == (nw, nh, depth)
    _, wrows = R.png_resize(raw, w, h, depth, 2, b"", b"", nw, nh)
    assert np.array_equal(rows, wrows)                                  # the twin, byte for byte
    got = (rows.view(">u2") if depth == 16 else rows).reshape(nh, nw, 3)
    for c in range(3):
        check_against_f64(got[:, :, c], planes[c], nw, nh, top, (src, dst, depth, c))
    if (w, h) == (1, 1):                                                # one tap of weight 1: a copy of the pixel
        assert (got == planes[:, 0, 0]).all()


@pytest.mark.parametrize("src,dst", K3_SHAPES, ids=K3_IDS)
def test_k3_jpeg_to_png_against_float64(L, O, src, dst):
    """the same shapes on the RGB of a decoded JPEG (the convert leg's device decode feeding K3), read back from a lossless PNG"""
    (w, h), (nw, nh) = src, dst
    data = jpeg_source(w, h, "444", False, seed=9)
    rgb = O.ycc_to_rgb(O.Jpeg(data).decode_native())
    out = L.convert_in_memory(data, _params(L, w=nw, h=nh, png_optimize=1, png_optimization_level=1), FMT_PNG)
    got = planar(np.asarray(Image.open(io.BytesIO(out)).convert("RGB")))
    assert got.shape == (3, nh, nw)
    for c in range(3):
        assert np.array_equal(got[c], O.resize_plane(rgb[c], nw, nh)), c
        check_against_f64(got[c], rgb[c].astype(np.int64), nw, nh, 255, (src, dst, c))
