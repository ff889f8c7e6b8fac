"""The device JPEG path at every legal sampling geometry (tests/jpeg_geometry.py), run with -m gpu on an H100: decode planes against
libjpeg-turbo directly, lossy and lossless files against the oracle, and on a subset resize, WebP conversion, compress-to-size,
trellis and the megabatch.  These geometries drive the upsampler's h1v2 fancy branch (4:4:0) and its box branch (3x, 4x, vertical,
luma upsampled under 2x2 chroma), components of one image on different transform paths, and the device Huffman decoder's and
encoder's MCU walk over block layouts other than {2x2, 2x1, 1x1} + 1 + 1.  Over-sized MCUs answer 4 and fractional ratios 3."""
import numpy as np
import pytest

import jpeg_geometry as G
from oracle import jpeg_trellis as T
from test_jpeg_gpu import _oracle_to_size
from test_webp_gpu import _jpeg_rgb

pytestmark = pytest.mark.gpu

FMT_WEBP = 3
CASES = [(name, w, h) for name, f in G.GEOMETRIES.items() for (w, h) in G.sizes_for(f)]
SUBSET = ["y12", "c22", "y41", "y32", "c21", "cr22"]
OUT_CASES = [(ss, prog, q) for ss in (420, 422, 411, 444) for prog in (True, False) for q in (80, 35)]


def _params(L, q=80, ss=420, prog=True, w=0, h=0):
    p = L.default_params()
    p.jpeg_quality, p.jpeg_chroma_subsampling, p.jpeg_progressive, p.width, p.height = q, ss, int(prog), w, h
    return p


@pytest.mark.parametrize("name,w,h", CASES)
def test_decode_lossy_and_lossless_match(L, O, name, w, h):
    f = G.GEOMETRIES[name]
    for prog in (False, True):
        data = G.make_jpeg(w, h, f, prog)
        lay, co = L.jpeg_decode_coefficients(data)
        assert np.array_equal(L.jpeg_decode_planes(lay, co), G.libjpeg_native(data)), prog
        # a progressive source takes the host decoder into the same transform kernels: two output cases are enough there
        for ss, oprog, q in (OUT_CASES if not prog else OUT_CASES[::7]):
            out = L.compress_in_memory(data, _params(L, q, ss, oprog))
            assert out == O.jpeg_lossy(data, O.params(q, ss, oprog)), (prog, ss, oprog, q)
            assert np.array_equal(G.libjpeg_native(out), O.Jpeg(out).decode_native())
        for oprog in (True, False):         # device decoder -> device encoder, both in the input's geometry
            p = _params(L, 80, 0, oprog)
            p.jpeg_optimize = 1
            assert L.compress_in_memory(data, p) == O.jpeg_lossless(data, O.params(80, 0, oprog)), (prog, oprog)


@pytest.mark.parametrize("name", SUBSET)
def test_resize_and_webp_match(L, O, name):
    f = G.GEOMETRIES[name]
    for (w, h) in [(67, 45), (130, 61), (17, 9)]:
        data = G.make_jpeg(w, h, f, False, seed=3)
        for tw, th in [(40, 0), (0, 23), (w + 9, h + 4)]:
            for q, ss, prog in [(80, 420, True), (60, 444, False)]:
                assert L.compress_in_memory(data, _params(L, q, ss, prog, tw, th)) == O.jpeg_lossy_resized(data, O.params(q, ss, prog), tw, th), (w, h, tw, th)
        p = L.default_params()
        p.webp_quality = 80
        assert L.convert_in_memory(data, p, FMT_WEBP) == O.webp_encode(_jpeg_rgb(O, data), 80)[0], (w, h)
        p.width = 40
        nw, nh = O.compute_dimensions(w, h, 40, 0)
        assert L.convert_in_memory(data, p, FMT_WEBP) == O.webp_encode(_jpeg_rgb(O, data, nw, nh), 80)[0], (w, h)


@pytest.mark.parametrize("name", SUBSET)
def test_compress_to_size_matches_bisection(L, O, name):
    data = G.make_jpeg(130, 61, G.GEOMETRIES[name], False, seed=5)
    for frac in (0.7, 0.3):
        target = int(len(data) * frac)
        want, want_q = _oracle_to_size(O, data, 420, True, target)
        p = _params(L, 80, 420, True)
        assert L.compress_to_size_in_memory(data, p, target) == want, frac
        if want_q is not None:
            assert p.jpeg_quality == want_q


@pytest.mark.parametrize("name", SUBSET)
def test_trellis_matches_oracle(L, O, name):
    assert L.set_jpeg_trellis(1) == 0
    try:
        for (w, h) in [(67, 45), (130, 61)]:
            data = G.make_jpeg(w, h, G.GEOMETRIES[name], False, seed=7)
            for q, ss, prog in [(80, 420, True), (60, 444, False), (70, 411, True)]:
                assert L.compress_in_memory(data, _params(L, q, ss, prog)) == T.jpeg_lossy(data, O.params(q, ss, prog)), (w, h, q, ss)
    finally:
        assert L.set_jpeg_trellis(0) == 0


@pytest.mark.parametrize("name", SUBSET)
def test_megabatch_of_one_geometry(L, O, golden, name):
    """Nine same-geometry baseline files form one megabatch (slot_run_group, generic transform path); a golden 4:2:0 file rides along."""
    datas = [G.make_jpeg(130, 61, G.GEOMETRIES[name], False, seed=100 + i) for i in range(9)] + [golden("in_420_base_355x237.jpg")]
    for q, ss, prog, opt in [(80, 420, True, 0), (60, 444, False, 0), (80, 0, True, 1)]:
        p = _params(L, q, ss, prog)
        p.jpeg_optimize = opt
        want = O.jpeg_lossless if opt else O.jpeg_lossy
        for i, (d, (out, code, msg)) in enumerate(zip(datas, L.compress_batch(datas, p, n_threads=4))):
            assert code == 0, msg
            assert out == want(d, O.params(q, ss, prog)), (i, q, ss, prog, opt)


def test_oversized_mcu_answers_corrupt_input(L, O, golden):
    good = golden("in_420_base_355x237.jpg")
    p = _params(L)
    want = O.jpeg_lossy(good, O.params(80, 420, True))
    bad = [G.make_jpeg(67, 45, f, prog) for f in G.OVERSIZED.values() for prog in (False, True)]
    for d in bad:
        with pytest.raises(L.B200Error) as e:
            L.compress_in_memory(d, p)
        assert e.value.code == L.ERR_CORRUPT_INPUT, str(e.value)
        assert L.compress_in_memory(good, p) == want
    same = [G.make_jpeg(67, 45, G.OVERSIZED["y42_c21_12"], False, seed=s) for s in range(4)]
    datas = [good] + bad + same + [good, good]
    for d, (out, code, msg) in zip(datas, L.compress_batch(datas, p, n_threads=4)):
        if d is good:
            assert code == 0 and out == want, msg
        else:
            assert code == L.ERR_CORRUPT_INPUT, msg
    assert L.compress_in_memory(good, p) == want


def test_fractional_ratio_answers_unsupported_everywhere(L, O, golden):
    good = golden("in_420_base_355x237.jpg")
    frac = [G.make_jpeg(67, 45, G.FRACTIONAL, False, seed=s) for s in range(4)]
    d = frac[0]
    calls = [lambda: L.compress_in_memory(d, _params(L)),
             lambda: L.compress_in_memory(d, _params(L, 80, 420, True, 40, 0)),
             lambda: L.convert_in_memory(d, L.default_params(), FMT_WEBP),
             lambda: L.compress_to_size_in_memory(d, _params(L), len(d) // 2)]
    for call in calls:
        with pytest.raises(L.B200Error) as e:
            call()
        assert e.value.code == L.ERR_UNSUPPORTED, str(e.value)
    for p in (_params(L), _params(L, 80, 420, True, 40, 0)):
        datas = [good] + frac + [good]
        for x, (out, code, msg) in zip(datas, L.compress_batch(datas, p, n_threads=2)):
            assert code == (0 if x is good else L.ERR_UNSUPPORTED), msg
    p = _params(L, 80, 0, True)
    p.jpeg_optimize = 1                    # no upsampling in a coefficient transcode: still done, on the device
    assert L.compress_in_memory(d, p) == O.jpeg_lossless(d, O.params(80, 0, True))
