"""Trellis quantisation on the device (b200_set_jpeg_trellis), run with -m gpu on an H100: every lossy JPEG leg, with the switch on,
answers the oracle's trellis file (oracle/jpeg_trellis.py) byte for byte; switching it off again answers exactly what a
process that never switched it on does."""
import os
import sys

import numpy as np
import pytest

from oracle import jpeg_trellis as T
from pngutil import pil_png, synth
from webputil import pil_decode

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools.synth import synth_jpeg  # noqa: E402

pytestmark = pytest.mark.gpu

FMT_JPEG = 0
INPUTS = ["in_420_base_355x237.jpg", "in_420_prog_355x237.jpg", "in_444_base_355x237.jpg", "in_422_base_355x237.jpg",
          "in_gray_base_355x237.jpg", "in_420_base_640x480.jpg", "in_420_tiny_17x9.jpg", "in_420_tiny_3x3.jpg"]
CASES = [(80, 420, True), (80, 420, False), (80, 444, True), (80, 422, False), (60, 0, True), (95, 420, True), (30, 444, False)]


def _params(L, q, ss, prog, w=0, h=0):
    p = L.default_params()
    p.jpeg_quality, p.jpeg_chroma_subsampling, p.jpeg_progressive, p.width, p.height = q, ss, int(prog), w, h
    return p


def _sample(name):
    with open(os.path.join(ROOT, "tests", "golden", "reference_samples", name), "rb") as f:
        return f.read()


def planar(img):
    return np.ascontiguousarray(np.asarray(img).transpose(2, 0, 1))


@pytest.fixture
def trellis(L):
    assert L.lib().b200_init(0) == 0
    assert L.set_jpeg_trellis(1) == 0
    yield
    assert L.set_jpeg_trellis(0) == 0


@pytest.mark.parametrize("name", INPUTS)
@pytest.mark.parametrize("q,ss,prog", CASES)
def test_file_matches_trellis_oracle(L, O, golden, trellis, name, q, ss, prog):
    data = golden(name)
    got = L.compress_in_memory(data, _params(L, q, ss, prog))
    assert got == T.jpeg_lossy(data, O.params(q, ss, prog))


@pytest.mark.parametrize("name", ["j0.JPG", "j1.jpg"])
def test_reference_samples_match_trellis_oracle(L, O, trellis, name):
    data = _sample(name)
    for q, prog in ((80, True), (60, False)):
        got = L.compress_in_memory(data, _params(L, q, 0, prog))
        assert got == T.jpeg_lossy(data, O.params(q, 0, prog))
        assert got != O.jpeg_lossy(data, O.params(q, 0, prog))


@pytest.mark.parametrize("name", ["in_420_base_355x237.jpg", "in_444_base_355x237.jpg", "in_gray_base_355x237.jpg", "in_420_tiny_17x9.jpg"])
@pytest.mark.parametrize("w,h", [(100, 0), (40, 30), (355, 237)])
def test_resized_file_matches_trellis_oracle(L, O, golden, trellis, name, w, h):
    data = golden(name)
    for q, ss, prog in ((80, 420, True), (60, 444, False)):
        got = L.compress_in_memory(data, _params(L, q, ss, prog, w, h))
        assert got == T.jpeg_lossy_resized(data, O.params(q, ss, prog), w, h)


@pytest.mark.parametrize("q,ss,prog", [(80, 0, True), (90, 444, False), (60, 422, True)])
def test_png_to_jpeg_matches_trellis_oracle(L, O, trellis, q, ss, prog):
    rgb = synth(93, 141, 3, seed=q)
    p = _params(L, q, ss, prog)
    op = O.params(q, ss, prog)
    assert L.convert_in_memory(pil_png(rgb), p, FMT_JPEG) == O.write(T.forward(O.rgb_to_ycc(planar(rgb)), op), op)
    grey = synth(50, 70, 1, seed=q)
    assert L.convert_in_memory(pil_png(grey), p, FMT_JPEG) == O.write(T.forward(planar(grey), op), op)
    p.width = 64
    nw, nh = O.compute_dimensions(141, 93, 64, 0)
    rz = np.stack([O.resize_plane(np.ascontiguousarray(rgb[:, :, c]), nw, nh) for c in range(3)])
    assert L.convert_in_memory(pil_png(rgb), p, FMT_JPEG) == O.write(T.forward(O.rgb_to_ycc(rz), op), op)


def test_webp_to_jpeg_matches_trellis_oracle(L, O, trellis):
    data = _sample("w0.webp")
    op = O.params(80, 420, True)
    assert L.convert_in_memory(data, _params(L, 80, 420, True), FMT_JPEG) == O.write(T.forward(O.rgb_to_ycc(planar(pil_decode(data))), op), op)


def test_batch_megabatches_match_trellis_oracle(L, O, golden, trellis):
    same = [synth_jpeg(320, 240, i) for i in range(10)]            # same-shaped baseline files: megabatches on the device decoder
    mixed = [golden(n) for n in INPUTS]
    for prog in (True, False):
        p, op = _params(L, 75, 420, prog), O.params(75, 420, prog)
        datas = same + mixed
        for d, (out, code, msg) in zip(datas, L.compress_batch(datas, p, n_threads=4)):
            assert code == 0, msg
            assert out == T.jpeg_lossy(d, op)


def test_resident_pipe_matches_trellis_oracle(L, O, trellis):
    datas = [synth_jpeg(256, 160, i) for i in range(9)]
    p = _params(L, 80, 420, True)
    pipe = L.JpegPipe(datas, p, group=4)
    try:
        pipe.run()
        sizes, bad, _ = pipe.finish()
        assert bad == 0
        for i, d in enumerate(datas):
            assert pipe.fetch(i) == T.jpeg_lossy(d, O.params(80, 420, True))
        times = pipe.kernel_times(iters=1)
        assert "k_jpeg_trellis" in times
    finally:
        pipe.close()


def _oracle_to_size(O, data, ss, prog, max_size):
    """libcaesium's quality bisection restated around the oracle's trellis encoder (one full encode per try)."""
    tol = max_size // 50
    lo, hi, q = 1, 100, 80
    best = best_q = None
    for _ in range(10):
        if lo > hi:
            break
        cur = T.jpeg_lossy(data, O.params(q, ss, prog))
        if len(cur) <= max_size:
            if best is None or len(cur) > len(best):
                best, best_q = cur, q
            if max_size - len(cur) <= tol:
                break
            lo = q + 1
        else:
            hi = q - 1
        q = (lo + hi) // 2
    return best, best_q


@pytest.mark.parametrize("name,ss,prog", [("in_420_base_640x480.jpg", 420, True), ("in_444_base_355x237.jpg", 0, False)])
def test_compress_to_size_matches_trellis_bisection(L, O, golden, trellis, name, ss, prog):
    data = golden(name)
    for frac in (0.35, 0.6):
        target = int(len(data) * frac)
        want, want_q = _oracle_to_size(O, data, ss, prog, target)
        assert want is not None
        p = _params(L, 80, ss, prog)
        assert L.compress_to_size_in_memory(data, p, target) == want
        assert p.jpeg_quality == want_q


def test_switching_off_recaptures(L, O, golden):
    """Graphs captured with the pass must not be replayed without it: off -> on -> off gives the never-switched bytes."""
    assert L.lib().b200_init(0) == 0
    datas = [synth_jpeg(320, 240, i) for i in range(6)]
    single = golden("in_420_base_640x480.jpg")
    p = _params(L, 80, 420, True)

    def run():
        batch = [out for out, code, msg in L.compress_batch(datas, p, n_threads=1)]
        pipe = L.JpegPipe(datas, p, group=3)
        try:
            pipe.run(); pipe.finish()
            piped = [pipe.fetch(i) for i in range(len(datas))]
        finally:
            pipe.close()
        return batch, piped, L.compress_in_memory(single, p)

    assert L.set_jpeg_trellis(0) == 0
    never = run()
    assert L.set_jpeg_trellis(1) == 0
    try:
        on = run()
    finally:
        assert L.set_jpeg_trellis(0) == 0
    off = run()
    assert off == never
    assert never[0] == [O.jpeg_lossy(d, O.params(80, 420, True)) for d in datas]
    assert on[0] == on[1] == [T.jpeg_lossy(d, O.params(80, 420, True)) for d in datas]
    assert on[2] == T.jpeg_lossy(single, O.params(80, 420, True))
    assert never[2] == O.jpeg_lossy(single, O.params(80, 420, True))


def test_switch_refuses_other_values(L):
    assert L.set_jpeg_trellis(2) == 1          # B200_ERR_INVALID_ARGUMENT
    assert L.set_jpeg_trellis(-1) == 1
