"""A slot's buffers grow while its captured launch sequences are replayed: one worker thread keeps reusing one slot, its CUDA
graphs and its coders through shapes that grow, shrink and grow again.  A graph that still pointed at a freed buffer would write
wrong bytes (or into memory the slot no longer owns), so every output must equal the single-image call's."""
import pytest

from pngutil import pil_png, synth

pytestmark = pytest.mark.gpu

SHAPES = [(64, 48), (640, 480), (64, 48), (2048, 1536)]


def _jpeg_params(L, optimize):
    p = L.default_params()
    p.jpeg_quality, p.jpeg_chroma_subsampling, p.jpeg_progressive, p.jpeg_optimize = 80, 420, 1, int(optimize)
    return p


@pytest.mark.parametrize("optimize", [False, True], ids=["lossy", "optimize"])
def test_jpeg_megabatches_through_growing_and_shrinking_shapes(L, O, optimize):
    from tools.synth import synth_jpeg
    p = _jpeg_params(L, optimize)
    for step, (w, h) in enumerate(SHAPES):
        datas = [synth_jpeg(w, h, 4 * step + i) for i in range(4)]
        res = L.compress_batch(datas, p, n_threads=1)
        for d, (out, code, msg) in zip(datas, res):
            assert code == 0, msg
            assert out == L.compress_in_memory(d, p), (w, h)
            if not optimize:
                assert out == O.jpeg_lossy(d, O.params(80, 420, True)), (w, h)


def test_lossy_png_small_large_small(L):
    assert L.set_png_lossy(True) == 0
    try:
        p = L.default_params()
        p.png_optimize, p.png_quality, p.png_optimization_level = 0, 70, 3
        for step, (h, w) in enumerate([(40, 56), (900, 1200), (40, 56)]):
            srcs = [pil_png(synth(h, w, 3, seed=10 * step + i)) for i in range(2)]
            res = L.compress_batch(srcs, p, n_threads=1)
            for s, (out, code, msg) in zip(srcs, res):
                assert code == 0, msg
                assert out == L.compress_in_memory(s, p), (h, w)
    finally:
        L.set_png_lossy(False)
