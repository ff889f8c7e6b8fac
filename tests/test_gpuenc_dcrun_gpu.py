"""The DC-first scan of progressive colour output, coded in MCU runs from the compact DC array (k_geb_dc_first), run with -m gpu on an
H100: at every colour sampling geometry, at sizes of several 128-MCU runs whose MCU count is not a multiple of 128, with DC
differences of every category (tests/wild_dc.py) and with Pillow-style content, lossy and --lossless, through single calls,
megabatches and the resident pipe, every output file equals the oracle.  Sequential output, which keeps the per-unit path, and
grey output, which has no interleaved scan, are checked alongside."""
import pytest

import jpeg_geometry as G
import wild_dc as W

pytestmark = pytest.mark.gpu

COLOUR = [name for name, f in G.GEOMETRIES.items() if len(f) > 1]
# (q, output sampling, progressive, lossless); 0 keeps the input's sampling
ARMS = [(80, 420, True, False), (80, 0, True, False), (80, 0, True, True), (80, 0, False, True), (60, 444, False, False)]


def _size(f):
    """A size of 3 to 4 rows of 128 MCUs plus a partial MCU at the right and bottom edges."""
    hmax, vmax = max(h for h, _ in f), max(v for _, v in f)
    return 8 * hmax * 117 + 5, 8 * vmax * 3 + 3


def _params(L, q, ss, prog, lossless):
    p = L.default_params()
    p.jpeg_quality, p.jpeg_chroma_subsampling, p.jpeg_progressive, p.jpeg_optimize = q, ss, int(prog), int(lossless)
    return p


def _oracle(O, data, q, ss, prog, lossless):
    return O.jpeg_lossless(data, O.params(q, ss, prog)) if lossless else O.jpeg_lossy(data, O.params(q, ss, prog))


def _members(name):
    f = G.GEOMETRIES[name]
    w, h = _size(f)
    return [W.wild_jpeg(w, h, f, "wild", 1), G.make_jpeg(w, h, f, False), W.wild_jpeg(w, h, f, "wild", 2)]


@pytest.mark.parametrize("name", COLOUR)
def test_single_calls_and_megabatch(L, O, name):
    datas = _members(name)
    for q, ss, prog, lossless in ARMS:
        p = _params(L, q, ss, prog, lossless)
        want = [_oracle(O, d, q, ss, prog, lossless) for d in datas]
        for d, wd in zip(datas, want):
            assert L.compress_in_memory(d, p) == wd, (q, ss, prog, lossless)
        for k, (out, code, msg) in enumerate(L.compress_batch(datas, p, n_threads=1)):
            assert code == 0, msg
            assert out == want[k], (k, q, ss, prog, lossless)


@pytest.mark.parametrize("lossless", [False, True])
@pytest.mark.parametrize("name", ["s420", "y42", "c21", "cr22"])
def test_resident_pipe(L, O, name, lossless):
    import torch
    assert L.lib().b200_init_device(0) == 0
    datas = _members(name)
    q, ss, prog = 80, 0 if lossless else 420, True
    want = [_oracle(O, d, q, ss, prog, lossless) for d in datas]
    pipe = L.JpegPipe(datas, _params(L, q, ss, prog, lossless), group=2)
    st = torch.cuda.Stream()
    try:
        for _ in range(2):
            pipe.run(st.cuda_stream)
            torch.cuda.synchronize()
            sizes, not_settled, retries = pipe.finish()
            assert not_settled == 0
            for i in range(len(datas)):
                assert pipe.fetch(i) == want[i], i
    finally:
        pipe.close()


def test_grey_progressive(L, O):
    f = G.GEOMETRIES["grey22"]
    d = W.wild_jpeg(*_size(f), f, "wild", 3)
    for lossless in (False, True):
        p = _params(L, 80, 0, True, lossless)
        assert L.compress_in_memory(d, p) == _oracle(O, d, 80, 0, True, lossless), lossless
