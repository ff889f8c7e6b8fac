"""GPU tests of the device encoder's byte stuffing (k_ge_ffcount / k_ge_layout / k_ge_scatter in jpeg_gpuenc.cu), run with -m gpu on
an H100: the device-encoded file is byte-identical to the host encoder on coefficient sets dense in 0xFF bytes (long runs of one
bits from large magnitudes), at sizes that put scans below one 16-byte group, inside one tile and across many tiles and chunks; in
8-image megabatches of different contents through b200_compress_batch; and on a re-encode that outgrows the output estimate, so
that the encoder repeats its back half with exact sizes, followed by a second run through the same buffers."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

BIG = [1023, 1023, 1023, 511, 255, -1023, -511]     # value bits all ones (1023, 511, 255) or all zeros with a one-bit sign


def _layout(L, w, h, ncomp=1):
    lay = L.JpegLayout()
    lay.width, lay.height, lay.ncomp = w, h, ncomp
    off = 0
    for c in range(ncomp):
        lay.hs[c] = lay.vs[c] = 1
        lay.bw[c] = lay.rbw[c] = -(-w // 8)
        lay.bh[c] = lay.rbh[c] = -(-h // 8)
        lay.comp_offset[c] = off
        off += lay.bw[c] * lay.bh[c] * 64
        for k in range(64):
            lay.qt[c][k] = 1
    lay.total_coefs = off
    return lay


def dense_ff(L, w, h, ncomp, density, seed):
    rng = np.random.default_rng(seed)
    lay = _layout(L, w, h, ncomp)
    co = np.zeros(lay.total_coefs, dtype=np.int16)
    nz = rng.random(lay.total_coefs) < density
    co[nz] = rng.choice(BIG, size=int(nz.sum()))
    co[::64] = rng.choice([1000, -1000, 511, 0], size=lay.total_coefs // 64)
    return lay, co


def stuffed_fraction(jpeg):
    """stuffed zeros per byte of the file (the headers dilute it a little)"""
    return jpeg.count(b"\xff\x00") / len(jpeg)


# (width, height, components, density): scans of a few bits (one 8x8 block), of less than one group, of one tile (2 KB), of a few
# tiles (one chunk each) and of many tiles per chunk
SHAPES = [(8, 8, 1, 0.0), (8, 8, 1, 0.05), (16, 8, 3, 0.1), (64, 64, 1, 0.3), (200, 120, 3, 0.5), (640, 480, 3, 0.9), (1024, 1024, 1, 0.7)]


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s[:3])) + f"_d{s[3]}")
@pytest.mark.parametrize("prog", [0, 1])
def test_dense_ff_coefficients_match_host_encoder(L, shape, prog):
    w, h, nc, density = shape
    lay, co = dense_ff(L, w, h, nc, density, seed=w * h + nc)
    ref = L.jpeg_encode_coefficients(lay, co, prog)
    if density >= 0.3:
        assert stuffed_fraction(ref) > 0.04
    assert L.jpeg_encode_coefficients_device(lay, co, prog) == ref


def test_megabatches_of_different_contents_equal_oracle(L, O, monkeypatch):
    """Eight same-shaped files a megabatch, each its own content and quality, so that every scan of a batch has its own length and
    its own 0xFF bytes; lossy and lossless, on 1 and 4 threads."""
    from tools.synth import synth_jpeg
    monkeypatch.setenv("B200_MEGABATCH", "8")
    datas = [synth_jpeg(720, 480, i, quality=q) for i, q in enumerate([90, 95, 75, 98, 60, 90, 85, 100] * 2)]
    for lossless in (False, True):
        p = L.default_params()
        p.jpeg_quality, p.jpeg_chroma_subsampling, p.jpeg_progressive, p.jpeg_optimize = 95, 420, 1, int(lossless)
        po = O.params(95, 420, True)
        want = [(O.jpeg_lossless if lossless else O.jpeg_lossy)(d, po) for d in datas]
        for nt in (1, 4):
            for i, (out, code, msg) in enumerate(L.compress_batch(datas, p, n_threads=nt)):
                assert code == 0, msg
                assert out == want[i], (lossless, nt, i)


def test_outgrown_estimate_retries_then_reuses_the_buffers(L, O):
    """Low-quality sources re-encoded at -q 100: the output is several times the sources' entropy-coded size, which sizes the
    encoder's output buffers, so the first run repeats its back half with exact sizes; the files equal the oracle's, and a second
    run through the same buffers needs no retry and gives the same files."""
    import torch
    from tools.synth import synth_jpeg
    assert L.lib().b200_init_device(0) == 0
    datas = [synth_jpeg(1280, 720, i, quality=20) for i in range(8)]
    p = L.default_params()
    p.jpeg_quality, p.jpeg_chroma_subsampling, p.jpeg_progressive = 100, 420, 1
    want = [O.jpeg_lossy(d, O.params(100, 420, True)) for d in datas]
    assert all(len(w) > 2 * len(d) for w, d in zip(want, datas))
    pipe = L.JpegPipe(datas, p, group=8)
    st = torch.cuda.Stream()
    try:
        for rep in range(2):
            pipe.run(st.cuda_stream)
            torch.cuda.synchronize()
            sizes, not_settled, retries = pipe.finish()
            assert not_settled == 0
            assert (retries > 0) == (rep == 0), (rep, retries)
            for i in range(len(datas)):
                assert pipe.fetch(i) == want[i], (rep, i)
    finally:
        pipe.close()
