"""GPU parity tests at the EXACT sizes of BASELINE.json's configs (round-1 verdict item 1c/1d), through the C-ABI:
  configs[1]/[2]  3840x2160 JPEG: q80 4:2:0 re-encode and --lossless transcode, bytes == oracle (single call, batch, resident pipe)
  configs[3]      4096x4096 RGBA PNG --lossless --png-opt-level 3: output decodes to the source pixels; the filtered stream it
                  carries equals the oracle's for one of the level's strategies; K6 / K7 stage outputs == oracle at full size
  configs[4]      6000x4000 JPEG -> -q 85 --width 1920 --format webp: bytes == oracle
and the reference's own sample files (tests/golden/reference_samples, copied from caesium-clt's samples) through the CUDA path:
bytes == oracle, plus the size facts the reference's tests assert (compressor.rs:1051-1068) on the PRODUCT's output."""
import io
import os
import zlib
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from pngutil import idat_stream, pil_pixels

pytestmark = pytest.mark.gpu

SAMPLES = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_samples")


def sample(name):
    with open(os.path.join(SAMPLES, name), "rb") as f:
        return f.read()


def jparams(L, q=80, ss=420, prog=True, lossless=False):
    p = L.default_params()
    p.jpeg_quality, p.jpeg_chroma_subsampling, p.jpeg_progressive, p.jpeg_optimize = q, ss, 1 if prog else 0, 1 if lossless else 0
    return p


@pytest.fixture(scope="module")
def jpegs_4k():
    from tools.synth import synth_jpeg
    with ThreadPoolExecutor(4) as ex:
        return list(ex.map(lambda i: synth_jpeg(3840, 2160, i), range(4)))


def test_config1_and_2_full_size_bytes_equal_oracle(L, O, jpegs_4k):
    po, pl = O.params(80, 420, True), O.params(80, 0, True)
    want_lossy = [O.jpeg_lossy(d, po) for d in jpegs_4k]
    want_lossless = [O.jpeg_lossless(d, pl) for d in jpegs_4k]
    # single calls
    assert L.compress_in_memory(jpegs_4k[0], jparams(L)) == want_lossy[0]
    assert L.compress_in_memory(jpegs_4k[1], jparams(L, lossless=True, ss=0)) == want_lossless[1]
    # megabatches (b200_compress_batch groups same-shaped files)
    work = jpegs_4k * 5
    for params, want in ((jparams(L), want_lossy), (jparams(L, lossless=True, ss=0), want_lossless)):
        res = L.compress_batch(work, params, n_threads=8)
        for i, (out, code, msg) in enumerate(res):
            assert code == 0, msg
            assert out == want[i % 4], f"image {i}"


@pytest.mark.parametrize("lossless", [False, True])
@pytest.mark.parametrize("group", [3, 8])
def test_resident_pipe_full_path_matches_oracle(L, O, jpegs_4k, lossless, group):
    """bench.py's `value` leg: scan bytes resident in HBM -> decode -> transform -> encode -> scan bytes in HBM, no host wait
    inside run(); every image fetched afterwards is the oracle's file, also after a second run on the same buffers."""
    import torch
    assert L.lib().b200_init_device(0) == 0
    work = jpegs_4k * 2 + jpegs_4k[:3]                     # 11 images: ragged last group
    p = jparams(L, lossless=lossless, ss=0 if lossless else 420)
    po = O.params(80, 0 if lossless else 420, True)
    want = [(O.jpeg_lossless if lossless else O.jpeg_lossy)(d, po) for d in jpegs_4k]
    pipe = L.JpegPipe(work, p, group=group)
    st = torch.cuda.Stream()
    for rep in range(2):
        n = pipe.run(st.cuda_stream)
        assert n > 20
        torch.cuda.synchronize()
        sizes, not_settled, retries = pipe.finish()
        assert not_settled == 0
        for i in (0, 5, 10):
            got = pipe.fetch(i)
            assert got == want[i % 4 if i < 8 else i - 8], (rep, i)
        assert all(s > 100000 for s in sizes)
    times = pipe.kernel_times(1)
    assert "k_gd_write" in times and "k_geb_emit" in times and (lossless or "k_fused_same" in times)
    if not lossless:
        # 4:2:0 -> 4:2:0 transform: fused luma, chroma IDCT, collapsed chroma resample + FDCT, each launched once per megabatch
        for name in ("k_fused_same", "k_idct_plane", "k_chroma420_refdct"):
            ms, launches = times[name]
            assert launches == 1 and ms > 0, (name, times[name])
    pipe.close()


@pytest.fixture(scope="module")
def png_4096():
    from tools.synth import synth_png_rgba
    return synth_png_rgba(4096, 4096, 1)


def test_config3_full_size_png_level3(L, O, png_4096):
    p = L.default_params(); p.png_optimize = 1; p.png_optimization_level = 3
    out = L.compress_in_memory(png_4096, p)
    src_px = np.asarray(pil_pixels(png_4096))
    assert src_px.shape == (4096, 4096, 4)
    assert np.array_equal(np.asarray(pil_pixels(out)), src_px), "not lossless"
    assert len(out) < len(png_4096)
    ihdr, idat, _ = idat_stream(out)
    assert ihdr[:2] == (4096, 4096)
    filt = np.frombuffer(zlib.decompress(idat), np.uint8)
    channels = {2: 3, 6: 4, 0: 1, 4: 2}[ihdr[3]]
    raw = src_px[:, :, :channels].reshape(4096, -1) if channels < 4 else src_px.reshape(4096, -1)
    filt = filt.reshape(4096, raw.shape[1] + 1)
    # the product tried the level's strategies and kept one: its filtered rows are the oracle's rows for that strategy
    strategies = L.png_level_strategies(3)
    with ThreadPoolExecutor(len(strategies)) as ex:
        oracle_rows = list(ex.map(lambda s: O.png_filter(raw, channels, s), strategies))
    match = [s for s, f in zip(strategies, oracle_rows) if np.array_equal(f, filt)]
    assert match, "the output's filtered stream is none of the oracle's level-3 candidates"
    # stage parity at full size: K6 on the device for every strategy of the level, K7 on the winner's stream
    for s, f in zip(strategies, oracle_rows):
        assert np.array_equal(L.png_filter(raw, channels, s), f), f"K6 strategy {s}"
    stream = filt.reshape(-1)
    tok, hist = L.png_lz77(stream, channels, filt.shape[1])
    wtok, whist = O.png_lz77(stream, channels, filt.shape[1])
    assert np.array_equal(hist, whist) and np.array_equal(tok, wtok)


def test_config4_full_size_jpeg_to_webp(L, O):
    from tools.synth import synth_jpeg
    src = synth_jpeg(6000, 4000, 0)
    p = L.default_params(); p.webp_quality = 85; p.width = 1920
    out = L.convert_in_memory(src, p, 3)
    ycc = O.Jpeg(src).decode_native()
    rgb = O.ycc_to_rgb(ycc)
    nw, nh = O.compute_dimensions(6000, 4000, 1920, 0)
    assert (nw, nh) == (1920, 1280)
    rgb = np.stack([O.resize_plane(rgb[c], nw, nh) for c in range(3)])
    assert out == O.webp_encode(rgb, 85)[0]
    from PIL import Image
    im = Image.open(io.BytesIO(out)); im.load()
    assert im.size == (1920, 1280)


# ---- the reference's own fixtures through the CUDA path -------------------------------------------------------------------------
def test_reference_jpeg_samples_bytes_equal_oracle_and_size_facts_hold(L, O):
    j0, j1 = sample("j0.JPG"), sample("j1.jpg")
    sizes = {}
    for q in (50, 80, 95, 100):
        p = jparams(L, q=q, ss=0)                    # caesiumclt -q N: auto subsampling, progressive
        out = L.compress_in_memory(j0, p)
        assert out == O.jpeg_lossy(j0, O.params(q, 0, True)), f"j0 q{q}"
        sizes[q] = len(out)
    # compressor.rs:1051-1068 (test_compress_quality / lossy size facts), asserted on the PRODUCT's bytes
    assert sizes[95] > 391657
    assert sizes[50] < 790435
    assert sizes[100] >= sizes[80] >= sizes[50]
    for q in (80, 40):
        assert L.compress_in_memory(j1, jparams(L, q=q, ss=0)) == O.jpeg_lossy(j1, O.params(q, 0, True)), f"j1 q{q}"
    # --lossless on both (progressive sources: host entropy decode, device encode)
    for d in (j0, j1):
        assert L.compress_in_memory(d, jparams(L, lossless=True, ss=0)) == O.jpeg_lossless(d, O.params(80, 0, True))
    # resize + quality on j0 (compressor.rs resize tests use --width / --height on the samples)
    p = jparams(L, q=80, ss=0); p.width = 800
    out = L.compress_in_memory(j0, p)
    from PIL import Image
    im = Image.open(io.BytesIO(out)); assert im.size[0] == 800


def test_reference_png_samples_lossless_through_the_device(L):
    for name in ("p0.png", "p2.png"):
        src = sample(name)
        for level in (2, 3, 6):
            p = L.default_params(); p.png_optimize = 1; p.png_optimization_level = level
            out = L.compress_in_memory(src, p)
            a, b = pil_pixels(src), pil_pixels(out)
            assert np.array_equal(np.asarray(a.convert("RGBA")), np.asarray(b.convert("RGBA"))), (name, level)
    # the all-formats batch of the reference's tests (compressor.rs:769-787): every sample the path takes succeeds
    items = [sample("j0.JPG"), sample("j1.jpg"), sample("p0.png"), sample("p2.png")]
    p = L.default_params(); p.png_optimize = 1; p.jpeg_quality = 80
    for out, code, msg in L.compress_batch(items, p, n_threads=4):
        assert code == 0, msg
