"""GPU parity tests (run with -m gpu on an H100): the CUDA path, called through the C-ABI, against the CPU oracle.

Bar: bit-exact (integer arithmetic end to end).  Three levels, mirroring how compress_in_memory is assembled
(caesium-clt's src/compressor.rs:305 -> libcaesium jpeg::lossy):
  1. stage: device dequant/IDCT/resample/FDCT/quantise == oracle coefficients,
  2. file: b200_compress_in_memory output bytes == oracle jpeg_lossy output bytes (and the committed sha256),
  3. full-size: BASELINE config sizes through size-independent properties + sampled block checks.
"""
import hashlib
import io
import json
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ZZ = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28,
               35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63])

INPUTS = ["in_420_base_355x237.jpg", "in_420_prog_355x237.jpg", "in_444_base_355x237.jpg", "in_422_base_355x237.jpg",
          "in_gray_base_355x237.jpg", "in_420_base_640x480.jpg", "in_420_tiny_17x9.jpg", "in_420_tiny_3x3.jpg"]
CASES = [(80, 420, True), (80, 420, False), (80, 0, True), (80, 444, True), (80, 422, False), (80, 411, True),
         (50, 420, True), (95, 420, True), (100, 444, False), (5, 420, True), (1, 420, False)]


def _params(L, q, ss, prog):
    p = L.default_params()
    p.jpeg_quality, p.jpeg_chroma_subsampling, p.jpeg_progressive = q, ss, int(prog)
    return p


def _expected():
    with open(os.path.join(os.path.dirname(__file__), "golden", "expected.json")) as f:
        return json.load(f)


def test_device_present(L):
    assert L.lib().b200_init(0) == 0
    assert L.lib().b200_device_count() >= 1


@pytest.mark.parametrize("name", INPUTS)
def test_decode_planes_matches_oracle(L, O, golden, name):
    """K1 + K2: device dequant + IDCT + fancy upsample == oracle decode (== libjpeg-turbo, see test_oracle_jpeg)."""
    data = golden(name)
    lay, co = L.jpeg_decode_coefficients(data)
    got = L.jpeg_decode_planes(lay, co)
    ref = O.Jpeg(data).decode_native()
    assert got.shape == ref.shape
    assert np.array_equal(got, ref)


@pytest.mark.parametrize("name", INPUTS)
@pytest.mark.parametrize("q,ss,prog", CASES)
def test_requantize_and_file_match_oracle(L, O, golden, name, q, ss, prog):
    data = golden(name)
    ref_bytes = O.jpeg_lossy(data, O.params(q, ss, prog))
    ref = O.Jpeg(ref_bytes)
    # 1. stage level
    lay, co = L.jpeg_decode_coefficients(data)
    p = _params(L, q, ss, prog)
    olay = L.jpeg_output_layout(lay, p)
    out = L.jpeg_requantize(lay, co, olay)
    for c in range(lay.ncomp):
        mine = L.component_view(olay, out, c)
        assert mine.shape[:2] == ref.coef(c).shape[:2]
        assert np.array_equal(mine, ref.coef(c)[:, :, ZZ]), f"component {c} coefficients differ"
    # 2. file level, and against the committed golden hash
    got = L.compress_in_memory(data, p)
    assert got == ref_bytes
    exp = _expected()[name]["lossy"][f"q{q}_s{ss}_p{int(prog)}"]
    assert hashlib.sha256(got).hexdigest() == exp["sha256"]


def test_random_coefficients_stage_parity(L, O):
    """Adversarial stage test: random (sparse, large-magnitude) coefficients, odd sizes, every sampling combination."""
    rng = np.random.default_rng(7)
    import ctypes as C
    for (w, h, hs, vs) in [(97, 61, 2, 2), (64, 64, 1, 1), (130, 35, 2, 1), (33, 130, 2, 2), (8, 8, 2, 2), (520, 24, 4, 1)]:
        lay = L.JpegLayout()
        lay.width, lay.height, lay.ncomp, lay.progressive = w, h, 3, 0
        hmax, vmax = hs, vs
        mcux, mcuy = -(-w // (8 * hmax)), -(-h // (8 * vmax))
        off = 0
        for c in range(3):
            lay.hs[c], lay.vs[c] = (hs, vs) if c == 0 else (1, 1)
            lay.bw[c], lay.bh[c] = mcux * lay.hs[c], mcuy * lay.vs[c]
            cw, ch = -(-w * lay.hs[c] // hmax), -(-h * lay.vs[c] // vmax)
            lay.rbw[c], lay.rbh[c] = -(-cw // 8), -(-ch // 8)
            lay.comp_offset[c] = off
            off += lay.bw[c] * lay.bh[c] * 64
            qt = rng.integers(1, 40, size=64).astype(np.uint16)
            for k in range(64):
                lay.qt[c][k] = int(qt[k])
        lay.total_coefs = off
        co = np.zeros(off, dtype=np.int16)
        nz = rng.random(off) < 0.15
        co[nz] = rng.integers(-60, 61, size=int(nz.sum())).astype(np.int16)
        co[::64] = rng.integers(-300, 301, size=off // 64).astype(np.int16)
        # oracle: build an orc_jpeg by hand
        j = O.Jpeg()
        s = j.s
        s.width, s.height, s.ncomp = w, h, 3
        keep = []
        for c in range(3):
            s.hs[c], s.vs[c], s.tq[c], s.cid[c] = lay.hs[c], lay.vs[c], c, c + 1
            s.bw[c], s.bh[c], s.rbw[c], s.rbh[c] = lay.bw[c], lay.bh[c], lay.rbw[c], lay.rbh[c]
            s.cw[c], s.ch[c] = -(-w * lay.hs[c] // hmax), -(-h * lay.vs[c] // vmax)
            nat = np.zeros((lay.bh[c], lay.bw[c], 64), dtype=np.int16)
            nat[:, :, ZZ] = L.component_view(lay, co, c)
            nat = np.ascontiguousarray(nat)
            keep.append(nat)
            s.coef[c] = nat.ctypes.data_as(C.POINTER(C.c_int16))
            qn = np.zeros(64, dtype=np.uint16)
            qn[ZZ] = np.array(lay.qt[c][:], dtype=np.uint16)
            for k in range(64):
                s.qt[c][k] = int(qn[k])
            s.qt_present[c] = 1
        s.hmax, s.vmax, s.mcux, s.mcuy = hmax, vmax, mcux, mcuy
        planes = j.decode_native()
        got_planes = L.jpeg_decode_planes(lay, co)
        assert np.array_equal(got_planes, planes), f"decode planes differ for {(w, h, hs, vs)}"
        for (q, ss) in [(80, 420), (35, 444), (90, 422), (60, 411)]:
            fw = O.forward(planes, O.params(q, ss, False))
            p = _params(L, q, ss, False)
            olay = L.jpeg_output_layout(lay, p)
            out = L.jpeg_requantize(lay, co, olay)
            for c in range(3):
                assert np.array_equal(L.component_view(olay, out, c), fw.coef(c)[:, :, ZZ]), f"{(w, h, hs, vs, q, ss)} comp {c}"


def test_wild_coefficients_wrap_semantics(L, O):
    """IJG range-limit wrap: coefficient values far outside the 8-bit gamut must wrap/clamp exactly like the oracle."""
    rng = np.random.default_rng(11)
    q = np.ones(64, dtype=np.uint16) * 3
    coefs = rng.integers(-700, 701, size=(64, 64)).astype(np.int16)
    lay = L.JpegLayout()
    lay.width, lay.height, lay.ncomp = 64, 64, 1
    lay.hs[0] = lay.vs[0] = 1
    lay.bw[0] = lay.bh[0] = lay.rbw[0] = lay.rbh[0] = 8
    lay.total_coefs = 64 * 64
    for k in range(64):
        lay.qt[0][k] = 3
    got = L.jpeg_decode_planes(lay, coefs.reshape(-1))[0]
    for b in range(64):
        nat = np.zeros(64, dtype=np.int16)
        nat[ZZ] = coefs[b]
        ref = O.idct_islow(nat, q)
        by, bx = divmod(b, 8)
        assert np.array_equal(got[by * 8:by * 8 + 8, bx * 8:bx * 8 + 8], ref)


def test_full_size_4k_properties(L, O):
    """BASELINE config 2 size (3840x2160, q80, 4:2:0): file decodes, idempotence-style and sampled-oracle checks."""
    from PIL import Image
    from tools.synth import synth_jpeg
    data = synth_jpeg(3840, 2160, 0)
    p = _params(L, 80, 420, True)
    out = L.compress_in_memory(data, p)
    im = Image.open(io.BytesIO(out))
    im.draft("YCbCr", im.size)
    assert im.size == (3840, 2160)
    dec = np.asarray(im)
    # (a) whole-file equality with the oracle (the oracle needs ~0.5 s at this size)
    ref = O.jpeg_lossy(data, O.params(80, 420, True))
    assert out == ref
    # (b) the output's decoded pixels equal the oracle's decode of the oracle's output (independent decoder: libjpeg-turbo)
    assert np.array_equal(dec.transpose(2, 0, 1), O.Jpeg(ref).decode_native())
    # (c) baseline and progressive entropy coding carry identical coefficients
    lay_p, co_p = L.jpeg_decode_coefficients(out)
    lay_b, co_b = L.jpeg_decode_coefficients(L.compress_in_memory(data, _params(L, 80, 420, False)))
    assert np.array_equal(co_p, co_b)
    # (d) re-quantising at the same tables is nearly a fixed point: second pass changes few coefficients
    olay = L.jpeg_output_layout(lay_p, p)
    again = L.jpeg_requantize(lay_p, co_p, olay)
    y = L.component_view(olay, again, 0)
    y0 = L.component_view(lay_p, co_p, 0)
    assert (y != y0).mean() < 0.02


def test_batch_matches_single(L, O, golden):
    datas = [golden(n) for n in INPUTS] * 3
    p = _params(L, 80, 420, True)
    res = L.compress_batch(datas, p, n_threads=8)
    for d, (out, code, msg) in zip(datas, res):
        assert code == 0, msg
        assert out == O.jpeg_lossy(d, O.params(80, 420, True))


@pytest.mark.parametrize("prog", [True, False])
def test_lossless_transcode_on_device_matches_oracle(L, O, golden, prog):
    """jpeg::lossless (BASELINE configs[2]): device entropy decode -> device entropy encode, bytes == oracle transcode;
    single calls and the megabatch path, mixed with inputs that take the host route (progressive)."""
    p = _params(L, 80, 0, prog)
    p.jpeg_optimize = 1
    p.keep_metadata = 1
    for name in INPUTS:
        assert L.compress_in_memory(golden(name), p) == O.jpeg_lossless(golden(name), O.params(80, 0, prog, keep_metadata=True)), name
    datas = [golden("in_420_base_355x237.jpg")] * 5 + [golden("in_420_prog_355x237.jpg")] + [golden("in_420_base_640x480.jpg")] * 4
    for d, (out, code, msg) in zip(datas, L.compress_batch(datas, p, n_threads=4)):
        assert code == 0, msg
        assert out == O.jpeg_lossless(d, O.params(80, 0, prog, keep_metadata=True))


@pytest.mark.parametrize("kw", [dict(quality=85, restart_marker_blocks=7), dict(quality=85, restart_marker_rows=1),
                                dict(quality=85, progressive=True, restart_marker_rows=2), dict(quality=92, optimize=True, subsampling=0)])
def test_inputs_that_take_the_host_decoder(L, O, kw):
    """DRI / progressive / multi-table inputs are not device-decodable: host Huffman decode, then the same CUDA transform and
    device encoder -- single calls, and inside a batch next to device-decodable files."""
    import io
    from PIL import Image
    yy, xx = np.mgrid[0:237, 0:355]
    rgb = np.stack([(xx * 3 + yy) % 256, (xx + yy * 2) % 256, (xx * yy // 64) % 256], -1).astype(np.uint8)
    b = io.BytesIO(); Image.fromarray(rgb).save(b, format="JPEG", **kw)
    data = b.getvalue()
    p = _params(L, 80, 420, True)
    want = O.jpeg_lossy(data, O.params(80, 420, True))
    assert L.compress_in_memory(data, p) == want
    plain = io.BytesIO(); Image.fromarray(rgb).save(plain, format="JPEG", quality=85)
    datas = [plain.getvalue()] * 3 + [data] + [plain.getvalue()] * 4
    for d, (out, code, msg) in zip(datas, L.compress_batch(datas, p, n_threads=4)):
        assert code == 0, msg
        assert out == O.jpeg_lossy(d, O.params(80, 420, True))


def _oracle_to_size(O, data, ss, prog, max_size, return_smallest=True):
    """libcaesium's quality bisection restated around the oracle's lossy encoder (one full encode per try)."""
    if len(data) <= max_size:
        return data, None
    tol = max_size // 50
    lo, hi, q = 1, 100, 80
    best = smallest = None
    best_q = None
    for _ in range(10):
        if lo > hi:
            break
        cur = O.jpeg_lossy(data, O.params(q, ss, prog))
        if smallest is None or len(cur) < len(smallest):
            smallest = cur
        if len(cur) <= max_size:
            if best is None or len(cur) > len(best):
                best, best_q = cur, q
            if max_size - len(cur) <= tol:
                break
            lo = q + 1
        else:
            hi = q - 1
        q = (lo + hi) // 2
    if best is not None:
        return best, best_q
    return (smallest if return_smallest else None), None


@pytest.mark.parametrize("name,ss,prog", [("in_420_base_640x480.jpg", 420, True), ("in_444_base_355x237.jpg", 0, True), ("in_420_prog_355x237.jpg", 420, False),
                                          ("in_gray_base_355x237.jpg", 0, True)])
def test_compress_to_size_decode_once_matches_oracle_bisection(L, O, golden, name, ss, prog):
    """compress_to_size_in_memory (compressor.rs:295,298): the source is decoded once and only transform + encode re-run per
    try; the file it answers with -- and the quality it leaves in the parameters -- are those of the restated bisection."""
    data = golden(name)
    for frac in (0.8, 0.45, 0.2, 0.07):
        target = int(len(data) * frac)
        p = _params(L, 80, ss, prog)
        want, want_q = _oracle_to_size(O, data, ss, prog, target)
        out = L.compress_to_size_in_memory(data, p, target)
        assert out == want, (name, frac)
        if want_q is not None:
            assert p.jpeg_quality == want_q and len(out) <= target
    p = _params(L, 80, ss, prog)
    assert L.compress_to_size_in_memory(data, p, len(data) + 10) == data
    # unreachable size: smallest result with return_smallest, code 9 without
    p = _params(L, 80, ss, prog)
    tiny, _ = _oracle_to_size(O, data, ss, prog, 300)
    assert L.compress_to_size_in_memory(data, p, 300, True) == tiny
    with pytest.raises(L.B200Error) as e:
        L.compress_to_size_in_memory(data, _params(L, 80, ss, prog), 300, False)
    assert e.value.code == L.ERR_TOO_LARGE


def test_compress_to_size_4k_costs_less_than_repeated_compress(L, O):
    """Decode-once bisection on a 3840x2160 source: same answer as the restated bisection, and the whole call costs less than
    the tries would as separate compress calls (each of which would parse, upload and entropy-decode the source again)."""
    import time
    from tools.synth import synth_jpeg
    data = synth_jpeg(3840, 2160, 5)
    target = len(data) // 4
    p = _params(L, 80, 420, True)
    L.compress_to_size_in_memory(data, p, target)          # warm buffers
    p = _params(L, 80, 420, True)
    t0 = time.perf_counter(); out = L.compress_to_size_in_memory(data, p, target); t_size = time.perf_counter() - t0
    want, want_q = _oracle_to_size(O, data, 420, True, target)
    assert out == want and p.jpeg_quality == want_q
    t0 = time.perf_counter(); L.compress_in_memory(data, _params(L, 80, 420, True)); t_one = time.perf_counter() - t0
    print(f"compress_to_size: {t_size * 1e3:.1f} ms for the bisection, one compress {t_one * 1e3:.1f} ms")
    assert t_size < 10 * t_one


def test_errors_do_not_abort(L, O, golden):
    p = _params(L, 80, 420, True)
    with pytest.raises(L.B200Error) as e:
        L.compress_in_memory(b"not an image at all", p)
    assert e.value.code == L.ERR_UNKNOWN_FORMAT
    data = golden("in_420_base_355x237.jpg")
    with pytest.raises(L.B200Error) as e:
        L.compress_in_memory(data[:200], p)
    assert e.value.code == L.ERR_CORRUPT_INPUT
    # truncated entropy data: the oracle's answer exactly -- its file (the blocks past the end decoded from zero bits), or
    # CORRUPT_INPUT where it refuses the file
    cut = data[:len(data) // 2] + b"\xff\xd9"
    try:
        want = O.jpeg_lossy(cut, O.params(80, 420, True))
    except O.OracleError:
        want = None
    if want is None:
        with pytest.raises(L.B200Error) as e:
            L.compress_in_memory(cut, p)
        assert e.value.code == L.ERR_CORRUPT_INPUT
    else:
        assert L.compress_in_memory(cut, p) == want
    # and the library is still usable afterwards
    assert L.compress_in_memory(data, p)[:2] == b"\xff\xd8"


def test_group_path_walks_the_scan_on_the_device(L, O, golden):
    """b200_compress_batch no longer walks every entropy-coded segment on the host: the segment is taken to end at the file's last
    EOI and the device counts stuffed bytes and looks for markers while it un-stuffs.  Files whose segment is not what it seems --
    a second image appended behind the first (MPF style: the last EOI is not ours), trailing bytes after EOI, a restart marker
    without a DRI segment -- must come out exactly as the oracle writes them (the host decoder takes the odd ones)."""
    base = [golden(n) for n in ("in_420_base_640x480.jpg", "in_420_base_355x237.jpg")]
    a = base[0]
    appended = a + base[1]                                   # two images back to back: the first is the picture
    trailing = a + b"\x00\x01\x02trailing bytes after EOI" * 50
    sos = a.index(b"\xff\xda")
    body = bytearray(a)
    k = len(a) // 2
    while body[k] == 0xFF or body[k - 1] == 0xFF or body[k + 1] == 0xFF:
        k += 1
    stray = bytes(body[:k]) + b"\xff\xd0" + bytes(body[k:])    # a marker in the middle of the scan
    assert k > sos
    work = [a, appended, a, trailing, a, a, a, a, a, a]
    p = _params(L, 80, 420, True)
    po = O.params(80, 420, True)
    res = L.compress_batch(work, p, n_threads=4)
    for i, (out, code, msg) in enumerate(res):
        assert code == 0, (i, msg)
        assert out == O.jpeg_lossy(work[i], po), i
    # the stray marker: whatever the host decoder makes of it (libjpeg resynchronises), the batch and the single call agree
    single = None
    try:
        single = L.compress_in_memory(stray, p)
    except L.B200Error as e:
        single = e.code
    out, code, msg = L.compress_batch([a, stray, a, a], p, n_threads=2)[1]
    assert (out if code == 0 else code) == single
