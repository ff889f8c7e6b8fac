"""Device entropy DECODER (self-synchronising parallel Huffman decoding, jpeg_gpudec_core.h).

CPU part: the kernel bodies run serially (tests/emul/gpudec_emul.cpp) must reproduce the host decoder's coefficients,
for several subsequence sizes; ineligible inputs (progressive, restart intervals) are refused; degenerate periodic
streams report non-convergence (the product then decodes on the host).
GPU part (-m gpu): the same through the library, end to end against the oracle, in every entropy mode."""
import ctypes as C
import io
import os
import subprocess

import numpy as np
import pytest
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMUL_DIR = os.path.join(ROOT, "tests", "emul")
BASELINE_INPUTS = ["in_420_base_355x237.jpg", "in_444_base_355x237.jpg", "in_422_base_355x237.jpg", "in_gray_base_355x237.jpg",
                   "in_420_base_640x480.jpg", "in_420_tiny_17x9.jpg", "in_420_tiny_3x3.jpg"]


@pytest.fixture(scope="module")
def emul():
    so = os.path.join(EMUL_DIR, "libgpudec_emul.so")
    srcs = [os.path.join(EMUL_DIR, "gpudec_emul.cpp"), os.path.join(ROOT, "caesium-clt_b200", "csrc", "jpeg_host.cpp"),
            os.path.join(ROOT, "caesium-clt_b200", "csrc", "jpeg_gpudec_core.h"), os.path.join(ROOT, "caesium-clt_b200", "csrc", "jpeg_gpuenc_core.h")]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-msse2", "-Wno-unknown-pragmas", "-o", so, srcs[0], srcs[1]])
    return C.CDLL(so)


def emul_decode(emul, data, total_coefs, subseq=1024, max_rounds=64):
    out = np.zeros(total_coefs, dtype=np.int16)
    r = C.c_int(0)
    rc = emul.emul_gpu_decode(data, C.c_size_t(len(data)), subseq, max_rounds, out.ctypes.data_as(C.c_void_p), C.c_longlong(out.size), C.byref(r))
    return rc, out, r.value


@pytest.mark.parametrize("name", BASELINE_INPUTS)
@pytest.mark.parametrize("subseq", [128, 1024, 2048, 4096])
def test_parallel_decode_matches_host_decoder(L, emul, golden, name, subseq):
    data = golden(name)
    lay, ref = L.jpeg_decode_coefficients(data)
    rc, out, rounds = emul_decode(emul, data, lay.total_coefs, subseq, 256)
    assert rc == 0
    assert np.array_equal(out, ref)


def test_ineligible_inputs_are_refused(L, emul, golden):
    data = golden("in_420_prog_355x237.jpg")                       # progressive
    lay, _ = L.jpeg_decode_coefficients(data)
    assert emul_decode(emul, data, lay.total_coefs)[0] == 10
    b = io.BytesIO()                                                 # restart interval
    Image.open(io.BytesIO(golden("in_420_base_640x480.jpg"))).save(b, "JPEG", quality=80, restart_marker_blocks=7)
    d2 = b.getvalue()
    if b"\xff\xdd" in d2:                                           # Pillow wrote a DRI segment
        lay, _ = L.jpeg_decode_coefficients(d2)
        assert emul_decode(emul, d2, lay.total_coefs)[0] == 10


def test_optimised_tables_and_high_quality(L, emul):
    """Files with per-image optimised Huffman tables and long codes (q=100) decode identically."""
    from tools.synth import synth_rgb
    for q, kw in [(100, {}), (30, {"optimize": True}), (95, {"optimize": True, "subsampling": "4:4:4"})]:
        b = io.BytesIO()
        Image.fromarray(synth_rgb(333, 211, 40 + q), "RGB").save(b, "JPEG", quality=q, **kw)
        data = b.getvalue()
        lay, ref = L.jpeg_decode_coefficients(data)
        rc, out, _ = emul_decode(emul, data, lay.total_coefs, 512, 256)
        assert rc == 0 and np.array_equal(out, ref)


def test_kernel_form_tables_equal_the_jdhuff_search(emul, golden):
    """Two-level lookup tables (what the kernels read) against the canonical maxcode search, for every 16-bit pattern and
    every table of the scan -- Annex K tables, per-image optimised tables, q=100 tables with 16-bit codes in use."""
    from tools.synth import synth_rgb
    files = [golden(n) for n in BASELINE_INPUTS[:5]]
    for q, kw in [(100, {}), (30, {"optimize": True}), (95, {"optimize": True, "subsampling": "4:4:4"}), (5, {"optimize": True})]:
        b = io.BytesIO()
        Image.fromarray(synth_rgb(333, 211, 40 + q), "RGB").save(b, "JPEG", quality=q, **kw)
        files.append(b.getvalue())
    emul.emul_gpu_dec_table_check.restype = C.c_longlong
    for data in files:
        used = C.c_int(-1)
        bad = emul.emul_gpu_dec_table_check(data, C.c_size_t(len(data)), C.byref(used))
        assert bad == 0, bad
        assert 0 <= used.value <= 1536


def test_adversarial_tables_fit_or_are_refused_cleanly(emul):
    """DHTs built to spread long codes over many 9-bit prefixes: the second-level pool either holds them (and the lookup equals the
    jdhuff.c search everywhere) or the table set is refused with an all-invalid, in-bounds result -- the image then goes to the
    host decoder, like a stream that does not converge.  Either way every block's selector names one of the first nlook slots,
    the only ones the kernels stage: a selector past them would read shared memory nobody wrote."""
    dc_bits = np.zeros(17, np.uint8); dc_bits[2] = 1; dc_bits[3] = 5; dc_bits[4] = 1; dc_bits[5] = 1; dc_bits[6] = 1; dc_bits[7] = 1; dc_bits[8] = 1; dc_bits[9] = 1
    dc_vals = np.zeros(256, np.uint8); dc_vals[:12] = np.arange(12)
    outcomes = set()
    for counts in ({1: 1, 10: 24, 11: 48, 12: 60, 13: 40, 14: 30, 15: 20, 16: 33},       # many prefixes with 10..16-bit codes
                   {2: 1, 3: 1, 9: 2, 16: 200},                                            # a block of 16-bit codes
                   {1: 1, 2: 1, 12: 100, 16: 150},
                   {8: 255}):                                                              # no long codes at all
        bits = np.zeros(17, np.uint8)
        for l, c in counts.items():
            bits[l] = c
        vals = np.zeros(256, np.uint8); n = int(bits.sum()); vals[:n] = np.arange(n)
        kraft = sum(int(bits[l]) * 2.0 ** -l for l in range(1, 17))
        assert kraft <= 1.0
        for ntab in (1, 4):
            used, bad = C.c_int(-1), C.c_longlong(-1)
            ok = emul.emul_build_tables_raw(bits.ctypes.data_as(C.c_void_p), vals.ctypes.data_as(C.c_void_p), dc_bits.ctypes.data_as(C.c_void_p),
                                            dc_vals.ctypes.data_as(C.c_void_p), ntab, C.byref(used), C.byref(bad))
            assert bad.value == 0 and 0 <= used.value <= 1536, (counts, ntab, ok, used.value, bad.value)
            outcomes.add(ok)
    assert outcomes == {1}             # up to four such AC tables still fit (<= 368 entries each)
    # a fifth adversarial table (the DC slot) overflows the pool: refused, nothing out of bounds, tables left all-invalid
    bits = np.zeros(17, np.uint8)
    for l, c in {1: 1, 10: 24, 11: 48, 12: 60, 13: 40, 14: 30, 15: 20, 16: 33}.items():
        bits[l] = c
    vals = np.arange(256).astype(np.uint8)
    used, bad = C.c_int(-1), C.c_longlong(-1)
    ok = emul.emul_build_tables_raw(bits.ctypes.data_as(C.c_void_p), vals.ctypes.data_as(C.c_void_p), bits.ctypes.data_as(C.c_void_p), vals.ctypes.data_as(C.c_void_p),
                                    4, C.byref(used), C.byref(bad))
    assert ok == 0 and bad.value == 0 and used.value == 0


def test_flat_image_reports_non_convergence_or_matches(L, emul):
    """A constant image is a periodic bit stream: a wrong phase can persist, so the round budget may run out.  Whatever
    the outcome, a 0 return code must mean identical coefficients."""
    b = io.BytesIO()
    Image.new("RGB", (1024, 1024), (90, 140, 200)).save(b, "JPEG", quality=90)
    data = b.getvalue()
    lay, ref = L.jpeg_decode_coefficients(data)
    rc, out, rounds = emul_decode(emul, data, lay.total_coefs, 1024, 8)
    assert rc in (0, 11)
    if rc == 0:
        assert np.array_equal(out, ref)
    rc, out, rounds = emul_decode(emul, data, lay.total_coefs, 1024, 100000)
    assert rc == 0 and np.array_equal(out, ref)


# ---------------------------------------------------------------------------------------------------------------- GPU
def _params(L, q=80, ss=420, prog=True):
    p = L.default_params()
    p.jpeg_quality, p.jpeg_chroma_subsampling, p.jpeg_progressive = q, ss, int(prog)
    return p


@pytest.mark.gpu
@pytest.mark.parametrize("name", BASELINE_INPUTS + ["in_420_prog_355x237.jpg"])
def test_device_decode_end_to_end_all_modes(L, O, golden, name):
    data = golden(name)
    ref = O.jpeg_lossy(data, O.params(80, 420, True))
    try:
        for mode in (3, 2, 1, 0):
            L.set_entropy_mode(mode)
            assert L.compress_in_memory(data, _params(L)) == ref, f"entropy mode {mode}"
    finally:
        L.set_entropy_mode(3)


@pytest.mark.gpu
def test_device_decode_4k_and_flat_fallback(L, O):
    from tools.synth import synth_jpeg
    L.set_entropy_mode(3)
    data = synth_jpeg(3840, 2160, 2)
    assert L.compress_in_memory(data, _params(L)) == O.jpeg_lossy(data, O.params(80, 420, True))
    b = io.BytesIO()
    Image.new("RGB", (2048, 2048), (90, 140, 200)).save(b, "JPEG", quality=90)       # periodic stream: host fallback path
    flat = b.getvalue()
    assert L.compress_in_memory(flat, _params(L)) == O.jpeg_lossy(flat, O.params(80, 420, True))
    for q, kw in [(100, {}), (30, {"optimize": True})]:
        from tools.synth import synth_rgb
        b = io.BytesIO()
        Image.fromarray(synth_rgb(1333, 811, 77), "RGB").save(b, "JPEG", quality=q, **kw)
        d = b.getvalue()
        assert L.compress_in_memory(d, _params(L, 70, 444, False)) == O.jpeg_lossy(d, O.params(70, 444, False))


@pytest.mark.gpu
def test_megabatch_groups_mixed_inputs(L, O, golden):
    """b200_compress_batch packs consecutive same-shaped baseline JPEGs into one launch sequence; everything else in the
    chunk (other shapes, progressive files, periodic streams, non-images) must still come out right, in input order."""
    from tools.synth import synth_rgb
    L.set_entropy_mode(3)
    same = []
    for i in range(11):                                  # 11 same-shaped baseline files with different content / quality
        b = io.BytesIO()
        Image.fromarray(synth_rgb(322, 199, 200 + i), "RGB").save(b, "JPEG", quality=70 + 2 * i, subsampling="4:2:0")
        same.append(b.getvalue())
    b = io.BytesIO()
    Image.new("RGB", (322, 199), (10, 200, 90)).save(b, "JPEG", quality=90, subsampling="4:2:0")     # same shape, periodic stream
    flat = b.getvalue()
    datas = same[:3] + [golden("in_420_prog_355x237.jpg")] + same[3:6] + [b"not an image"] + [flat] + same[6:] + [golden("in_444_base_355x237.jpg"), golden("in_gray_base_355x237.jpg")]
    for q, ss, prog in [(80, 420, True), (60, 444, False)]:
        res = L.compress_batch(datas, _params(L, q, ss, prog), n_threads=4)
        for d, (out, code, msg) in zip(datas, res):
            if d == b"not an image":
                assert code == L.ERR_UNKNOWN_FORMAT
            else:
                assert code == 0, msg
                assert out == O.jpeg_lossy(d, O.params(q, ss, prog))


@pytest.mark.gpu
def test_device_decode_concurrent(L, O, golden):
    datas = [golden(n) for n in BASELINE_INPUTS] * 8
    L.set_entropy_mode(3)
    res = L.compress_batch(datas, _params(L, 85, 0, True), n_threads=16)
    for d, (out, code, msg) in zip(datas, res):
        assert code == 0, msg
        assert out == O.jpeg_lossy(d, O.params(85, 0, True))
