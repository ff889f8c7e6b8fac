"""The device decoder's write pass stores every coefficient block whole and clears nothing beforehand.

A slot keeps its coefficient buffers from call to call, so whatever the previous image left there is what an unwritten sector
would show.  The worst pair is a dense image (a noisy picture at high quality: non-zero coefficients up to index 63) followed
by a sparse one of the same shape (flat areas at low quality: most blocks a DC coefficient and an end-of-block), and the
reverse: every `--lossless` output must be the oracle's byte for byte, on one worker thread so that the same buffers are used
again.

CPU part: a serial run of the kernels with the write pass as the device runs it (tests/emul/gpudec_write_emul.cpp: one owner
per block, whole sectors, a poisoned buffer, the stores counted per block) on the golden files and the dense and sparse files
at every subsequence size, and on damaged files against the emulation that writes coefficient by coefficient
(tests/emul/gpudec_emul.cpp): the same answer, the same anomalies, the same coefficients.
GPU part (-m gpu): the pairs through the single call and the megabatch, at the shapes of the golden files, for a grey file that
declares sampling factors 2x2, for one 3840x2160 pair, and at small subsequence sizes (B200_DEC_SUBSEQ is read once per
process: one subprocess per value)."""
import ctypes as C
import io
import os
import subprocess
import sys

import numpy as np
import pytest
from PIL import Image

import test_gpudec_damaged as D
from test_gpudec import BASELINE_INPUTS, EMUL_DIR, ROOT, emul  # noqa: F401  (emul: module fixture, the coefficient-by-coefficient emulation)

HERE = os.path.dirname(os.path.abspath(__file__))
SUBSEQ = [128, 256, 512, 1024, 2048]
SHAPES = [("420", 355, 237), ("444", 355, 237), ("422", 355, 237), ("grey", 355, 237), ("grey22", 355, 237), ("420", 640, 480), ("420", 17, 9)]
SMALL_SUBSEQ = [128, 512]


def _pixels(kind, w, h, seed):
    rng = np.random.default_rng(seed)
    if kind == "dense":             # a picture under noise: pure noise needs more synchronisation rounds than the decoder launches
        from tools.synth import synth_rgb
        return np.clip(synth_rgb(w, h, seed).astype(np.int32) + rng.integers(-40, 41, (h, w, 3)), 0, 255).astype(np.uint8)
    img = np.empty((h, w, 3), np.uint8)             # sparse: four flat areas with one sharp edge each way
    img[:] = rng.integers(0, 256, 3)
    img[h // 3:, w // 2:] = rng.integers(0, 256, 3)
    img[2 * h // 3:, :w // 4] = rng.integers(0, 256, 3)
    img[:h // 5, 3 * w // 4:] = rng.integers(0, 256, 3)
    return img


def make_file(kind, layout, w, h, seed):
    """kind: 'dense' (noisy picture, q96) or 'sparse' (flat areas, q25); layout: '420' / '422' / '444' / 'grey' / 'grey22'"""
    px = _pixels(kind, w, h, seed)
    q = 96 if kind == "dense" else 25
    b = io.BytesIO()
    if layout.startswith("grey"):
        Image.fromarray(px[:, :, 1], "L").save(b, "JPEG", quality=q)
    else:
        Image.fromarray(px, "RGB").save(b, "JPEG", quality=q, subsampling={"420": "4:2:0", "422": "4:2:2", "444": "4:4:4"}[layout])
    data = bytearray(b.getvalue())
    if layout == "grey22":
        # the only component declares 2x2: legal, and without meaning for a single-component scan (one block per MCU); a reader
        # that believed it would lay the plane out wider than the blocks the scan codes
        sof = data.index(b"\xff\xc0")
        assert data[sof + 9] == 1 and data[sof + 11] == 0x11
        data[sof + 11] = 0x22
    return bytes(data)


def pair(layout, w, h, seed=1):
    return make_file("dense", layout, w, h, seed), make_file("sparse", layout, w, h, seed + 1)


def _lossless_params(L):
    p = L.default_params()
    p.jpeg_quality, p.jpeg_chroma_subsampling, p.jpeg_progressive, p.jpeg_optimize = 80, 0, 1, 1
    return p


def check_pairs(L, O, shapes, batch=True):
    """dense -> sparse -> dense -> sparse through the same buffers: the single call, then megabatches of one kind each"""
    p = _lossless_params(L)
    for layout, w, h in shapes:
        dense, sparse = pair(layout, w, h)
        want = {d: O.jpeg_lossless(d, O.params(80, 0, True)) for d in (dense, sparse)}
        for d in (dense, sparse, dense, sparse):
            assert L.compress_in_memory(d, p) == want[d], (layout, w, h, "single", d is dense)
        if not batch:
            continue
        for d in (dense, sparse, dense, sparse):
            for out, code, msg in L.compress_batch([d] * 3, p, n_threads=1):
                assert code == 0 and out == want[d], (layout, w, h, "batch", d is dense, msg)


# ---------------------------------------------------------------------------------------------------------------- CPU
@pytest.fixture(scope="module")
def write_emul():
    so = os.path.join(EMUL_DIR, "libgpudec_write_emul.so")
    csrc = os.path.join(ROOT, "caesium-clt_b200", "csrc")
    srcs = [os.path.join(EMUL_DIR, "gpudec_write_emul.cpp"), os.path.join(csrc, "jpeg_host.cpp"), os.path.join(csrc, "jpeg_gpudec_core.h"), os.path.join(csrc, "jpeg_gpuenc_core.h")]
    if not os.path.exists(so) or any(os.path.getmtime(f) > os.path.getmtime(so) for f in srcs):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-msse2", "-Wno-unknown-pragmas", "-o", so, srcs[0], srcs[1]])
    return C.CDLL(so)


def write_decode(lib, data, total_coefs, subseq, max_rounds=256, fn="emul_gpu_write_checked"):
    """-> (rc, coefficients, ANOM_* mask); rc 13 / 15 = a block addressed wrongly / not stored whole exactly once"""
    out = np.zeros(total_coefs, dtype=np.int16)
    r, a = C.c_int(0), C.c_int(0)
    rc = getattr(lib, fn)(data, C.c_size_t(len(data)), subseq, max_rounds, out.ctypes.data_as(C.c_void_p), C.c_longlong(out.size), C.byref(r), C.byref(a))
    return rc, out, a.value


@pytest.mark.parametrize("subseq", SUBSEQ)
@pytest.mark.parametrize("name", BASELINE_INPUTS)
def test_emulated_write_pass_on_the_golden_files(L, write_emul, golden, name, subseq):
    data = golden(name)
    lay, ref = L.jpeg_decode_coefficients(data)
    rc, out, _ = write_decode(write_emul, data, lay.total_coefs, subseq)
    assert rc == 0 and np.array_equal(out, ref)


@pytest.mark.parametrize("subseq", SUBSEQ)
@pytest.mark.parametrize("layout,w,h", [("420", 131, 77), ("444", 67, 45), ("grey", 93, 61), ("grey22", 93, 61)])
def test_emulated_write_pass_stores_every_block_once(L, write_emul, layout, w, h, subseq):
    for data in pair(layout, w, h):
        lay, ref = L.jpeg_decode_coefficients(data)
        rc, out, _ = write_decode(write_emul, data, lay.total_coefs, subseq)
        assert rc == 0 and np.array_equal(out, ref)


@pytest.mark.parametrize("subseq", [128, 2048])
@pytest.mark.parametrize("name", ["in_420_base_355x237.jpg", "in_444_base_355x237.jpg", "in_gray_base_355x237.jpg", "in_420_tiny_17x9.jpg"])
def test_owner_reports_what_the_single_store_pass_reports(L, emul, write_emul, golden, name, subseq):
    """Damaged scans: the owner of a block reports its anomalies, past the end of its subsequence too, and nobody reports the
    head it skips.  Answer, rules and (where the image is decoded) coefficients equal the coefficient-by-coefficient emulation's,
    whose expectations tests/test_gpudec_damaged.py pins against the host decoder."""
    data = golden(name)
    n = D.total_coefs(L, data)
    start, end = D.scan_bounds(data)
    small = end - start < 400
    files = D.cuts(data, end - start if small else 150, 0 if small else 60, 5) + D.bit_flips(data, 60, 15) + D.byte_replacements(data, 20, 16)
    rules = decoded = 0
    for i, d in enumerate(files):
        rc0, out0, a0 = write_decode(emul, d, n, subseq, fn="emul_gpu_decode_checked")
        rc1, out1, a1 = write_decode(write_emul, d, n, subseq)
        assert (rc1, a1) == (rc0, a0), i
        if rc0 == 0:
            assert np.array_equal(out1, out0), i
            decoded += 1
        rules |= a0
    assert decoded and rules & D.ANOM_END and (small or rules & (D.ANOM_CODE | D.ANOM_RUN))


# ---------------------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("layout,w,h", SHAPES)
def test_dense_then_sparse_through_the_same_buffers(L, O, layout, w, h):
    L.set_entropy_mode(3)
    check_pairs(L, O, [(layout, w, h)])


@pytest.mark.gpu
def test_dense_then_sparse_at_3840x2160(L, O):
    L.set_entropy_mode(3)
    check_pairs(L, O, [("420", 3840, 2160)])


@pytest.mark.gpu
@pytest.mark.parametrize("layout,w,h", [("420", 640, 480), ("444", 355, 237), ("422", 355, 237), ("grey22", 355, 237)])
def test_resident_pipe_settles_on_dense_and_sparse(L, O, layout, w, h):
    """The resident pipe has no host decoder behind it: both kinds must be decoded on the device, in either order, in one pipe."""
    import torch
    assert L.lib().b200_init_device(0) == 0
    dense, sparse = pair(layout, w, h)
    p = _lossless_params(L)
    want = {d: O.jpeg_lossless(d, O.params(80, 0, True)) for d in (dense, sparse)}
    st = torch.cuda.Stream()
    for work in ([dense] * 2 + [sparse] * 2, [sparse] * 2 + [dense] * 2):
        pipe = L.JpegPipe(work, p, group=2)
        try:
            for _ in range(2):
                pipe.run(st.cuda_stream)
            torch.cuda.synchronize()
            _, not_settled, _ = pipe.finish()
            assert not_settled == 0
            for i, d in enumerate(work):
                assert pipe.fetch(i) == want[d], i
        finally:
            pipe.close()


@pytest.mark.gpu
@pytest.mark.parametrize("subseq", SMALL_SUBSEQ)
def test_small_subsequences(subseq):
    """Blocks longer than a subsequence: the threads in the middle of such a block own nothing."""
    env = dict(os.environ, B200_DEC_SUBSEQ=str(subseq))
    code = "import test_gpudec_write_gpu as t; t.subprocess_main()"
    r = subprocess.run([sys.executable, "-c", code], cwd=HERE, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]


def subprocess_main():
    import conftest
    conftest._import_pkg()
    import caesium_clt_b200._lib as L
    from oracle import oracle as O
    L.lib()
    O.lib()
    L.set_entropy_mode(3)
    check_pairs(L, O, [("420", 355, 237), ("444", 131, 77), ("grey22", 355, 237), ("420", 17, 9)])
    print("ok")
