"""Device entropy DECODER on damaged scans: truncated files, bit flips and replaced bytes inside the entropy-coded segment.

The device decoder (jpeg_gpudec_core.h) may only report an image as decoded when its coefficients are the host decoder's
(jpeg_host.cpp).  On a stream it cannot decode the way the host does -- an invalid code, a run past index 63, a stream that
ends before its last block -- it reports the image as not settled, and the host decoder then answers with its coefficients or
with CORRUPT_INPUT, whichever it would have answered with the device decoder switched off.

CPU part: the serial run of the kernels (tests/emul/gpudec_emul.cpp) against L.jpeg_decode_coefficients, and the host transcode
against the oracle on the same damaged files.
GPU part (-m gpu): every entropy mode gives the same answer, the megabatch path gives what the single call gives, and the resident
pipe decodes clean files of every shape on the device (not_settled == 0) and refuses exactly the damaged ones."""
import ctypes as C
import io
import random

import numpy as np
import pytest
from PIL import Image

from test_gpudec import emul  # noqa: F401  (module fixture: the serial CPU run of the decoder's passes)

ANOM_CODE, ANOM_RUN, ANOM_END = 1, 2, 4
BASE_355 = ["in_420_base_355x237.jpg", "in_444_base_355x237.jpg", "in_422_base_355x237.jpg", "in_gray_base_355x237.jpg"]
SUBSEQ = [128, 2048]            # the smallest subsequence size and the product's default
EOI = b"\xff\xd9"


def emul_decode(emul, data, total_coefs, subseq, max_rounds, anomalies):
    """-> (rc, coefficients, rounds); appends to `anomalies` the ANOM_* mask of the run (non-zero only with rc 14)."""
    out = np.zeros(total_coefs, dtype=np.int16)
    r, a = C.c_int(0), C.c_int(0)
    rc = emul.emul_gpu_decode_checked(data, C.c_size_t(len(data)), subseq, max_rounds, out.ctypes.data_as(C.c_void_p), C.c_longlong(out.size),
                                      C.byref(r), C.byref(a))
    anomalies.append(a.value)
    return rc, out, r.value


def scan_bounds(data):
    """(first byte of the entropy-coded segment, position of the EOI that ends it)"""
    sos = data.index(b"\xff\xda")
    return sos + 2 + int.from_bytes(data[sos + 2:sos + 4], "big"), data.rindex(EOI)


def cut(data, at, eoi=True):
    return data[:at] + (EOI if eoi else b"")


def editable(data, i):
    """a scan byte that can change without creating or destroying a marker or a stuffed zero"""
    return data[i] != 0xFF and data[i - 1] != 0xFF


def bit_flips(data, n, seed):
    start, end = scan_bounds(data)
    rng, out = random.Random(seed), []
    while len(out) < n:
        i = rng.randrange(start, end)
        v = data[i] ^ (1 << rng.randrange(8))
        if editable(data, i) and v != 0xFF:
            out.append(data[:i] + bytes([v]) + data[i + 1:])
    return out


def byte_replacements(data, n, seed):
    start, end = scan_bounds(data)
    rng, out = random.Random(seed), []
    while len(out) < n:
        i = rng.randrange(start, end)
        v = rng.randrange(0xFF)
        if editable(data, i) and v != data[i]:
            out.append(data[:i] + bytes([v]) + data[i + 1:])
    return out


def cuts(data, n_tail, n_random, seed):
    """cuts in the last n_tail bytes of the scan plus n_random seeded cuts anywhere in it, each with and without an EOI"""
    start, end = scan_bounds(data)
    at = set(range(max(start + 1, end - n_tail), end + 1))
    rng = random.Random(seed)
    at |= {rng.randrange(start + 1, end) for _ in range(n_random)}
    return [cut(data, a, eoi) for a in sorted(at) for eoi in (True, False)]


def synth_file(w, h, seed, **kw):
    from tools.synth import synth_rgb
    b = io.BytesIO()
    Image.fromarray(synth_rgb(w, h, seed), "RGB").save(b, "JPEG", **kw)
    return b.getvalue()


def synth_gray(w, h, seed, **kw):
    from tools.synth import synth_rgb
    b = io.BytesIO()
    Image.fromarray(synth_rgb(w, h, seed)[:, :, 1], "L").save(b, "JPEG", **kw)
    return b.getvalue()


def synth_440(L, w, h, seed):
    """A baseline 4:4:0 file (luma 1x2, which Pillow does not write): seeded coefficients entropy-coded by the host encoder."""
    lay, _ = L.jpeg_decode_coefficients(synth_file(w, h, seed, quality=85, subsampling="4:4:4"))
    lay.hs[0], lay.vs[0] = 1, 2
    mcux, mcuy = -(-w // 8), -(-h // 16)
    ch = -(-h // 2)
    geo = [(mcux, 2 * mcuy, -(-w // 8), -(-h // 8))] + [(mcux, mcuy, -(-w // 8), -(-ch // 8))] * 2
    rng, parts, off = np.random.default_rng(seed), [], 0
    for c, (bw, bh, rbw, rbh) in enumerate(geo):
        lay.bw[c], lay.bh[c], lay.rbw[c], lay.rbh[c], lay.comp_offset[c] = bw, bh, rbw, rbh, off
        blk = np.zeros((bh, bw, 64), np.int16)
        blk[:, :, 0] = rng.integers(-60, 61, (bh, bw))
        blk[:, :, 1:12] = rng.integers(-7, 8, (bh, bw, 11))
        parts.append(blk.reshape(-1))
        off += bw * bh * 64
    lay.total_coefs = off
    return L.jpeg_encode_coefficients(lay, np.concatenate(parts), False)


def host_coefficients(L, data):
    try:
        return L.jpeg_decode_coefficients(data)[1]
    except L.B200Error:
        return None


class Tally:
    """what the emulator answered over a set of damaged files"""

    def __init__(self):
        self.n = self.settled = self.host_failed = 0
        self.rules = 0

    def check(self, L, emul, data, total_coefs, subseq):
        ref = host_coefficients(L, data)
        fired = []
        rc, out, _ = emul_decode(emul, data, total_coefs, subseq, 256, fired)
        self.n += 1
        self.rules |= fired[0]
        if ref is None:
            self.host_failed += 1
            assert rc != 0, "the host decoder refuses the file, the device decoder reports it decoded"
        if rc == 0:
            assert ref is not None and np.array_equal(out, ref), "the device decoder reports success with other coefficients"
            self.settled += 1
        if rc == 14:
            assert fired[0] and not fired[0] & ~(ANOM_CODE | ANOM_RUN | ANOM_END)
        else:
            assert fired[0] == 0


def total_coefs(L, data):
    return L.jpeg_decode_coefficients(data)[0].total_coefs


# ---------------------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("subseq", SUBSEQ)
@pytest.mark.parametrize("name", ["in_420_tiny_17x9.jpg", "in_420_tiny_3x3.jpg"])
def test_every_cut_of_a_tiny_scan(L, emul, golden, name, subseq):
    data = golden(name)
    start, end = scan_bounds(data)
    t = Tally()
    for d in cuts(data, end - start, 0, 0):
        t.check(L, emul, d, total_coefs(L, data), subseq)
    assert t.rules & ANOM_END
    assert t.settled >= 1           # the cut at the scan's end is the clean file


@pytest.mark.parametrize("subseq", SUBSEQ)
@pytest.mark.parametrize("name", BASE_355)
def test_cuts_of_the_355x237_files(L, emul, golden, name, subseq):
    data = golden(name)
    t = Tally()
    for d in cuts(data, 300, 200, 7):
        t.check(L, emul, d, total_coefs(L, data), subseq)
    assert t.rules & ANOM_END
    assert t.settled >= 1


@pytest.mark.parametrize("subseq", SUBSEQ)
@pytest.mark.parametrize("name", BASE_355 + ["in_420_base_640x480.jpg"])
def test_bit_flips_and_replaced_bytes(L, emul, golden, name, subseq):
    data = golden(name)
    t = Tally()
    for d in bit_flips(data, 120, 11) + byte_replacements(data, 40, 12):
        t.check(L, emul, d, total_coefs(L, data), subseq)
    # not vacuous: many damaged files still decode (and must equal the host's coefficients), others are sent to the host
    assert t.settled >= t.n // 5, (t.settled, t.n)
    assert t.rules & (ANOM_CODE | ANOM_RUN)


def _long_code_files():
    return [("q100", dict(quality=100)), ("opt30", dict(quality=30, optimize=True)), ("opt95_444", dict(quality=95, optimize=True, subsampling="4:4:4"))]


@pytest.mark.parametrize("subseq", SUBSEQ)
@pytest.mark.parametrize("kind,kw", _long_code_files(), ids=[k for k, _ in _long_code_files()])
def test_damaged_files_with_optimised_tables_and_16_bit_codes(L, emul, subseq, kind, kw):
    data = synth_file(171, 113, 5, **kw)
    t = Tally()
    for d in cuts(data, 60, 40, 3) + bit_flips(data, 80, 13) + byte_replacements(data, 30, 14):
        t.check(L, emul, d, total_coefs(L, data), subseq)
    assert t.settled >= t.n // 10, (t.settled, t.n)
    assert t.rules & ANOM_END


def test_every_rule_fires(L, emul, golden):
    """Each of the three rules is met on the damaged set, and each one alone is enough to send the image to the host."""
    seen = {}
    data = golden("in_420_base_640x480.jpg")
    n = total_coefs(L, data)
    start, end = scan_bounds(data)
    for d in [cut(data, start + (end - start) * f // 100) for f in (50, 80, 97)] + bit_flips(data, 400, 21):
        fired = []
        rc, _, _ = emul_decode(emul, d, n, 2048, 64, fired)
        if rc == 14 and fired[0] in (ANOM_CODE, ANOM_RUN, ANOM_END):
            seen.setdefault(fired[0], d)
    assert set(seen) == {ANOM_CODE, ANOM_RUN, ANOM_END}, seen.keys()
    # the invalid-code file is one the host refuses; the others it decodes with coefficients the device would have got wrong
    assert host_coefficients(L, seen[ANOM_CODE]) is None
    for rule in (ANOM_RUN, ANOM_END):
        assert host_coefficients(L, seen[rule]) is not None


def test_truncations_of_the_640x480_file_go_to_the_host(L, emul, golden):
    """The three cuts that showed the difference: the host decodes every block with zero bits past the end, the device
    decoder must not claim those coefficients."""
    data = golden("in_420_base_640x480.jpg")
    start, end = scan_bounds(data)
    for f in (50, 80, 97):
        d = cut(data, start + (end - start) * f // 100)
        ref = host_coefficients(L, d)
        assert ref is not None
        for subseq in (128, 2048):
            fired = []
            rc, _, _ = emul_decode(emul, d, ref.size, subseq, 256, fired)
            assert rc == 14 and fired[0] & ANOM_END, (f, subseq, rc, fired)


def _host_transcode_set(golden):
    out = []
    for name in ("in_420_base_355x237.jpg", "in_444_base_355x237.jpg", "in_420_tiny_17x9.jpg"):
        data = golden(name)
        start, end = scan_bounds(data)
        out += [cut(data, start + (end - start) * f // 100, eoi) for f in (0, 1, 30, 50, 80, 97, 100) for eoi in (True, False)]
        out += bit_flips(data, 25, 31) + byte_replacements(data, 10, 32)
    return out


def test_host_transcode_of_damaged_files_matches_oracle(L, O, golden):
    """The reference the device defers to: the host decoder's answer on damaged files is the oracle's (same file, or both refuse)."""
    p = L.default_params()
    p.jpeg_optimize = 1
    L.set_entropy_mode(0)
    try:
        ok = failed = 0
        for d in _host_transcode_set(golden):
            try:
                want = O.jpeg_lossless(d, O.params(80, 0, True))
            except O.OracleError:
                want = None
            try:
                got = L.compress_in_memory(d, p)
            except L.B200Error as e:
                assert e.code == L.ERR_CORRUPT_INPUT
                got = None
            assert got == want
            ok += got is not None
            failed += got is None
        assert ok > 0 and failed > 0
    finally:
        L.set_entropy_mode(3)


# ---------------------------------------------------------------------------------------------------------------- GPU
def _jparams(L, q=80, ss=420, prog=True, lossless=False):
    p = L.default_params()
    p.jpeg_quality, p.jpeg_chroma_subsampling, p.jpeg_progressive, p.jpeg_optimize = q, ss, int(prog), int(lossless)
    return p


def _answer(fn):
    try:
        return fn()
    except Exception as e:          # B200Error / OracleError: compared by kind below
        return type(e).__name__ + ":" + str(getattr(e, "code", ""))


def _damaged_set(golden):
    out = []
    for name in ("in_420_base_640x480.jpg", "in_444_base_355x237.jpg", "in_gray_base_355x237.jpg"):
        data = golden(name)
        start, end = scan_bounds(data)
        out += [cut(data, start + (end - start) * f // 100) for f in (50, 80, 97)]
        out += bit_flips(data, 12, 41) + byte_replacements(data, 4, 42)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("lossless", [False, True])
def test_damaged_files_same_answer_in_every_entropy_mode(L, O, golden, lossless):
    p = _jparams(L, 80, 0 if lossless else 420, True, lossless)
    po = O.params(80, 0 if lossless else 420, True)
    ref_fn = O.jpeg_lossless if lossless else O.jpeg_lossy
    settled = 0
    try:
        for i, d in enumerate(_damaged_set(golden)):
            answers = []
            for mode in (3, 2, 1, 0):
                L.set_entropy_mode(mode)
                try:
                    answers.append(L.compress_in_memory(d, p))
                except L.B200Error as e:
                    answers.append(e.code)
            assert all(a == answers[0] for a in answers), (i, [a if isinstance(a, int) else len(a) for a in answers])
            try:
                want = ref_fn(d, po)
            except O.OracleError:
                want = None
            if isinstance(answers[0], bytes):
                assert answers[0] == want, i
                settled += 1
            else:
                assert answers[0] == L.ERR_CORRUPT_INPUT and want is None, i
        assert settled > 0
    finally:
        L.set_entropy_mode(3)


@pytest.mark.gpu
@pytest.mark.parametrize("lossless", [False, True])
def test_batch_with_damaged_files_matches_single_calls(L, golden, lossless):
    """b200_compress_batch walks the segments of same-shaped files on the device (megabatch path): damaged files among clean
    ones of the same shape come out exactly as the single call answers them, and the clean ones are unaffected."""
    L.set_entropy_mode(3)
    clean = golden("in_420_base_640x480.jpg")
    start, end = scan_bounds(clean)
    damaged = [cut(clean, start + (end - start) * f // 100) for f in (50, 80, 97)] + bit_flips(clean, 10, 51) + byte_replacements(clean, 4, 52)
    work = []
    for d in damaged:
        work += [clean, d]
    work += [clean] * 3
    p = _jparams(L, 80, 0 if lossless else 420, True, lossless)
    single = {}
    for d in set(work):
        try:
            single[d] = (L.compress_in_memory(d, p), 0)
        except L.B200Error as e:
            single[d] = (None, e.code)
    for i, (out, code, msg) in enumerate(L.compress_batch(work, p, n_threads=4)):
        assert (out, code) == single[work[i]], (i, code, msg)


def _clean_sweep(L, golden):
    files ={n: golden(n) for n in ("in_420_base_355x237.jpg", "in_444_base_355x237.jpg", "in_422_base_355x237.jpg", "in_gray_base_355x237.jpg",
                                    "in_420_base_640x480.jpg", "in_420_tiny_17x9.jpg", "in_420_tiny_3x3.jpg")}
    for w, h in ((1, 1), (8, 8), (16, 16), (17, 9)):
        files[f"synth_{w}x{h}"] = synth_file(w, h, w + h, quality=90)
    files["synth_422"] = synth_file(77, 41, 3, quality=85, subsampling="4:2:2")
    files["synth_440"] = synth_440(L, 53, 37, 4)
    files["synth_gray"] = synth_gray(61, 45, 5, quality=85)
    files["synth_opt30"] = synth_file(211, 133, 6, quality=30, optimize=True)
    files["synth_opt95_444"] = synth_file(133, 97, 7, quality=95, optimize=True, subsampling="4:4:4")
    files["synth_q100"] = synth_file(129, 65, 8, quality=100)
    files["synth_gray_q100"] = synth_gray(64, 40, 9, quality=100)
    return files


@pytest.mark.gpu
@pytest.mark.parametrize("lossless", [False, True])
def test_resident_pipe_decodes_every_clean_shape_on_the_device(L, O, golden, lossless):
    """The resident pipe has no host fallback: not_settled counts the images the device decoder handed back.  Every clean file
    -- odd sizes, every subsampling, gray, optimised tables, q=100 -- must be decoded on the device and come out as the oracle's."""
    import torch
    assert L.lib().b200_init_device(0) == 0
    p = _jparams(L, 80, 0 if lossless else 420, True, lossless)
    po = O.params(80, 0 if lossless else 420, True)
    st = torch.cuda.Stream()
    for name, data in _clean_sweep(L, golden).items():
        want = (O.jpeg_lossless if lossless else O.jpeg_lossy)(data, po)
        pipe = L.JpegPipe([data] * 3, p, group=2)
        try:
            pipe.run(st.cuda_stream)
            torch.cuda.synchronize()
            _, not_settled, _ = pipe.finish()
            assert not_settled == 0, name
            for i in range(3):
                assert pipe.fetch(i) == want, (name, i)
        finally:
            pipe.close()


@pytest.mark.gpu
def test_resident_pipe_counts_the_damaged_files(L, O, golden):
    """A pipe of one shape holding damaged files (truncated, EOI appended) reports exactly those as not settled; the clean
    files between them still come out as the oracle's."""
    import torch
    assert L.lib().b200_init_device(0) == 0
    clean = golden("in_420_base_640x480.jpg")
    start, end = scan_bounds(clean)
    damaged = []
    for f in (30, 50, 80, 97):
        at = start + (end - start) * f // 100
        while clean[at - 1] == 0xFF:
            at += 1
        damaged.append(cut(clean, at))
    work = [clean, damaged[0], damaged[1], clean, damaged[2], clean, damaged[3]]
    p = _jparams(L)
    want = O.jpeg_lossy(clean, O.params(80, 420, True))
    st = torch.cuda.Stream()
    for group in (3, 8):
        pipe = L.JpegPipe(work, p, group=group)
        try:
            pipe.run(st.cuda_stream)
            torch.cuda.synchronize()
            _, not_settled, _ = pipe.finish()
            assert not_settled == len(damaged), group
            for i in (0, 3, 5):
                assert pipe.fetch(i) == want, (group, i)
        finally:
            pipe.close()
