"""Device JPEG decoder, un-stuffing: the kernels k_gd_unstuff_count / k_gd_unstuff_scatter against the plain reference
raw.replace(b"\\xff\\x00", b"\\xff"), on CPU.

The kernels' per-thread bodies (jpeg_gpudec_core.h) run serially over whole decode batches laid out the way GpuDecoder lays them
out (tests/emul/unstuff_emul.cpp): 16-byte groups, counts scanned over a high-water length with a stale tail, CTAs of 128 threads
that compact their bytes in shared memory at the output's word alignment and store whole words in the middle and single bytes at
the ends of their range.  Every output byte is compared with the reference, the 0xFF padding behind each stream and the bytes
between the images' regions (which no pass may write) are checked, and on the path where the host did not walk the segment the
true length and the marker flag the kernels publish are checked too.  The inputs are byte strings built to put stuffed pairs,
markers and segment ends at the group and CTA boundaries where a compaction of this kind goes wrong."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMUL_DIR = os.path.join(ROOT, "tests", "emul")
THREADS = 128                   # UNSTUFF_THREADS in jpeg_gpudec.cu
CTA_BYTES = THREADS * 16        # raw bytes un-stuffed by one CTA
SUBSEQ_BITS = 2048              # GpuDecoder::SUBSEQ_BITS
CANARY = 0xA5                   # what the emulator leaves in stream bytes no pass writes
ST_CTAS, ST_FIRST_MOD4, ST_END_MOD4, ST_DOUBLE, ST_STRAY, ST_N = 0, 1, 5, 9, 10, 11


@pytest.fixture(scope="module")
def emul():
    so = os.path.join(EMUL_DIR, "libunstuff_emul.so")
    srcs = [os.path.join(EMUL_DIR, "unstuff_emul.cpp"), os.path.join(ROOT, "caesium-clt_b200", "csrc", "jpeg_gpudec_core.h"),
            os.path.join(ROOT, "caesium-clt_b200", "csrc", "jpeg_gpuenc_core.h")]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-msse2", "-Wno-unknown-pragmas", "-o", so, srcs[0]])
    lib = C.CDLL(so)
    lib.emul_unstuff_stream_bytes.restype = C.c_size_t
    return lib


# ---- the reference -------------------------------------------------------------------------------------------------------------
def unstuff(raw):
    return raw.replace(b"\xff\x00", b"\xff")


def has_marker(raw):
    """an 0xFF followed inside the segment by anything but 0x00"""
    a = np.frombuffer(raw, np.uint8)
    return bool(np.any((a[:-1] == 0xFF) & (a[1:] != 0x00)))


# ---- the corpus ------------------------------------------------------------------------------------------------------------------
DENSITIES = {"none": 0.0, "sparse": 0.0076, "dense": 0.143}     # P(a token is FF 00): ~0 %, ~1.5 %, ~25 % of the bytes in pairs


def clean(rng, n, p):
    """n bytes of a segment without markers: bytes 00..FE, and with probability p per token the pair FF 00 instead"""
    pairs = rng.random(n) < p
    vals = rng.integers(0, 0xFF, n, dtype=np.uint8)
    lens = 1 + pairs
    starts = np.cumsum(lens) - lens
    out = np.empty(int(lens.sum()), np.uint8)
    out[starts] = np.where(pairs, 0xFF, vals)
    out[starts[pairs] + 1] = 0
    return out[:n].tobytes()


def put(seg, at, pattern):
    """seg with `pattern` at `at`, and the byte in front of it made plain so that no marker or extra pair appears there"""
    b = bytearray(seg)
    b[at:at + len(pattern)] = pattern
    if at > 0 and b[at - 1] == 0xFF:
        b[at - 1] = 0x11
    end = at + len(pattern)
    if end < len(b) and b[end] == 0x00 and pattern[-1] == 0xFF:
        b[end] = 0x22
    return bytes(b[:len(seg)])


def corpus():
    """(tags, segment) pairs; the tags name what the case was built to hit"""
    rng = np.random.default_rng(2024)
    cases = []
    lengths = [k * CTA_BYTES + d for k in (1, 2, 3) for d in range(-17, 18)]
    for name, p in DENSITIES.items():
        for n in lengths:
            cases.append(({f"density_{name}"}, clean(rng, n, p)))
    for n in lengths[::5] + [1, 2, 15, 16, 17, 31, 32, 33]:
        cases.append(({"density_all_pairs"}, (b"\xff\x00" * n)[:n]))
    for n in range(1, 40):                                   # segments shorter than a few groups, down to one byte
        cases.append(({"short"}, clean(rng, n, 0.3)))
    # a pair at every offset around the first CTA boundary, and split across groups in mid-CTA and late in the third CTA
    for at in range(CTA_BYTES - 8, CTA_BYTES + 9):
        for name in ("none", "dense"):
            cases.append(({f"pair_at_{at}"}, put(clean(rng, 2 * CTA_BYTES + 40, DENSITIES[name]), at, b"\xff\x00")))
    for at in (15, 16 * 37 + 15, 2 * CTA_BYTES + 16 * 70 + 15):
        cases.append(({"pair_split_group"}, put(clean(rng, 3 * CTA_BYTES - 5, DENSITIES["sparse"]), at, b"\xff\x00")))
    # how a segment can end
    for n in (16 * 3 + 5, CTA_BYTES - 1, CTA_BYTES + 2, 2 * CTA_BYTES + 9):
        for name in ("none", "dense"):
            s = clean(rng, n, DENSITIES[name])
            cases.append(({"ends_ff00"}, put(s[:-2] + b"\x11\x11", n - 2, b"\xff\x00")))
            cases.append(({"ends_lone_ff"}, put(s[:-1] + b"\x11", n - 1, b"\xff")))
    for groups in (1, 5, THREADS, THREADS + 3, 2 * THREADS):   # the last group holds only the 00 of a pair (at THREADS: a CTA of it alone)
        for name in ("none", "dense"):
            s = clean(rng, 16 * groups + 1, DENSITIES[name])
            cases.append(({"last_group_only_00"}, put(s, 16 * groups - 1, b"\xff\x00")))
    # markers (and fill) at group and CTA edges, at the segment's end, and between pairs
    for m in (b"\xff\xd0", b"\xff\xd9", b"\xff\xff"):
        for at, edge in ((16 * 9 + 15, "group"), (CTA_BYTES - 1, "cta"), (2 * CTA_BYTES - 1, "cta"), (16 * 3, "mid")):
            for name in ("none", "dense"):
                cases.append(({f"marker_{m[1]:02x}_{edge}"}, put(clean(rng, 2 * CTA_BYTES + 100, DENSITIES[name]), at, m)))
        cases.append(({"marker_at_end"}, put(clean(rng, 16 * 11, DENSITIES["sparse"]), 16 * 11 - 2, m)))
    return cases


def batches(cases, rng):
    """the corpus cut into batches of 1..8 images (the sizes cycle), each batch shuffled; one-byte images go into larger batches"""
    order = list(rng.permutation(len(cases)))
    out, i, size = [], 0, 1
    ones = [({"one_byte"}, bytes([v])) for v in (0x00, 0x7F, 0xFF)]
    while i < len(order):
        b = [cases[j] for j in order[i:i + size]]
        if size >= 3 and ones:
            b.insert(size // 2, ones.pop())
        out.append(b)
        i += size
        size = size % 8 + 1
    return out


# ---- the run -----------------------------------------------------------------------------------------------------------------------
def run_batch(emul, segs, verify, seed):
    n = len(segs)
    lens = np.array([len(s) for s in segs], np.uint32)
    cap = int(emul.emul_unstuff_stream_bytes(n, lens.ctypes.data_as(C.c_void_p))) + 64
    stream = np.zeros(cap, np.uint8)
    ver = np.array(verify, np.int32)
    off, nbits, nsub, mark = (np.zeros(n, np.uint32) for _ in range(4))
    stats = np.zeros(ST_N, np.int64)
    blob = b"".join(segs)
    rc = emul.emul_unstuff_batch(n, blob, lens.ctypes.data_as(C.c_void_p), ver.ctypes.data_as(C.c_void_p), THREADS, SUBSEQ_BITS, C.c_uint64(seed),
                                 stream.ctypes.data_as(C.c_void_p), C.c_size_t(cap), off.ctypes.data_as(C.c_void_p), nbits.ctypes.data_as(C.c_void_p),
                                 nsub.ctypes.data_as(C.c_void_p), mark.ctypes.data_as(C.c_void_p), stats.ctypes.data_as(C.c_void_p))
    assert rc == 0
    return stream.tobytes(), off, nbits, nsub, mark, stats


def check_batch(emul, segs, verify, seed):
    stream, off, nbits, nsub, mark, stats = run_batch(emul, segs, verify, seed)
    assert stats[ST_DOUBLE] == 0, "an output byte was written by two CTAs"
    assert stats[ST_STRAY] == 0, "a byte outside its image's stream region was written"
    ends = list(off[1:]) + [len(stream)]
    for k, raw in enumerate(segs):
        ref = unstuff(raw)
        ns, o = len(ref), int(off[k])
        pad_end = ((ns + 3) & ~3) + 16
        what = f"image {k} of {len(segs)}, {len(raw)} raw bytes, verify={verify[k]}"
        assert o % 16 == 0
        assert stream[o:o + ns] == ref, what
        assert stream[o + ns:o + pad_end] == b"\xff" * (pad_end - ns), what
        assert stream[o + pad_end:ends[k]] == bytes([CANARY]) * (ends[k] - o - pad_end), what
        assert nbits[k] == 8 * ns, what
        assert nsub[k] == -(-8 * ns // SUBSEQ_BITS), what
        assert mark[k] == (verify[k] and has_marker(raw)), what
    return stats


def edges_of(raw):
    """the named edges a segment hits, measured on the bytes rather than taken from how the case was built"""
    a = np.frombuffer(raw, np.uint8)
    n, hit = len(a), set()
    hit.add(f"len_mod16_{n % 16}")
    if CTA_BYTES - 17 <= n % CTA_BYTES or n % CTA_BYTES <= 17:
        hit.add(f"cta_multiple_{n // CTA_BYTES + (n % CTA_BYTES > 17)}_pm17")
    pair = np.flatnonzero((a[:-1] == 0xFF) & (a[1:] == 0x00))       # FF of every stuffed pair
    frac = 2 * len(pair) / max(n, 1)
    if n >= 1024:
        hit.add("density_0" if len(pair) == 0 else "density_1.5pct" if 0.01 <= frac <= 0.02 else "density_25pct" if 0.2 <= frac <= 0.3 else
                "density_all_pairs" if frac > 0.99 else "density_other")
    for p in pair:
        if CTA_BYTES - 8 <= p <= CTA_BYTES + 8:
            hit.add(f"pair_at_{p}")
        if p % 16 == 15:
            hit.add("pair_split_group")
        if p % CTA_BYTES == CTA_BYTES - 1:
            hit.add("pair_split_cta")
    if n >= 2 and raw[-2:] == b"\xff\x00":
        hit.add("ends_ff00")
        if n % 16 == 1:
            hit.add("last_group_only_00")
            if n % CTA_BYTES == 1:
                hit.add("last_cta_only_00")
    if raw[-1:] == b"\xff" and (n < 2 or raw[-2] != 0xFF):
        hit.add("ends_lone_ff")
    if n < 16:
        hit.add("shorter_than_a_group")
    mk = np.flatnonzero((a[:-1] == 0xFF) & (a[1:] != 0x00))
    for p in mk:
        kind = f"{a[p + 1]:02x}"
        if p % 16 == 15:
            hit.add(f"marker_ff{kind}_at_group_edge")
        if p % CTA_BYTES == CTA_BYTES - 1:
            hit.add(f"marker_ff{kind}_at_cta_edge")
    return hit


REQUIRED = ({f"len_mod16_{r}" for r in range(16)} | {f"cta_multiple_{k}_pm17" for k in (1, 2, 3)} |
            {"density_0", "density_1.5pct", "density_25pct", "density_all_pairs"} |
            {f"pair_at_{p}" for p in range(CTA_BYTES - 8, CTA_BYTES + 9)} | {"pair_split_group", "pair_split_cta"} |
            {"ends_ff00", "ends_lone_ff", "last_group_only_00", "last_cta_only_00", "shorter_than_a_group"} |
            {f"marker_ff{k}_at_{e}_edge" for k in ("d0", "d9", "ff") for e in ("group", "cta")} |
            {f"batch_of_{k}" for k in range(1, 9)} | {"one_byte_in_a_batch", "verify_0", "verify_1", "verify_mixed_batch"} |
            {f"cta_first_mod4_{r}" for r in range(4)} | {f"cta_end_mod4_{r}" for r in range(4)})


def run_corpus(emul, mode):
    """every case of the corpus, in batches of 1..8 images; returns the edges the run hit"""
    rng = np.random.default_rng({"host_walked": 1, "device_verified": 2, "mixed": 3}[mode])
    hit = set()
    for bi, b in enumerate(batches(corpus(), rng)):
        segs = [s for _, s in b]
        verify = [0] * len(segs) if mode == "host_walked" else [1] * len(segs) if mode == "device_verified" else [int(x) for x in rng.integers(0, 2, len(segs))]
        stats = check_batch(emul, segs, verify, seed=bi)
        hit.add(f"batch_of_{len(segs)}")
        hit |= {f"verify_{v}" for v in verify}
        if len(set(verify)) == 2:
            hit.add("verify_mixed_batch")
        if len(segs) > 1 and any(len(s) == 1 for s in segs):
            hit.add("one_byte_in_a_batch")
        hit |= {f"cta_first_mod4_{r}" for r in range(4) if stats[ST_FIRST_MOD4 + r]}
        hit |= {f"cta_end_mod4_{r}" for r in range(4) if stats[ST_END_MOD4 + r]}
        for s in segs:
            hit |= edges_of(s)
    return hit


@pytest.mark.parametrize("mode", ["host_walked", "device_verified", "mixed"])
def test_unstuff_batches_equal_the_reference(emul, mode):
    """With the host's walk (verify = 0, the single-call path: the host gives the exact length), without it (verify = 1, the
    megabatch path, where the kernels publish the length and flag markers), and both in one batch."""
    run_corpus(emul, mode)


def test_corpus_hits_every_edge(emul):
    """The corpus really puts stuffed pairs, markers and segment ends at each boundary named in REQUIRED, and the CTAs' output
    ranges really start and end at every residue mod 4 (where the edge bytes of a range leave one by one)."""
    hit = run_corpus(emul, "mixed") | run_corpus(emul, "host_walked")
    missing = REQUIRED - hit
    assert not missing, sorted(missing)


def test_a_wrong_kernel_would_be_seen(emul):
    """The checks themselves: a stream region overrun by one byte, a pair left in place, a wrong length or marker flag fails them."""
    segs = [b"\x12\xff\x00\x34" * 600, b"\xff\xd0" + b"\x00" * 40]
    stream, off, nbits, nsub, mark, _ = run_batch(emul, segs, [1, 1], 0)
    assert stream[int(off[0]):int(off[0]) + 1800] == unstuff(segs[0])[:1800]
    assert mark[0] == 0 and mark[1] == 1
    assert nbits[0] == 8 * 1800 and nsub[0] == -(-8 * 1800 // SUBSEQ_BITS)
    assert unstuff(b"\xff\x00\x00\xff\xff\x00") == b"\xff\x00\xff\xff"
    assert has_marker(b"\x00\xff\xff\x00") and not has_marker(b"\xff\x00\xff") and not has_marker(b"\x01\xff")
