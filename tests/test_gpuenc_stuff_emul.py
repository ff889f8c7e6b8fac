"""Device JPEG encoder, byte stuffing: the kernels k_ge_ffcount / k_ge_layout / k_ge_scatter against the plain loop of the
sequential writer (byte i of the scan's words, big-endian; the padding ones in the last byte; a 0x00 after every 0xFF), on CPU.

The kernels' per-thread bodies (jpeg_gpuenc_stuff_core.h) run serially over whole megabatches laid out the way the encoder lays
them out (tests/emul/stuff_emul.cpp): every scan's words 16-byte aligned with garbage behind them, a scan's 16-byte groups cut into
tiles of one group per thread and the tiles into chunks of one CTA each, an 0xFF count per chunk, each image's scans laid out back
to back in its output region, and CTAs that stuff a tile at a time into a shared buffer and store whole words in the middle and
single bytes at the ends of each tile's range.  The tile and chunk counts are small here, so that a test scan spans many chunks,
and the kernels' own (128 groups a tile, 32 chunks a scan) run too.  Every output byte, the offsets and lengths, the overflow flags
and the canary bytes around and behind each image's scans are checked."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMUL_DIR = os.path.join(ROOT, "tests", "emul")
KERNEL_TILE, KERNEL_CHUNKS = 128, 32    # STUFF_THREADS, STUFF_CHUNKS in jpeg_gpuenc.cu
SHAPES = [(4, 3), (8, 5), (1, 1), (KERNEL_TILE, KERNEL_CHUNKS)]   # (groups per tile, chunks per scan)
SPI = 8                                 # scans per image in the batches
CANARY = 0xA5                           # what the emulator leaves in output bytes no pass writes
FAULTS = {"no_padding": 1, "no_clear": 2, "whole_edge_words": 3, "chunk_prefix": 4, "no_tile_carry": 5}
ST_TILES, ST_FIRST_MOD4, ST_END_MOD4, ST_DOUBLE, ST_STRAY, ST_N = 0, 1, 5, 9, 10, 11


@pytest.fixture(scope="module")
def emul():
    so = os.path.join(EMUL_DIR, "libstuff_emul.so")
    srcs = [os.path.join(EMUL_DIR, "stuff_emul.cpp"), os.path.join(ROOT, "caesium-clt_b200", "csrc", "jpeg_gpuenc_stuff_core.h"),
            os.path.join(ROOT, "caesium-clt_b200", "csrc", "jpeg_gpuenc_core.h")]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-msse2", "-Wno-unknown-pragmas", "-o", so, srcs[0]])
    return C.CDLL(so)


# ---- the reference -------------------------------------------------------------------------------------------------------------
def reference(words, total_bits):
    """gpuenc_emul.cpp's pad + stuff loop: byte i of the words (big-endian), the padding ones in the last byte, a 0x00 after every
    0xFF"""
    nbytes = (total_bits + 7) // 8
    d = bytearray(np.asarray(words, np.uint32).astype(">u4").tobytes()[:nbytes])
    if total_bits & 7:
        d[-1] |= (1 << (8 - (total_bits & 7))) - 1
    return bytes(d).replace(b"\xff", b"\xff\x00")


# ---- scans -----------------------------------------------------------------------------------------------------------------------
def scan(content, total_bits=None, tail=0xFF):
    """(words, total_bits) of a scan whose bytes are `content` (total_bits defaults to all of them); the bytes that fill its last
    word are `tail` (0xFF: garbage that must not be counted or stored), the low bits of a partial last byte are left as given"""
    total_bits = 8 * len(content) if total_bits is None else total_bits
    assert (total_bits + 7) // 8 == len(content)
    b = bytes(content) + bytes([tail]) * (-len(content) % 4)
    return np.frombuffer(b, ">u4").astype(np.uint32), total_bits


def noise(rng, n, p_ff):
    """n bytes, 0xFF with probability p_ff, otherwise 00..FE"""
    a = rng.integers(0, 0xFF, n, dtype=np.uint8)
    a[rng.random(n) < p_ff] = 0xFF
    return a


def ff_at(rng, n, positions, p_ff=0.0):
    a = noise(rng, n, p_ff)
    a[[p for p in positions if p < n]] = 0xFF
    return a


def corpus(tile, nchunks):
    """(tag, scan) pairs; the tags name what the case was built to hit"""
    rng = np.random.default_rng(tile * 1000 + nchunks)
    tb, cb = 16 * tile, 16 * tile * nchunks             # bytes of a tile; of a scan of nchunks tiles, one tile a chunk
    cases = [("empty", scan(b""))]
    cases += [(f"bits_{k}", scan(noise(rng, 1, 0.5), k)) for k in range(1, 8)]
    cases += [(f"bytes_{n}", scan(noise(rng, n, 0.2))) for n in (1, 15, 16, 17, 31, 32, 33)]
    cases += [(f"short_of_{what}", scan(noise(rng, n, 0.1))) for what, n in (("a_group", 15), ("a_tile", tb - 1), ("a_chunk", cb - 1),
                                                                            ("two_chunks", 2 * cb - 1), ("three_tiles_a_chunk", 3 * cb - 1))]
    cases += [("all_ff", scan(np.full(n, 0xFF, np.uint8), 8 * n - k)) for n, k in ((5, 0), (tb, 3), (2 * cb + 7, 0), (3 * cb, 1))]
    for k in range(1, 8):                               # a last byte that the padding ones make an 0xFF, at every partial length
        c = noise(rng, 2 * tb + 3, 0.05)
        c[-1] = (0xFF << (8 - k)) & 0xFF
        cases.append(("padding_makes_ff", scan(c, 8 * len(c) - 8 + k)))
        c = noise(rng, 16 * k + 1, 0.05)
        c[-1] = 0x00
        cases.append(("padding_without_ff", scan(c, 8 * len(c) - 8 + k, tail=0x00)))
    for p in range(16):                                 # an 0xFF at every position of a group, in the first and in a middle group
        cases.append((f"ff_at_group_pos_{p}", scan(ff_at(rng, 3 * tb + 5, [p, 16 * 5 + p]))))
    edges = sorted({e + d for e in range(tb, 4 * cb, tb) for d in (-1, 0, 1)})
    cases.append(("ff_at_tile_and_chunk_edges", scan(ff_at(rng, 4 * cb + 9, edges))))
    cases.append(("ff_at_tile_and_chunk_edges_dense", scan(ff_at(rng, 4 * cb + 9, edges, 0.3))))
    for p_ff in (0.004, 0.05, 0.5, 0.97):
        for n in (int(rng.integers(1, 3 * cb)), 5 * cb + int(rng.integers(0, tb))):
            cases.append((f"random_{p_ff}", scan(noise(rng, n, p_ff), 8 * n - int(rng.integers(0, 8)))))
    return cases


def images(cases, rng):
    """the corpus cut into images of SPI scans (shuffled), the last image filled with empty scans"""
    order = list(rng.permutation(len(cases)))
    order += [None] * (-len(order) % SPI)
    return [[cases[j] if j is not None else ("empty", scan(b"")) for j in order[i:i + SPI]] for i in range(0, len(order), SPI)]


# ---- the run -----------------------------------------------------------------------------------------------------------------------
def run_batch(emul, imgs, tile, nchunks, stride=None, fault=0, seed=0):
    scans = [s for im in imgs for _, s in im]
    tbits = np.array([t for _, t in scans], np.uint32)
    words = np.concatenate([w for w, _ in scans] + [np.zeros(1, np.uint32)])
    refs = [reference(w, t) for w, t in scans]
    if stride is None:
        stride = max(sum(len(r) for r in refs[i:i + SPI]) for i in range(0, len(refs), SPI)) + 64
    stride = -(-stride // 4) * 4
    n = len(imgs)
    out = np.zeros(n * stride, np.uint8)
    off, length = np.zeros(n * SPI, np.uint32), np.zeros(n * SPI, np.uint32)
    flags, stats = np.zeros(8, np.uint32), np.zeros(ST_N, np.int64)
    ptr = lambda a: a.ctypes.data_as(C.c_void_p)
    rc = emul.emul_stuff_batch(n, SPI, ptr(tbits), ptr(words), nchunks, tile, C.c_uint32(stride), fault, C.c_uint64(seed),
                               ptr(out), ptr(off), ptr(length), ptr(flags), ptr(stats))
    assert rc == 0
    return refs, stride, out.tobytes(), off, length, flags, stats


def check_batch(emul, imgs, tile, nchunks, stride=None, fault=0, seed=0):
    refs, stride, out, off, length, flags, stats = run_batch(emul, imgs, tile, nchunks, stride, fault, seed)
    totals = [sum(len(r) for r in refs[i:i + SPI]) for i in range(0, len(refs), SPI)]
    assert flags[3] == max(totals)
    assert flags[4] == (max(totals) > stride)
    assert [int(x) for x in length] == [len(r) for r in refs]
    if flags[4]:
        assert out == bytes([CANARY]) * len(out), "an image outgrew its region, yet something was written"
        return stats
    assert stats[ST_DOUBLE] == 0, "an output byte was written twice"
    assert stats[ST_STRAY] == 0, "a byte outside its scan's output range was written"
    for i in range(len(imgs)):
        region, at = out[i * stride:(i + 1) * stride], 0
        for k in range(SPI):
            si = i * SPI + k
            what = f"image {i}, scan {k}: {imgs[i][k][0]}, {len(refs[si])} stuffed bytes, tile {tile}, {nchunks} chunks"
            assert off[si] == at, what
            assert region[at:at + len(refs[si])] == refs[si], what
            at += len(refs[si])
        assert region[at:] == bytes([CANARY]) * (stride - at), f"image {i}: bytes written behind its scans"
    return stats


@pytest.mark.parametrize("tile,nchunks", SHAPES)
def test_stuffing_equals_the_reference(emul, tile, nchunks):
    """The whole corpus in megabatches of 1..8 images x 8 scans; the tiles' output ranges start and end at every residue mod 4
    (where the edge bytes of a range leave one by one), and scans span every chunk."""
    rng = np.random.default_rng(tile + 7 * nchunks)
    imgs = images(corpus(tile, nchunks), rng)
    hit = np.zeros(ST_N, np.int64)
    i, size = 0, 1
    while i < len(imgs):
        hit += check_batch(emul, imgs[i:i + size], tile, nchunks, seed=i)
        i += size
        size = size % 8 + 1
    if tile * 16 < 2048:
        assert all(hit[ST_FIRST_MOD4 + r] and hit[ST_END_MOD4 + r] for r in range(4))
    longest = max(len(reference(w, t)) for _, (w, t) in corpus(tile, nchunks))
    assert longest > 3 * 16 * tile * nchunks          # the longest scans hold several tiles in every chunk


@pytest.mark.parametrize("tile,nchunks", SHAPES[:2])
def test_an_image_outgrowing_its_region_writes_nothing(emul, tile, nchunks):
    """flags[4] is raised when one image's stuffed scans exceed the region (here: by one byte), and then no byte is written for
    any image; flags[3] is the largest image, which sizes the retry.  At exactly the region's size it fits."""
    rng = np.random.default_rng(5)
    imgs = [[(f"dense_{k}", scan(noise(rng, 300 + 40 * k, 0.5 if i == 1 else 0.01))) for k in range(SPI)] for i in range(3)]
    refs, *_ = run_batch(emul, imgs, tile, nchunks)
    big = sum(len(r) for r in refs[SPI:2 * SPI])
    stats = check_batch(emul, imgs, tile, nchunks, stride=big - 4)
    assert stats[ST_TILES] == 0
    check_batch(emul, imgs, tile, nchunks, stride=big)


@pytest.mark.parametrize("fault", list(FAULTS))
def test_a_wrong_body_would_be_seen(emul, fault):
    """The checks themselves: a stuffing pass without the padding ones, one that counts the garbage past a scan's end, one that
    stores its edge words whole, one that sums the chunks before its own wrongly, or one that loses a byte between tiles fails
    them -- while the same batch passes with the real bodies."""
    rng = np.random.default_rng(11)
    imgs = [[("dense", scan(noise(rng, 16 * 4 * 3 * 4 + 13 * k + 1, 0.2), 8 * (16 * 4 * 3 * 4 + 13 * k + 1) - (k % 8)))
             for k in range(SPI)] for _ in range(2)]
    check_batch(emul, imgs, 4, 3)
    with pytest.raises(AssertionError):
        check_batch(emul, imgs, 4, 3, fault=FAULTS[fault])
    assert reference(np.array([0xFFF80000], np.uint32), 13) == b"\xff\x00\xff\x00"
    assert reference(np.array([0x12FF3400], np.uint32), 24) == b"\x12\xff\x00\x34"
