"""Device JPEG decoder on scans dense in stuffed bytes (tests/stuffed_jpeg.py), on every route into it: single calls, megabatches
(b200_compress_batch, where the un-stuff kernels also find markers and the stream's true length) and the resident pipe.

The reference of every output is the oracle's file, and for lossless outputs also the coefficients the file was written from.
A megabatch member the device decoder does not settle goes quietly to the per-image path and still comes out right, so the
megabatch's rescue count (printed at exit with B200_TRACE) is checked too: 0 on the dense files that settle, more than 0 on a
file with a stray RST marker in its scan.

CPU part: the corpus itself -- its stuffing density, the host decoder's round trip, and which files the decoder's serial emulation
settles within GpuDecoder::ROUNDS at the product's subsequence size (only those are used where settling is asserted on the GPU)."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import stuffed_jpeg as S
from test_gpudec import emul, emul_decode  # noqa: F401  (module fixture: the serial CPU run of the decoder's passes)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ROUNDS, SUBSEQ_BITS = 24, 2048          # GpuDecoder::ROUNDS, GpuDecoder::SUBSEQ_BITS
GOLDEN_355 = {"420": "in_420_base_355x237.jpg", "444": "in_444_base_355x237.jpg", "422": "in_422_base_355x237.jpg", "grey": "in_gray_base_355x237.jpg"}


@pytest.fixture(scope="module")
def dense(L):
    return S.dense_corpus(L)


@pytest.fixture(scope="module")
def settles(dense, emul):  # noqa: F811
    """names of the files the decoder's emulation settles within the product's round budget"""
    out = set()
    for name, (data, lay, co) in dense.items():
        rc, got, _ = emul_decode(emul, data, lay.total_coefs, SUBSEQ_BITS, ROUNDS)
        if rc == 0:
            assert np.array_equal(got, co), name
            out.add(name)
    return out


def stray_rst(data):
    """the file with an RST0 marker written over two bytes in the middle of its scan"""
    s, e = S.scan_bounds(data)
    i = (s + e) // 2
    while data[i - 1] == 0xFF or data[i] == 0xFF or data[i + 1] in (0x00, 0xFF) or data[i + 2] == 0x00:
        i += 1
    return data[:i] + b"\xff\xd0" + data[i + 2:]


# ---------------------------------------------------------------------------------------------------------------- CPU
def test_dense_corpus(L, dense, settles):
    assert len(dense) == 4 * 4 + 16
    residues = set()
    for name, (data, lay, co) in dense.items():
        s, e = S.scan_bounds(data)
        # a one-block file has too few bytes for the share to settle near the large files' ~21 %
        assert S.stuffing_density(data) >= (0.2 if e - s >= 256 else 0.15), name
        assert np.array_equal(L.jpeg_decode_coefficients(data)[1], co), name
        if name.startswith("420_355x237_len_mod16_"):
            residues.add((e - s) % 16)
    assert residues == set(range(16))
    assert max(e - s for s, e in (S.scan_bounds(d) for d, _, _ in dense.values())) >= 64 * 1024
    # most settle; the 4:2:0 files at 355x237 and 640x480 with these seeds need more rounds and go to the host decoder
    assert {f"{k}_{w}x{h}" for k in S.KINDS for w, h in S.SHAPES} - settles <= {"420_355x237", "420_640x480"}
    assert {f"420_355x237_len_mod16_{r}" for r in range(16)} <= settles
    for name in ("444_355x237", "grey_640x480"):
        data, lay, co = dense[name]
        for v in (S.with_fill(data, 1), S.with_fill(data, 5), S.with_trailer(data)):
            assert np.array_equal(L.jpeg_decode_coefficients(v)[1], co), name


# ---------------------------------------------------------------------------------------------------------------- GPU
def jparams(L, lossless, q=80, ss=420, prog=True):
    p = L.default_params()
    p.jpeg_quality, p.jpeg_chroma_subsampling, p.jpeg_progressive, p.jpeg_optimize = q, ss, int(prog), int(lossless)
    return p


def oracle(O, data, lossless):
    return O.jpeg_lossless(data, O.params(80, 420, True)) if lossless else O.jpeg_lossy(data, O.params(80, 420, True))


def single(L, data, lossless):
    try:
        return L.compress_in_memory(data, jparams(L, lossless)), 0
    except L.B200Error as e:
        return None, e.code


@pytest.mark.gpu
@pytest.mark.parametrize("lossless", [True, False], ids=["lossless", "lossy"])
def test_single_calls_equal_oracle(L, O, dense, lossless):
    L.set_entropy_mode(3)
    for name, (data, lay, co) in dense.items():
        out = L.compress_in_memory(data, jparams(L, lossless))
        assert out == oracle(O, data, lossless), name
        if lossless:
            assert S.same_coefficients(L, out, lay, co), name


def megabatch_sets(dense, golden):
    """same-shaped groups: dense 355x237 files of a kind next to the golden file of that kind"""
    sets = []
    for kind in S.KINDS:
        ds = [dense[n][0] for n in dense if n.startswith(f"{kind}_355x237")]
        sets.append(ds[:4] + [golden(GOLDEN_355[kind])] + ds[4:8] + [golden(GOLDEN_355[kind])])
    return sets


@pytest.mark.gpu
@pytest.mark.parametrize("lossless", [True, False], ids=["lossless", "lossy"])
def test_megabatches_equal_single_calls_and_oracle(L, O, monkeypatch, dense, golden, lossless):
    """Groups of 2, 3 and 8 on the verify path (lossy: with the deferred DC of the transform), on 1 and 4 threads."""
    L.set_entropy_mode(3)
    p = jparams(L, lossless)
    for datas in megabatch_sets(dense, golden):
        want = [single(L, d, lossless) for d in datas]
        for d, w in zip(datas, want):
            assert w == (oracle(O, d, lossless), 0)
        for K in (2, 3, 8):
            monkeypatch.setenv("B200_MEGABATCH", str(K))
            for nt in (1, 4):
                res = L.compress_batch(datas, p, n_threads=nt)
                for i, (out, code, msg) in enumerate(res):
                    assert (out, code) == want[i], (i, K, nt, msg)


@pytest.mark.gpu
@pytest.mark.parametrize("lossless", [True, False], ids=["lossless", "lossy"])
def test_long_scans_then_short_ones_on_one_thread(L, O, monkeypatch, dense, golden, lossless):
    """One slot, one shape, one group size: the dense files' long scans set the decoder's high-water sizes, the golden files' short
    scans then run in the same buffers (stale bytes and counts behind them) and, with graphs, replay the captured sequence."""
    L.set_entropy_mode(3)
    monkeypatch.setenv("B200_MEGABATCH", "4")
    p = jparams(L, lossless)
    longs = [dense[f"420_355x237_len_mod16_{r}"][0] for r in range(8)]
    shorts = [golden(GOLDEN_355["420"])] * 4
    for datas in (longs, shorts, longs[:4], shorts):
        res = L.compress_batch(datas, p, n_threads=1)
        for d, (out, code, msg) in zip(datas, res):
            assert code == 0, msg
            assert out == oracle(O, d, lossless)


@pytest.mark.gpu
@pytest.mark.parametrize("lossless", [True, False], ids=["lossless", "lossy"])
@pytest.mark.parametrize("group", [3, 8])
def test_resident_pipe_settles_dense_files(L, O, dense, settles, group, lossless):
    import torch
    assert L.lib().b200_init_device(0) == 0
    names = sorted(n for n in settles if n.startswith("420_355x237_len_mod16_"))[:9] + ["420_355x237_len_mod16_0"]
    datas = [dense[n][0] for n in names]
    want = [oracle(O, d, lossless) for d in datas]
    pipe = L.JpegPipe(datas, jparams(L, lossless), group=group)
    st = torch.cuda.Stream()
    try:
        for rep in range(2):
            pipe.run(st.cuda_stream)
            torch.cuda.synchronize()
            sizes, not_settled, _ = pipe.finish()
            assert not_settled == 0
            for i in range(len(datas)):
                assert pipe.fetch(i) == want[i], (rep, names[i])
    finally:
        pipe.close()


@pytest.mark.gpu
@pytest.mark.parametrize("lossless", [True, False], ids=["lossless", "lossy"])
def test_fill_bytes_and_trailers_agree_on_every_route(L, O, monkeypatch, dense, lossless):
    """One fill byte before the EOI, several, and bytes after the EOI: whatever route each file takes, the single call, the
    megabatch and the pipe give the same file, and a lossless output holds the source's coefficients."""
    import torch
    L.set_entropy_mode(3)
    monkeypatch.setenv("B200_MEGABATCH", "8")
    p = jparams(L, lossless)
    base = [dense[f"420_355x237_len_mod16_{r}"] for r in range(3)]
    variants = {"one_fill": lambda d: S.with_fill(d, 1), "five_fill": lambda d: S.with_fill(d, 5), "trailer": S.with_trailer}
    datas, coefs, kinds = [], [], []
    for data, _, co in base:
        for kind, make in variants.items():
            datas.append(make(data))
            coefs.append(co)
            kinds.append(kind)
    want = [single(L, d, lossless) for d in datas]
    for d, co, (out, code) in zip(datas, coefs, want):
        assert code == 0 and out == oracle(O, d, lossless)
        if lossless:
            assert S.same_coefficients(L, out, base[0][1], co)
    for nt in (1, 4):
        res = L.compress_batch(datas, p, n_threads=nt)
        assert [(o, c) for o, c, _ in res] == want
    # the pipe takes only files whose scan the host walk ends at an EOI; it may refuse fill bytes, and must take the trailer
    assert L.lib().b200_init_device(0) == 0
    st = torch.cuda.Stream()
    taken = set()
    for kind in variants:
        idx = [i for i, k in enumerate(kinds) if k == kind]
        try:
            pipe = L.JpegPipe([datas[i] for i in idx], p, group=3)
        except L.B200Error:
            continue
        taken.add(kind)
        try:
            pipe.run(st.cuda_stream)
            torch.cuda.synchronize()
            _, not_settled, _ = pipe.finish()
            assert not_settled == 0, kind
            for j, i in enumerate(idx):
                assert pipe.fetch(j) == want[i][0], (kind, i)
        finally:
            pipe.close()
    assert "trailer" in taken


_CHILD = """
import os, sys
sys.path.insert(0, {tests!r}); sys.path.insert(0, {root!r})
from conftest import _import_pkg
_import_pkg()
import caesium_clt_b200._lib as L
from oracle import oracle as O
import stuffed_jpeg as S
import test_gpudec_unstuff_gpu as T
assert L.lib().b200_init_device(0) == 0
L.set_entropy_mode(3)
dense = S.dense_corpus(L)
datas = [dense[f"420_355x237_len_mod16_{{r}}"][0] for r in range(8)]
if {stray!r}:
    datas[3] = T.stray_rst(datas[3])
for lossless in (True, False):
    for d, (out, code, msg) in zip(datas, L.compress_batch(datas, T.jparams(L, lossless), n_threads=2)):
        if code == 0:
            assert out == T.oracle(O, d, lossless)
print("ok")
"""


def rescued(stray):
    env = dict(os.environ, B200_TRACE="1", B200_MEGABATCH="8")
    r = subprocess.run([sys.executable, "-c", _CHILD.format(tests=os.path.join(ROOT, "tests"), root=ROOT, stray=stray)], env=env,
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    assert r.stdout.strip().endswith("ok")
    m = re.search(r"\[b200 trace\] megabatch: (\d+) members, (\d+) left to the per-image path", r.stderr)
    assert m, r.stderr[-2000:]
    return int(m.group(1)), int(m.group(2))


@pytest.mark.gpu
def test_megabatch_rescue_count(dense, settles):
    """0 for dense files that settle (the 4:2:0 355x237 files with seed 77, all of which the emulation settles); more than 0 when
    one member has a stray RST0 in its scan, which the un-stuff pass flags -- the counter counts."""
    assert {f"420_355x237_len_mod16_{r}" for r in range(16)} <= settles
    members, left = rescued(False)
    assert members == 16 and left == 0
    members, left = rescued(True)
    assert members == 16 and left >= 2
