"""Megabatches and the resident pipe over same-shaped JPEGs that differ in everything else (tests/mixed_jpeg.py), run with -m gpu
on an H100.

b200_compress_batch and the resident pipe run K images of one shape through one launch sequence, replayed as CUDA graphs while its
signature (counts, high-water sizes, buffer addresses) holds.  Huffman tables, selectors, dequantisation tables, tq maps,
component ids and marker segments are per image and reach the device through copies the graphs read again on every replay.  Every
output here is compared with the oracle's file and with the single-call answer, with each variant leading a group (the layout and
the output geometry come from a group's first member), at several group sizes and thread counts, with graphs on and off, and in the
resident pipe under the call pattern of bench.py.  The variants' headers are pinned to libjpeg-turbo by
test_megabatch_mixed_host.py."""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

import pytest

from mixed_jpeg import KINDS, variants, pillow

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ARMS = {"q80_420_progressive": (80, 420, True, False), "q60_444_sequential": (60, 444, False, False), "lossless": (80, 0, True, True)}


def jparams(L, q, ss, prog, lossless):
    p = L.default_params()
    p.jpeg_quality, p.jpeg_chroma_subsampling, p.jpeg_progressive, p.jpeg_optimize = q, ss, int(prog), int(lossless)
    return p


def oracle_file(O, data, q, ss, prog, lossless, trellis=False):
    if lossless:
        return O.jpeg_lossless(data, O.params(q, ss, prog))
    if trellis:
        from oracle import jpeg_trellis
        return jpeg_trellis.jpeg_lossy(data, O.params(q, ss, prog))
    return O.jpeg_lossy(data, O.params(q, ss, prog))


def single(L, data, p):
    try:
        return L.compress_in_memory(data, p), 0
    except L.B200Error as e:
        return None, e.code


def batch_inputs(kind):
    """The variants, then inputs no megabatch takes: one that is not an image, a truncated file and a progressive file of the same
    shape, which must answer what a single call answers."""
    vs = variants(kind)
    base = vs[0].data
    return [v.data for v in vs] + [b"not an image", base[:len(base) // 2], pillow(kind, progressive=True)]


def check_rotations(L, O, kind, arm, Ks, threads, trellis=False):
    q, ss, prog, lossless = ARMS[arm]
    p = jparams(L, q, ss, prog, lossless)
    datas = batch_inputs(kind)
    nv = len(variants(kind))
    want = [single(L, d, p) for d in datas]
    for i in range(nv):
        assert want[i] == (oracle_file(O, datas[i], q, ss, prog, lossless, trellis), 0), variants(kind)[i].name
    assert want[nv][1] == L.ERR_UNKNOWN_FORMAT
    for K in Ks:
        os.environ["B200_MEGABATCH"] = str(K)
        for nt in threads:
            for r in range(K):                   # every variant leads a group in one of the K rotations
                order = list(range(r, len(datas))) + list(range(r))
                res = L.compress_batch([datas[i] for i in order], p, n_threads=nt)
                for i, (out, code, msg) in zip(order, res):
                    name = variants(kind)[i].name if i < nv else f"extra input {i - nv}"
                    assert (out, code) == want[i], (name, K, nt, r, msg)


@pytest.mark.parametrize("arm", list(ARMS))
@pytest.mark.parametrize("kind", KINDS)
def test_megabatch_rotations_equal_oracle_and_single_calls(L, O, monkeypatch, kind, arm):
    """Group sizes 2, 3 and 8 over 1 and 4 threads: with one thread, consecutive megabatches of one shape and count run on one slot
    and replay its captured graphs with other images' tables."""
    monkeypatch.setenv("B200_MEGABATCH", "8")
    L.set_entropy_mode(3)
    check_rotations(L, O, kind, arm, (2, 3, 8), (1, 4))


@pytest.mark.parametrize("kind", ["420", "444"])
def test_megabatch_rotations_with_trellis(L, O, monkeypatch, kind):
    monkeypatch.setenv("B200_MEGABATCH", "8")
    L.set_entropy_mode(3)
    assert L.set_jpeg_trellis(1) == 0
    try:
        check_rotations(L, O, kind, "q80_420_progressive", (3, 8), (1, 4), trellis=True)
    finally:
        assert L.set_jpeg_trellis(0) == 0


_CHILD = """
import os, sys
sys.path.insert(0, {tests!r}); sys.path.insert(0, {root!r})
from conftest import _import_pkg
_import_pkg()
import caesium_clt_b200._lib as L
from oracle import oracle as O
import test_megabatch_mixed_gpu as T
assert L.lib().b200_init_device(0) == 0
L.set_entropy_mode(3)
for kind in ("420", "grey"):
    for arm in ("q80_420_progressive", "lossless"):
        T.check_rotations(L, O, kind, arm, (3, 8), (1, 4))
print("ok")
"""


def test_megabatch_rotations_without_graphs():
    """B200_GRAPHS=0 (read once per process, hence a child process): the launch sequence is issued call by call."""
    env = dict(os.environ, B200_GRAPHS="0")
    r = subprocess.run([sys.executable, "-c", _CHILD.format(tests=os.path.join(ROOT, "tests"), root=ROOT)], env=env, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    assert r.stdout.strip().endswith("ok")


# ---- resident pipe -------------------------------------------------------------------------------------------------------------------
def pipe_inputs(kind):
    """The variants the pipe takes (device-decodable files), plus the first one again so that no group size divides the count."""
    vs = [v for v in variants(kind) if v.pipe]
    return vs + vs[:1]


def check_pipe(pipe, vs, want):
    import torch
    torch.cuda.synchronize()
    sizes, not_settled, retries = pipe.finish()
    assert not_settled == sum(not v.settles for v in vs)
    for i, v in enumerate(vs):
        if v.settles:                      # an image the device did not settle is the caller's to re-run (the batch path does so)
            got = pipe.fetch(i)
            assert got == want[i], (i, v.name)
            assert sizes[i] < len(got)


@pytest.mark.parametrize("lossless", [False, True])
@pytest.mark.parametrize("group", [1, 3, 8])
@pytest.mark.parametrize("kind", KINDS)
def test_resident_pipe_heterogeneous_inputs(L, O, kind, group, lossless):
    import torch
    assert L.lib().b200_init_device(0) == 0
    q, ss, prog, _ = ARMS["lossless" if lossless else "q80_420_progressive"]
    vs = pipe_inputs(kind)
    want = [oracle_file(O, v.data, q, ss, prog, lossless) if v.settles else None for v in vs]
    pipe = L.JpegPipe([v.data for v in vs], jparams(L, q, ss, prog, lossless), group=group)
    st = torch.cuda.Stream()
    try:
        for rep in range(2):
            pipe.run(st.cuda_stream)
            check_pipe(pipe, vs, want)
    finally:
        pipe.close()


@pytest.mark.parametrize("lossless", [False, True])
def test_resident_pipe_bench_call_pattern(L, O, lossless):
    """What bench.py does to one pipe: warm-up runs, 20 runs queued back to back without a host wait, the stage-only runs, the
    per-kernel timing, one more full run -- every image must still be the oracle's file, over two such cycles."""
    import torch
    assert L.lib().b200_init_device(0) == 0
    q, ss, prog, _ = ARMS["lossless" if lossless else "q80_420_progressive"]
    vs = pipe_inputs("420")
    want = [oracle_file(O, v.data, q, ss, prog, lossless) if v.settles else None for v in vs]
    pipe = L.JpegPipe([v.data for v in vs], jparams(L, q, ss, prog, lossless), group=8)
    st = torch.cuda.Stream()
    try:
        for cycle in range(2):
            for _ in range(2):
                pipe.run(st.cuda_stream)
            torch.cuda.synchronize()
            for _ in range(20):
                pipe.run(st.cuda_stream)
            check_pipe(pipe, vs, want)
            for which in (1, 2, 3):
                pipe.run(st.cuda_stream, which)
            torch.cuda.synchronize()
            pipe.kernel_times(1)
            pipe.run(st.cuda_stream)
            check_pipe(pipe, vs, want)
    finally:
        pipe.close()


@pytest.fixture(scope="module")
def jpegs_4k():
    from tools.synth import synth_jpeg
    with ThreadPoolExecutor(4) as ex:
        return list(ex.map(lambda i: synth_jpeg(3840, 2160, i), range(4)))


@pytest.mark.parametrize("lossless", [False, True])
@pytest.mark.parametrize("group", [3, 8])
def test_resident_pipe_4k_every_image_equals_oracle(L, O, jpegs_4k, group, lossless):
    """bench.py's configs[1] / [2] pipe (3840x2160 q90 4:2:0 sources, 11 images, ragged last group): all 11 fetched and compared."""
    import torch
    assert L.lib().b200_init_device(0) == 0
    q, ss, prog, _ = ARMS["lossless" if lossless else "q80_420_progressive"]
    with ThreadPoolExecutor(4) as ex:
        want4 = list(ex.map(lambda d: oracle_file(O, d, q, ss, prog, lossless), jpegs_4k))
    work = jpegs_4k * 2 + jpegs_4k[:3]
    pipe = L.JpegPipe(work, jparams(L, q, ss, prog, lossless), group=group)
    st = torch.cuda.Stream()
    try:
        for rep in range(2):
            pipe.run(st.cuda_stream)
            torch.cuda.synchronize()
            sizes, not_settled, _ = pipe.finish()
            assert not_settled == 0
            for i in range(len(work)):
                assert pipe.fetch(i) == want4[i % 4], (rep, i)
    finally:
        pipe.close()
