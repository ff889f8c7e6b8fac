"""The deferred DC of lossy megabatches and the resident pipe at every sampling geometry and at DC values that wrap int16 and int32
(tests/wild_dc.py, pinned to libjpeg-turbo and restated by test_deferred_dc_wrap_host.py), run with -m gpu on an H100.

A megabatch member's DC comes from the decoder's batch-wide int32 prefix sum (put_dc, GpuDecoder::dc_sums); a single call's from
the decoder's scatter.  Every member below must come out byte for byte as its single call and as the oracle (and the trellis
oracle, with trellis on), in batches whose members differ in DC content, so that every member has its own dc_prev: Pillow-style
content next to wild DC differences at every geometry and size, and grey files whose batch-wide sum passes +2^31 or -2^31.  Those
batches are shown to have been decoded on the device: the resident pipe reports what it did not settle, and a child process
reads the megabatch counter B200_TRACE prints at exit."""
import os
import re
import subprocess
import sys

import pytest

import jpeg_geometry as G
import wild_dc as W

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = [(name, w, h) for name, f in G.GEOMETRIES.items() for (w, h) in G.sizes_for(f)]
OUTPUTS = [(0, True), (444, False), (420, True)]           # (output sampling, progressive); 0 keeps the input's: all on k_fused_same
CHROMA_ABOVE_1 = [name for name, f in G.GEOMETRIES.items() if len(f) == 3 and max(max(f[1]), max(f[2])) > 1]
PIPE_SUBSET = ["y12", "y41", "y32", "c21", "c12", "cr22", "c22", "grey22"]
GREY = G.GEOMETRIES["grey22"]


def group_of(name, w, h):
    """Three same-shaped members with different DC content: wild, Pillow-style (jpeg_geometry), wild with another seed."""
    f = G.GEOMETRIES[name]
    return [W.wild_jpeg(w, h, f, "wild", 1), G.make_jpeg(w, h, f, False), W.wild_jpeg(w, h, f, "wild", 2)]


def wrap_group(direction):
    return [W.wild_jpeg(*W.CLIMB_SIZE, GREY, p) for p in W.WRAP_BATCHES[direction]]


def lossy(L, O, ss, prog, q=80):
    p = L.default_params()
    p.jpeg_quality, p.jpeg_chroma_subsampling, p.jpeg_progressive = q, ss, int(prog)
    return p, O.params(q, ss, prog)


def check_batch(L, O, datas, ss, prog, trellis=False):
    """compress_batch (one thread: one megabatch) against the single calls and the oracle, member by member."""
    from oracle import jpeg_trellis as T
    L.set_entropy_mode(3)
    assert L.set_jpeg_trellis(1 if trellis else 0) == 0
    try:
        p, op = lossy(L, O, ss, prog)
        res = L.compress_batch(datas, p, n_threads=1)
        for i, (d, (out, code, msg)) in enumerate(zip(datas, res)):
            assert code == 0, (i, msg)
            assert out == L.compress_in_memory(d, p), (i, "megabatch differs from the single call")
            assert out == (T.jpeg_lossy if trellis else O.jpeg_lossy)(d, op), (i, "megabatch differs from the oracle")
    finally:
        assert L.set_jpeg_trellis(0) == 0


@pytest.mark.parametrize("name,w,h", CASES)
def test_geometry_megabatch_equals_single_calls_and_oracle(L, O, name, w, h):
    datas = group_of(name, w, h)
    for ss, prog in OUTPUTS:
        check_batch(L, O, datas, ss, prog)


@pytest.mark.parametrize("name,w,h", [(n, w, h) for n, w, h in CASES if n in CHROMA_ABOVE_1])
def test_geometry_megabatch_trellis(L, O, name, w, h):
    datas = group_of(name, w, h)
    for ss, prog in ((0, True), (420, False)):
        check_batch(L, O, datas, ss, prog, trellis=True)


@pytest.mark.parametrize("direction", list(W.WRAP_BATCHES))
def test_prefix_sum_past_int32_megabatch(L, O, direction):
    """Three 1448 x 1448 grey files, each climbing its running DC to about +-2^30 in its own steps: the batch-wide sum passes
    +-2^31 inside the third member.  (Grey output: the output sampling does not matter, the scan layout does.)"""
    for prog in (True, False):
        check_batch(L, O, wrap_group(direction), 0, prog)


def run_pipe(L, work, p, group):
    import torch
    assert L.lib().b200_init_device(0) == 0
    st = torch.cuda.Stream()
    pipe = L.JpegPipe(work, p, group=group)
    try:
        for _ in range(2):
            pipe.run(st.cuda_stream)
        torch.cuda.synchronize()
        _, not_settled, _ = pipe.finish()
        assert not_settled == 0, "a member went to the host decoder"
        return [pipe.fetch(i) for i in range(len(work))]
    finally:
        pipe.close()


@pytest.mark.parametrize("name", PIPE_SUBSET)
def test_resident_pipe_geometry(L, O, name):
    for (w, h) in [(130, 61), (G.sizes_for(G.GEOMETRIES[name])[-1])]:
        datas = group_of(name, w, h)
        work = datas + datas[:1]
        for ss, prog in ((0, True), (420, True)):
            p, op = lossy(L, O, ss, prog)
            for d, out in zip(work, run_pipe(L, work, p, group=2)):
                assert out == O.jpeg_lossy(d, op), (w, h, ss)


@pytest.mark.parametrize("direction", list(W.WRAP_BATCHES))
def test_resident_pipe_prefix_sum_past_int32(L, O, direction):
    work = wrap_group(direction)
    p, op = lossy(L, O, 0, True)
    for d, out in zip(work, run_pipe(L, work, p, group=3)):
        assert out == O.jpeg_lossy(d, op)


_CHILD = """
import sys
sys.path.insert(0, {tests!r}); sys.path.insert(0, {root!r})
import conftest
conftest._import_pkg()
import caesium_clt_b200._lib as L
import test_deferred_dc_wrap_gpu as T
assert L.lib().b200_init_device(0) == 0
L.set_entropy_mode(3)
p = L.default_params()
p.jpeg_quality, p.jpeg_chroma_subsampling, p.jpeg_progressive = 80, 420, 1
groups = [T.group_of(*c) for c in T.CASES] + [T.wrap_group(d) for d in T.W.WRAP_BATCHES]
for datas in groups:
    for out, code, msg in L.compress_batch(datas, p, n_threads=1):
        assert code == 0, msg
print("ok", sum(len(g) for g in groups))
"""


def test_megabatch_members_are_decoded_on_the_device():
    """Every member of the groups above stays in its megabatch: none is left to the per-image path (the host decoder), which would
    come out right without the deferred DC having been tested at all."""
    env = dict(os.environ, B200_TRACE="1", B200_MEGABATCH="8")
    r = subprocess.run([sys.executable, "-c", _CHILD.format(tests=os.path.join(ROOT, "tests"), root=ROOT)], env=env, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    n = int(r.stdout.split()[-1])
    m = re.search(r"\[b200 trace\] megabatch: (\d+) members, (\d+) left to the per-image path", r.stderr)
    assert m, r.stderr[-2000:]
    assert (int(m.group(1)), int(m.group(2))) == (n, 0)
