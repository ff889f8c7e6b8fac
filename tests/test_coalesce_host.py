"""Opt-in coalescing of per-image calls (B200_COALESCE=1, api.cpp): many threads calling b200_compress_in_memory at once must each
get exactly what the direct call returns -- same bytes, same error codes -- whatever mix of parameters, formats and bad inputs
arrives together.  Runs in a subprocess (the switch is read when the library is first used); on a box without a GPU the batch the
collector runs falls through to the per-image host transcode, so the queueing logic is what is exercised here."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SCRIPT = r"""
import json, os, sys, threading, random
sys.path.insert(0, %(root)r)
import bench
L = bench.load_pkg()
G = os.path.join(%(root)r, "tests", "golden")
names = ["in_420_base_355x237.jpg", "in_444_base_355x237.jpg", "in_420_prog_355x237.jpg", "in_gray_base_355x237.jpg", "in_420_tiny_17x9.jpg"]
datas = [open(os.path.join(G, n), "rb").read() for n in names]
LOSSY = %(lossy)d
def params(prog, meta):
    p = L.default_params(); p.jpeg_progressive = prog; p.keep_metadata = meta
    if LOSSY: p.jpeg_quality = 80; p.jpeg_chroma_subsampling = 420
    else: p.jpeg_optimize = 1
    return p
variants = [(1, 0), (0, 0), (1, 1)]
jobs = []
rng = random.Random(5)
for i in range(240):
    v = variants[rng.randrange(3)]
    kind = rng.random()
    if kind < 0.8: d = datas[rng.randrange(len(datas))]
    elif kind < 0.9: d = b"\xff\xd8\xff\xe0 not really a jpeg" + bytes(50)
    else: d = datas[0][:400]                                   # truncated
    jobs.append((d, v))
def run(job):
    d, v = job
    try: return ("ok", L.compress_in_memory(d, params(*v)))
    except L.B200Error as e: return ("err", e.code)
results = [None] * len(jobs)
def worker(lo, hi):
    for i in range(lo, hi): results[i] = run(jobs[i])
T = 24
th = [threading.Thread(target=worker, args=(k * len(jobs) // T, (k + 1) * len(jobs) // T)) for k in range(T)]
[t.start() for t in th]; [t.join() for t in th]
out = []
for r in results:
    out.append([r[0], len(r[1]) if r[0] == "ok" else r[1], __import__("hashlib").sha1(r[1]).hexdigest() if r[0] == "ok" else ""])
print(json.dumps(out))
"""


def _run(coalesce, lossy=False):
    env = dict(os.environ)
    env.pop("B200_COALESCE", None)
    if coalesce:
        env.update(B200_COALESCE="1", B200_COALESCE_TARGET="8", B200_COALESCE_US="2000")
    r = subprocess.run([sys.executable, "-c", SCRIPT % {"root": ROOT, "lossy": 1 if lossy else 0}], capture_output=True, text=True, env=env, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


def test_coalesced_calls_return_what_direct_calls_return():
    direct = _run(False)
    merged = _run(True)
    assert len(direct) == len(merged) == 240
    assert merged == direct
    assert sum(1 for r in direct if r[0] == "ok") > 150 and sum(1 for r in direct if r[0] == "err") > 10


@pytest.mark.gpu
def test_coalesced_lossy_calls_on_the_gpu_return_what_direct_calls_return():
    """the same on an H100 with the lossy path: the collector's batch takes the megabatch route (same-shaped files decoded,
    transformed and encoded together), the direct calls the one-image route -- the bytes must not differ"""
    direct = _run(False, lossy=True)
    merged = _run(True, lossy=True)
    assert merged == direct and sum(1 for r in direct if r[0] == "ok") > 150
