"""Measure Adam7-interlaced PNG input on the device (b200_set_png_interlaced(1); GPU box only).
Seeded 4096x4096 photographs -- RGBA8, RGB16 and 1-bit grey -- each written as an Adam7 file and as its non-interlaced twin
(tests/adam7.py).  Prints one JSON line: the card's name and power limit, and per input and file the median compress_in_memory
time (lossless, level 3) over --iters calls after a warm-up, the B200_TRACE=2 stage split (parse + inflate, h2d + un-filter, back
end), the per-kernel device times of b200_png_device_times (the pass wavefront k_png_adam7_unfilter and k_png_adam7_gather for
the Adam7 file, k_png_unfilter for the twin), and whether both files' outputs are identical.
usage: python tools/png_interlaced_probe.py [--iters N]"""
import argparse
import json
import os
import re
import statistics
import subprocess
import sys

os.environ["B200_TRACE"] = "2"          # read once when the library loads
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import numpy as np  # noqa: E402

from adam7 import adam7_pair  # noqa: E402
from conftest import _import_pkg  # noqa: E402
from pngutil import synth  # noqa: E402

_import_pkg()
import caesium_clt_b200._lib as L  # noqa: E402
from tools.png_resize_probe import _timed  # noqa: E402

STAGES = re.compile(r"png stages (\d+)x(\d+) -> (\d+)x(\d+): parse \+ inflate ([\d.]+) ms, h2d \+ un-filter ([\d.]+) ms, "
                    r"expand \+ K3 \+ pack ([\d.]+) ms, back end ([\d.-]+) ms")
N = 4096
KERNELS = ("h2d", "k_png_adler", "k_png_unfilter", "k_png_adam7_unfilter", "k_png_adam7_gather")


def _inputs():
    """(name, Adam7 file, twin)"""
    yy, xx = np.mgrid[:N, :N]
    a = np.clip(300 - np.hypot(yy - N / 2, xx - N / 2) * 600 / N, 0, 255).astype(np.uint8)
    rgba = np.concatenate([synth(N, N, 3, seed=1), a[:, :, None]], axis=2)
    yield ("rgba8_photo_4096x4096",) + adam7_pair(rgba.reshape(N, -1), N, N, 6, 8, seed=1, level=1)
    img = synth(N, N, 3, seed=2).astype(np.uint16) * 257 + (np.arange(N * N * 3).reshape(N, N, 3) % 199).astype(np.uint16)
    yield ("rgb16_photo_4096x4096",) + adam7_pair(img.astype(">u2").view(np.uint8).reshape(N, -1), N, N, 2, 16, seed=2, level=1)
    grey = synth(N, N, 1, seed=3)[..., 0]
    bits = (grey > np.random.default_rng(3).integers(0, 256, (N, N))).astype(np.uint8)    # a dithered photograph
    yield ("grey1_photo_4096x4096",) + adam7_pair(np.packbits(bits, axis=1), N, N, 0, 1, seed=3, level=1)


def _stage_split(lines):
    recs = [m for m in (STAGES.search(s) for s in lines) if m]
    if not recs:
        return None
    med = lambda k: round(statistics.median(float(m.group(k)) for m in recs), 3)  # noqa: E731
    return {"parse_inflate_ms": med(5), "h2d_unfilter_ms": med(6), "back_end_ms": med(8)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    L.set_png_interlaced(1)
    result = {"probe": "png_interlaced", "card": card, "iters": args.iters, "level": 3, "inputs": {}}
    p = L.default_params(); p.png_optimize, p.png_optimization_level = 1, 3
    for name, inter, twin in _inputs():
        entry = {}
        outs = []
        for kind, src in (("adam7", inter), ("twin", twin)):
            out, dt, lines = _timed(src, p, args.iters)
            outs.append(out)
            k = L.png_device_times(src, level=3, iters=args.iters)
            entry[kind] = {"source_bytes": len(src), "ms_per_call": round(dt * 1e3, 3), "out_bytes": len(out), "stages": _stage_split(lines),
                           "kernel_ms": {n: round(k[n][0], 4) for n in KERNELS if n in k}}
        entry["outputs_identical"] = outs[0] == outs[1]
        a, t = entry["adam7"], entry["twin"]
        if a["stages"] and t["stages"] and t["stages"]["h2d_unfilter_ms"] > 0:
            entry["h2d_unfilter_ratio"] = round(a["stages"]["h2d_unfilter_ms"] / t["stages"]["h2d_unfilter_ms"], 3)
        entry["call_time_ratio"] = round(a["ms_per_call"] / t["ms_per_call"], 3)
        result["inputs"][name] = entry
    L.set_png_interlaced(0)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
