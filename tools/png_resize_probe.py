"""Measure the PNG resize leg: compress_in_memory on PNG sources with width set and b200_set_png_resize(1) (GPU box only).
Seeded 4096x4096 inputs, an RGBA8 and an RGB16 photograph, stored as PNG; long edge 1920, level 3, lossless and lossy at q 80.
Prints one JSON line: the card's name and power limit, and per input and mode the median call time over --iters calls after a
warm-up, the B200_TRACE=2 stage split of the lossless call (parse + inflate, h2d + un-filter, expand + K3 + pack, back end), the same
file's call without the resize, and the resize stage's algorithmic bytes with the bandwidth they imply at the measured stage time.
usage: python tools/png_resize_probe.py [--iters N]"""
import argparse
import json
import os
import re
import statistics
import subprocess
import sys
import tempfile
import time
import zlib

os.environ["B200_TRACE"] = "2"          # read once when the library loads
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import numpy as np  # noqa: E402

from conftest import _import_pkg  # noqa: E402
from pngutil import frame_png, pil_png, synth  # noqa: E402

_import_pkg()
import caesium_clt_b200._lib as L  # noqa: E402

STAGES = re.compile(r"png stages (\d+)x(\d+) -> (\d+)x(\d+): parse \+ inflate ([\d.]+) ms, h2d \+ un-filter ([\d.]+) ms, "
                    r"expand \+ K3 \+ pack ([\d.]+) ms, back end ([\d.-]+) ms")
N = 4096
LONG_EDGE = 1920


def _inputs():
    yy, xx = np.mgrid[:N, :N]
    a = np.clip(300 - np.hypot(yy - N / 2, xx - N / 2) * 600 / N, 0, 255).astype(np.uint8)
    yield "rgba8_photo_4096x4096", pil_png(np.concatenate([synth(N, N, 3, seed=1), a[:, :, None]], axis=2), compress_level=1), 4, 1
    img = synth(N, N, 3, seed=2).astype(np.uint16) * 257 + (np.arange(N * N * 3).reshape(N, N, 3) % 199).astype(np.uint16)
    rows = b"".join(b"\x00" + img[y].astype(">u2").tobytes() for y in range(N))
    yield "rgb16_photo_4096x4096", frame_png(N, N, 16, 2, zlib.compress(rows, 1)), 3, 2


def _traced(fn):
    """run fn() with fd 2 captured; returns (result, stderr lines)"""
    with tempfile.TemporaryFile(mode="w+b") as f:
        sys.stderr.flush()
        saved = os.dup(2)
        os.dup2(f.fileno(), 2)
        try:
            r = fn()
        finally:
            os.dup2(saved, 2); os.close(saved)
        f.seek(0)
        return r, f.read().decode(errors="replace").splitlines()


def _timed(src, p, iters):
    L.compress_in_memory(src, p)                                           # warm-up: buffers, module load
    times = []

    def run():
        out = None
        for _ in range(iters):
            t0 = time.perf_counter()
            out = L.compress_in_memory(src, p)
            times.append(time.perf_counter() - t0)
        return out
    out, lines = _traced(run)
    return out, statistics.median(times), lines


def _stage_split(lines):
    recs = [m for m in (STAGES.search(s) for s in lines) if m]
    if not recs:
        return None
    med = lambda k: round(statistics.median(float(m.group(k)) for m in recs), 3)  # noqa: E731
    return {"parse_inflate_ms": med(5), "h2d_unfilter_ms": med(6), "expand_k3_pack_ms": med(7), "back_end_ms": med(8)}


def resize_bytes(ch, bps, w, h, nw, nh):
    """algorithmic HBM traffic of expand + K3 + pack: each array read or written once"""
    raw_in = h * w * ch * bps
    planes = ch * h * w * bps
    tmp = ch * nh * w * 4
    out_planes = ch * nh * nw * bps
    rows = nh * nw * ch * bps
    return {"raw_in": raw_in, "planes_written": planes, "planes_read": planes, "f32_written": tmp, "f32_read": tmp,
            "planes_out_written": out_planes, "planes_out_read": out_planes, "rows_packed": rows,
            "total": raw_in + 2 * planes + 2 * tmp + 2 * out_planes + rows}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    L.set_png_resize(True)
    L.set_png_lossy(True)
    result = {"probe": "png_resize", "card": card, "iters": args.iters, "long_edge": LONG_EDGE, "level": 3, "inputs": {}}
    for name, src, ch, bps in _inputs():
        entry = {"source_bytes": len(src)}
        for mode, optimize in (("lossless", 1), ("lossy_q80", 0)):
            p = L.default_params(); p.png_optimize, p.png_optimization_level, p.png_quality, p.width = optimize, 3, 80, LONG_EDGE
            out, dt, lines = _timed(src, p, args.iters)
            q = L.default_params(); q.png_optimize, q.png_optimization_level, q.png_quality = optimize, 3, 80
            out0, dt0, lines0 = _timed(src, q, args.iters)
            rec = {"resize_ms_per_call": round(dt * 1e3, 3), "out_bytes": len(out),
                   "no_resize_ms_per_call": round(dt0 * 1e3, 3), "no_resize_out_bytes": len(out0)}
            if optimize:
                rec["stages"] = _stage_split(lines)
                rec["no_resize_stages"] = _stage_split(lines0)
                if rec["stages"]:
                    b = resize_bytes(ch, bps, N, N, LONG_EDGE, LONG_EDGE)
                    rec["resize_bytes"] = b
                    ms = rec["stages"]["expand_k3_pack_ms"]
                    rec["resize_gb_per_s"] = round(b["total"] / (ms * 1e-3) / 1e9, 1) if ms > 0 else None
            entry[mode] = rec
        result["inputs"][name] = entry
    print(json.dumps(result))


if __name__ == "__main__":
    main()
