"""Measure the lossy PNG leg: compress_in_memory with png_optimize = 0 and b200_set_png_lossy(1) (GPU box only).
Seeded inputs: a 4096x4096 RGBA photograph with soft alpha and 1920x1080 flat art, stored as PNG.  Prints one JSON line: the card's
name and power limit, and per input the MP/s of the lossy call at q80 (level 3), its device time and per-kernel event times from the
B200_TRACE=2 lines, the same image's lossless call, and Pillow's quantize(256) + optimize on one core.
usage: python tools/png_lossy_probe.py [--iters N]"""
import argparse
import io
import json
import os
import re
import subprocess
import sys
import tempfile
import time

os.environ["B200_TRACE"] = "2"          # read once when the library loads
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import numpy as np  # noqa: E402
from PIL import Image  # noqa: E402

from conftest import _import_pkg  # noqa: E402
from pngutil import pil_png, synth  # noqa: E402

_import_pkg()
import caesium_clt_b200._lib as L  # noqa: E402

LOSSY = re.compile(r"png-lossy \d+x\d+ q\d+: (\d+) colours, device ([\d.]+) ms \(median cut ([\d.]+)\); kernels ms:(.*)$")
LOSSLESS = re.compile(r"png \d+x\d+: parse \+ inflate ([\d.]+) ms, device \(.*?\) ([\d.]+) ms, container")


def _inputs():
    h = w = 4096
    yy, xx = np.mgrid[:h, :w]
    a = np.clip(300 - np.hypot(yy - h / 2, xx - w / 2) * 600 / w, 0, 255).astype(np.uint8)
    yield "rgba_photo_4096x4096", np.concatenate([synth(h, w, 3, seed=1, kind="photo"), a[:, :, None]], axis=2)
    yield "flat_1920x1080", synth(1080, 1920, 3, seed=2, kind="flat")


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
    t0 = time.perf_counter()
    outs, lines = _traced(lambda: [L.compress_in_memory(src, p) for _ in range(iters)])
    return outs[-1], (time.perf_counter() - t0) / iters, lines


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    L.set_png_lossy(True)
    result = {"probe": "png_lossy", "card": card, "iters": args.iters, "inputs": {}}
    for name, img in _inputs():
        src = pil_png(img, compress_level=1)
        h, w = img.shape[:2]
        p = L.default_params(); p.png_optimize, p.png_quality = 0, 80
        out, dt, lines = _timed(src, p, args.iters)
        recs = [m for m in (LOSSY.search(s) for s in lines) if m]
        kern = {}
        for m in recs:
            for kv in m.group(4).split():
                k, v = kv.split("="); kern.setdefault(k, []).append(float(v))
        q = L.default_params(); q.png_optimize = 1
        out_ll, dt_ll, lines_ll = _timed(src, q, args.iters)
        ll = [float(m.group(2)) for m in (LOSSLESS.search(s) for s in lines_ll) if m]
        c0 = time.process_time()
        im = Image.fromarray(img)
        pq = im.quantize(256, method=Image.Quantize.FASTOCTREE if img.shape[2] == 4 else Image.Quantize.MEDIANCUT)
        b = io.BytesIO(); pq.save(b, "PNG", optimize=True)
        pil_cpu = time.process_time() - c0
        result["inputs"][name] = {
            "pixels": w * h, "source_bytes": len(src),
            "lossy_q80": {"mp_per_s": round(w * h / dt / 1e6, 2), "ms_per_call": round(dt * 1e3, 3), "out_bytes": len(out),
                          "colours": int(recs[-1].group(1)) if recs else None,
                          "device_ms": round(float(np.median([float(m.group(2)) for m in recs])), 3) if recs else None,
                          "median_cut_ms": round(float(np.median([float(m.group(3)) for m in recs])), 3) if recs else None,
                          "kernel_ms": {k: round(float(np.median(v)), 4) for k, v in sorted(kern.items())}},
            "lossless": {"mp_per_s": round(w * h / dt_ll / 1e6, 2), "ms_per_call": round(dt_ll * 1e3, 3), "out_bytes": len(out_ll),
                         "device_ms": round(float(np.median(ll)), 3) if ll else None},
            "pillow_quantize_optimize_one_core": {"cpu_s": round(pil_cpu, 3), "out_bytes": len(b.getvalue())},
        }
    print(json.dumps(result))


if __name__ == "__main__":
    main()
