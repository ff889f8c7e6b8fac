"""Measure the lossless WebP (VP8L) leg: compress_in_memory with webp_lossless on WebP sources (GPU box only).
Seeded inputs: a 3840x2160 photograph, 3840x2160 flat art, and a 1920x1080 RGBA image with soft alpha, each stored as a lossless WebP.
Prints one JSON line: per input the MP/s of the call, its host decode and device encode from the B200_TRACE=2 lines, the per-kernel
event times, the output bytes, and the bytes and CPU time of Pillow's libwebp at lossless=True, method=4, quality=70.
usage: python tools/webp_lossless_probe.py [--iters N]"""
import argparse
import io
import json
import os
import re
import sys
import tempfile
import time

os.environ["B200_TRACE"] = "2"          # read once when the library loads
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import numpy as np  # noqa: E402
from PIL import Image  # noqa: E402

from conftest import _import_pkg  # noqa: E402
from pngutil import synth  # noqa: E402

_import_pkg()
import caesium_clt_b200._lib as L  # noqa: E402

TRACE = re.compile(r"webp-lossless \d+x\d+ -> \d+x\d+: host decode ([\d.]+) ms, resize ([\d.]+) ms, device encode ([\d.]+) ms .*cache bits (\d+).*kernels ms:(.*)$")


def _inputs():
    yield "photo_3840x2160", synth(2160, 3840, 3, seed=1, kind="photo")
    yield "flat_3840x2160", synth(2160, 3840, 3, seed=2, kind="flat")
    h, w = 1080, 1920
    yy, xx = np.mgrid[:h, :w]
    a = np.clip(300 - np.hypot(yy - h / 2, xx - w / 2) * 600 / w, 0, 255).astype(np.uint8)
    yield "rgba_soft_alpha_1920x1080", np.concatenate([synth(h, w, 3, seed=3, kind="photo"), a[:, :, None]], axis=2)


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    args = ap.parse_args()
    p = L.default_params(); p.webp_lossless = 1
    result = {"probe": "webp_lossless", "iters": args.iters, "inputs": {}}
    for name, img in _inputs():
        b = io.BytesIO(); Image.fromarray(img).save(b, "WEBP", lossless=True, method=0, exact=True); src = b.getvalue()
        h, w = img.shape[:2]
        L.compress_in_memory(src, p)                                       # warm-up: buffers, module load
        t0 = time.perf_counter()
        outs, lines = _traced(lambda: [L.compress_in_memory(src, p) for _ in range(args.iters)])
        dt = (time.perf_counter() - t0) / args.iters
        recs = [m for m in (TRACE.search(s) for s in lines) if m]
        dec = [float(m.group(1)) for m in recs]; enc = [float(m.group(3)) for m in recs]
        kern = {}
        for m in recs:
            for kv in m.group(5).split():
                k, v = kv.split("="); kern.setdefault(k, []).append(float(v))
        c0 = time.process_time(); t1 = time.perf_counter()
        b = io.BytesIO(); Image.fromarray(img).save(b, "WEBP", lossless=True, method=4, quality=70)
        pil_cpu, pil_wall = time.process_time() - c0, time.perf_counter() - t1
        result["inputs"][name] = {
            "pixels": w * h, "source_bytes": len(src), "mp_per_s": round(w * h / dt / 1e6, 2), "ms_per_call": round(dt * 1e3, 3),
            "host_decode_ms": round(float(np.median(dec)), 3) if dec else None, "device_encode_ms": round(float(np.median(enc)), 3) if enc else None,
            "cache_bits": int(recs[-1].group(4)) if recs else None,
            "kernel_ms": {k: round(float(np.median(v)), 4) for k, v in sorted(kern.items())},
            "out_bytes": len(outs[-1]), "libwebp_m4_q70_bytes": len(b.getvalue()),
            "libwebp_m4_q70_cpu_s": round(pil_cpu, 3), "libwebp_m4_q70_wall_s": round(pil_wall, 3),
        }
    print(json.dumps(result))


if __name__ == "__main__":
    main()
