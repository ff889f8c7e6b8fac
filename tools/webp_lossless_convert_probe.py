"""Measure the JPEG / PNG -> lossless WebP conversion (convert_in_memory with webp_lossless, the switch on; GPU box only).
Seeded inputs: a 3840x2160 photograph as JPEG (4:2:0, q90) and as RGB PNG, a 1920x1080 RGBA PNG with soft alpha, a 3840x2160 8-bit
palette PNG (flat art), and a 24 MP JPEG converted with width = 1920.  Prints one JSON line with the card's name and power limit and,
per input: MP/s of the call (median of --iters calls after a warm-up), the stage split and the bytes fetched from the device from the
B200_TRACE=2 line (a separate traced run: the trace waits for the device between stages), output against source bytes, and the bytes
and CPU time of Pillow's libwebp at lossless=True, method=4 on the same host.
usage: python tools/webp_lossless_convert_probe.py [--iters N]"""
import argparse
import io
import json
import os
import re
import subprocess
import sys
import time

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import numpy as np  # noqa: E402
from PIL import Image  # noqa: E402

from conftest import _import_pkg  # noqa: E402
from pngutil import pil_png, synth  # noqa: E402

TRACE = re.compile(r"webp-lossless-convert (\w+) \d+x\d+ -> \d+x\d+: (.+?) ([\d.]+) ms, front end ([\d.]+) ms, resize ([\d.]+) ms, encode ([\d.]+) ms "
                   r"\(cache bits (\d+)\); fetched (\d+) bytes \(encoder\), sample planes fetched (\d+)")


def _jpeg(img, q=90):
    b = io.BytesIO(); Image.fromarray(img).save(b, "JPEG", quality=q, subsampling=2); return b.getvalue()


def _inputs():
    photo = synth(2160, 3840, 3, seed=1, kind="photo")
    yield "jpeg_photo_3840x2160_q90", _jpeg(photo), photo, 0
    yield "png_rgb_3840x2160", pil_png(photo), photo, 0
    h, w = 1080, 1920
    yy, xx = np.mgrid[:h, :w]
    a = np.clip(300 - np.hypot(yy - h / 2, xx - w / 2) * 600 / w, 0, 255).astype(np.uint8)
    rgba = np.concatenate([synth(h, w, 3, seed=3, kind="photo"), a[:, :, None]], axis=2)
    yield "png_rgba_soft_alpha_1920x1080", pil_png(rgba), rgba, 0
    pal = Image.fromarray(synth(2160, 3840, 3, seed=2, kind="flat")).quantize(256)
    yield "png_palette8_flat_3840x2160", pil_png(pal), np.asarray(pal.convert("RGB")), 0
    big = synth(4000, 6000, 3, seed=4, kind="photo")
    yield "jpeg_24mp_width1920", _jpeg(big), None, 1920


def _card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=7)
    args = ap.parse_args()
    _import_pkg()
    import caesium_clt_b200._lib as L
    assert L.set_webp_lossless_convert(1) == 0
    result = {"probe": "webp_lossless_convert", "card": _card(), "iters": args.iters, "inputs": {}}
    for name, src, img, width in _inputs():
        p = L.default_params(); p.webp_lossless = 1; p.width = width
        out = L.convert_in_memory(src, p, L.FMT_WEBP)                       # warm-up: buffers, module load
        ts = []
        for _ in range(args.iters):
            t0 = time.perf_counter(); L.convert_in_memory(src, p, L.FMT_WEBP); ts.append(time.perf_counter() - t0)
        dt = float(np.median(ts))
        w, h = Image.open(io.BytesIO(src)).size
        entry = {"pixels": w * h, "source_bytes": len(src), "mp_per_s": round(w * h / dt / 1e6, 2), "ms_per_call": round(dt * 1e3, 3), "out_bytes": len(out)}
        if img is not None:
            c0 = time.process_time()
            b = io.BytesIO(); Image.fromarray(img).save(b, "WEBP", lossless=True, method=4)
            entry.update({"libwebp_m4_bytes": len(b.getvalue()), "libwebp_m4_cpu_s": round(time.process_time() - c0, 3)})
        result["inputs"][name] = entry
    # the stage split: a second process with B200_TRACE=2 (read once when the library loads)
    env = dict(os.environ, B200_TRACE="2", B200_PROBE_CHILD="1")
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--iters", "3"], env=env, capture_output=True, text=True)
    names = [n for n, *_ in _inputs()] if r.returncode == 0 else []
    recs = [m for m in (TRACE.search(s) for s in r.stderr.splitlines()) if m]
    per = max(1, len(recs) // max(1, len(names))) if names else 0
    for k, name in enumerate(names):
        mine = recs[k * per:(k + 1) * per][1:] or recs[k * per:(k + 1) * per]
        if not mine:
            continue
        med = lambda g: round(float(np.median([float(m.group(g)) for m in mine])), 3)  # noqa: E731
        result["inputs"][name].update({"stage0": mine[0].group(2), "stage0_ms": med(3), "front_end_ms": med(4), "resize_ms": med(5), "encode_ms": med(6),
                                       "cache_bits": int(mine[-1].group(7)), "d2h_bytes_encoder": int(mine[-1].group(8)), "d2h_sample_bytes": int(mine[-1].group(9))})
    print(json.dumps(result))


def child(iters):
    _import_pkg()
    import caesium_clt_b200._lib as L
    assert L.set_webp_lossless_convert(1) == 0
    for name, src, img, width in _inputs():
        p = L.default_params(); p.webp_lossless = 1; p.width = width
        for _ in range(iters + 1):
            L.convert_in_memory(src, p, L.FMT_WEBP)


if __name__ == "__main__":
    if os.environ.get("B200_PROBE_CHILD"):
        child(int(sys.argv[sys.argv.index("--iters") + 1]) if "--iters" in sys.argv else 3)
    else:
        main()
