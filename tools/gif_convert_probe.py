"""Measure the conversions to and from GIF (convert_in_memory, the GIF conversion switch on; GPU box only).  Inputs: a seeded 24 MP
JPEG (6000x4000, q90) -> GIF, a seeded 4096x4096 RGBA PNG with soft alpha -> GIF, and frame 0 of caesium-clt's sample g1.gif (the
repository keeps its first two frames as tests/golden/g1_head.gif) -> lossy WebP.  Prints one JSON line with the card's name and
power limit and, per input: MP/s of the call (median of --iters calls after a warm-up), output and source bytes, and the stage split
from the B200_TRACE=2 line (a separate traced run: the trace waits for the device between stages).
usage: python tools/gif_convert_probe.py [--iters N]"""
import argparse
import io
import json
import os
import re
import subprocess
import sys
import time

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
from PIL import Image  # noqa: E402

from conftest import _import_pkg  # noqa: E402
from pngutil import pil_png, synth  # noqa: E402

TO_GIF = re.compile(r"gif-convert (\w+) \d+x\d+ -> gif q\d+: (.+?) ([\d.]+) ms, device front end \+ canvas ([\d.]+) ms, quantise \+ LZW \+ container ([\d.]+) ms")
FROM_GIF = re.compile(r"gif-convert gif \d+x\d+ -> (\w+): frame 0 host decode ([\d.]+) ms, back end ([\d.]+) ms")
FMT_JPEG, FMT_PNG, FMT_GIF, FMT_WEBP = 0, 1, 2, 3


def _inputs():
    b = io.BytesIO(); Image.fromarray(synth(1000, 1500, 3, seed=4)).resize((6000, 4000)).save(b, "JPEG", quality=90)
    yield "jpeg_24mp_to_gif", b.getvalue(), FMT_GIF
    n = 4096
    yy, xx = np.mgrid[:n, :n]
    a = np.clip(300 - np.hypot(yy - n / 2, xx - n / 2) * 600 / n, 0, 255).astype(np.uint8)
    yield "png_rgba_4096_to_gif", pil_png(np.concatenate([synth(n, n, 3, seed=3), a[:, :, None]], axis=2)), FMT_GIF
    with open(os.path.join(ROOT, "tests", "golden", "g1_head.gif"), "rb") as f:
        yield "g1_frame0_to_webp", f.read(), FMT_WEBP


def _card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else None


def _lib():
    _import_pkg()
    import caesium_clt_b200._lib as L
    assert L.set_gif_convert(1) == 0
    return L


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=7)
    args = ap.parse_args()
    L = _lib()
    result = {"probe": "gif_convert", "card": _card(), "iters": args.iters, "inputs": {}}
    for name, src, fmt in _inputs():
        p = L.default_params()
        out = L.convert_in_memory(src, p, fmt)                               # warm-up: buffers, module load
        ts = []
        for _ in range(args.iters):
            t0 = time.perf_counter(); L.convert_in_memory(src, p, fmt); ts.append(time.perf_counter() - t0)
        dt = float(np.median(ts))
        w, h = Image.open(io.BytesIO(src)).size
        result["inputs"][name] = {"pixels": w * h, "source_bytes": len(src), "out_bytes": len(out), "ms_per_call": round(dt * 1e3, 3),
                                  "mp_per_s": round(w * h / dt / 1e6, 2)}
    # the stage split: a second process with B200_TRACE=2 (read once when the library loads); the first call of each input is a warm-up
    env = dict(os.environ, B200_TRACE="2", B200_PROBE_CHILD="1")
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--iters", "3"], env=env, capture_output=True, text=True)
    lines = r.stderr.splitlines() if r.returncode == 0 else []
    to = [m for m in (TO_GIF.search(s) for s in lines) if m]
    fr = [m for m in (FROM_GIF.search(s) for s in lines) if m]
    med = lambda ms, g: round(float(np.median([float(m.group(g)) for m in ms])), 3)  # noqa: E731
    for name, recs in (("jpeg_24mp_to_gif", [m for m in to if m.group(1) == "jpeg"][1:]), ("png_rgba_4096_to_gif", [m for m in to if m.group(1) == "png"][1:])):
        if recs:
            result["inputs"][name].update({"stage0": recs[0].group(2), "stage0_ms": med(recs, 3), "front_end_canvas_ms": med(recs, 4), "quantise_lzw_container_ms": med(recs, 5)})
    if fr[1:]:
        result["inputs"]["g1_frame0_to_webp"].update({"frame0_host_decode_ms": med(fr[1:], 2), "back_end_ms": med(fr[1:], 3)})
    print(json.dumps(result))


def child(iters):
    L = _lib()
    for name, src, fmt in _inputs():
        for _ in range(iters + 1):
            L.convert_in_memory(src, L.default_params(), fmt)


if __name__ == "__main__":
    if os.environ.get("B200_PROBE_CHILD"):
        child(int(sys.argv[sys.argv.index("--iters") + 1]) if "--iters" in sys.argv else 3)
    else:
        main()
