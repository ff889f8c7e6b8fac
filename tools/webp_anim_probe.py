"""Animated WebP leg probe (b200_set_webp_anim): seeded 480x270 (60 frames) and 1280x720 (30 frames) animations, re-encoded lossy at
webp_quality 80 and lossless.  Reports frames/s and MP/s (canvas pixels of every source frame over the call), and, from the library's
B200_TRACE=2 line of one traced call, the split into host decode, compose + diff, the encoder (K8 or VP8L) and its host coder (VP8's
boolean coder, or VP8L's header and emission).  Prints one JSON line per input and mode, with the card's name and power limit.

    python tools/webp_anim_probe.py [--reps 5] [--out <dir>/webp_anim_probe.json]
"""
import argparse
import io
import json
import os
import re
import subprocess
import sys
import tempfile
import time

import numpy as np
from PIL import Image

os.environ.setdefault("B200_TRACE", "2")             # read once, at the library's first traced call
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as E  # noqa: E402


def synthetic(w, h, n, seed=0):
    """a textured background, a sprite that moves and a panel that fades in and out; written lossy by Pillow with alpha"""
    rng = np.random.default_rng(seed)
    bg = np.zeros((h, w, 4), np.uint8)
    bg[..., :3] = (np.add.outer(np.arange(h) // 5, np.arange(w) // 5)[..., None] * np.array([3, 5, 7]) + rng.integers(0, 6, (h, w, 1))) % 256
    bg[..., 3] = 255
    frames = []
    for k in range(n):
        f = bg.copy()
        x, y = (17 * k) % (w - w // 4), (11 * k) % (h - h // 4)
        f[y:y + h // 4, x:x + w // 4, :3] = (np.add.outer(np.arange(h // 4), np.arange(w // 4))[..., None] * np.array([1, 2, 3]) + 9 * k) % 256
        f[h - h // 6:, : w // 3, 3] = int(255 * abs((k % 20) - 10) / 10)
        frames.append(Image.fromarray(f, "RGBA"))
    buf = io.BytesIO()
    frames[0].save(buf, "WEBP", save_all=True, append_images=frames[1:], duration=40, loop=0, quality=85, method=0)
    return buf.getvalue()


def traced(L, data, p):
    """the library's B200_TRACE=2 line of one call (stderr captured at the descriptor)"""
    with tempfile.TemporaryFile() as tmp:
        saved = os.dup(2)
        os.dup2(tmp.fileno(), 2)
        try:
            L.compress_in_memory(data, p)
        finally:
            os.dup2(saved, 2)
            os.close(saved)
        tmp.seek(0)
        lines = [s for s in tmp.read().decode(errors="replace").splitlines() if "webp-anim" in s]
    line = lines[-1] if lines else ""
    num = lambda key: float(m.group(1)) if (m := re.search(key + r" ([0-9.]+) ms", line)) else None
    return {"host_decode_ms": num("host decode"), "compose_diff_ms": num(r"compose \+ diff"), "encoder_ms": num("(?:K8|VP8L)"),
            "host_coder_ms": num("host coder")}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    L = E._pkg()
    assert L.lib().b200_init_device(0) == 0, "no GPU: this probe measures the device leg only"
    L.set_webp_anim(1)
    gpu = card()
    rows = []
    for w, h, n in ((480, 270, 60), (1280, 720, 30)):
        data = synthetic(w, h, n)
        for lossless in (False, True):
            p = L.default_params()
            p.webp_quality, p.webp_lossless = 80, int(lossless)
            out = L.compress_in_memory(data, p)                # warm-up: buffers, modules
            times = []
            for _ in range(a.reps):
                t = time.perf_counter()
                L.compress_in_memory(data, p)
                times.append(time.perf_counter() - t)
            med = float(np.median(times))
            row = {"input": f"{w}x{h}x{n}", "mode": "lossless" if lossless else "lossy q80", "call_ms": round(med * 1e3, 2),
                   "frames_per_s": round(n / med, 1), "mp_per_s": round(w * h * n / med / 1e6, 1), "source_bytes": len(data),
                   "output_bytes": len(out), "gpu": gpu, **traced(L, data, p)}
            rows.append(row)
            print(json.dumps(row), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            for r in rows:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
