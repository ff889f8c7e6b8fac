"""GIF leg probe (b200_set_gif): for GIF files (tests/golden/g1_head.gif, the first two frames of caesium-clt's animated
sample g1.gif, unless --gif names others, such as the whole sample) and a seeded 1920x1080, 60-frame animation: the call time
and MP/s (canvas pixels of every frame over the call), the host decoder's time inside the call (B200_TRACE=2) against the rest
of the call per frame, and output bytes against the source and against Pillow's optimize=True re-save, at gif_quality 80
(caesiumclt's default).  Prints one JSON line per input, with the card's name and power limit.

    python tools/gif_probe.py [--gif a.gif ...] [--reps 5] [--out <dir>/gif_probe.json]
"""
import argparse
import io
import json
import os
import subprocess
import sys
import time

import numpy as np
from PIL import Image

os.environ.setdefault("B200_TRACE", "2")             # read once, at the library's first GIF call
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as E  # noqa: E402


def synthetic(w=1920, h=1080, n=60, seed=0):
    """a static textured background with a sprite that moves and a panel that changes colour, 256 global colours"""
    rng = np.random.default_rng(seed)
    pal = rng.integers(0, 256, (256, 3)).astype(np.uint8)
    bg = ((np.add.outer(np.arange(h) // 6, np.arange(w) // 6) + rng.integers(0, 3, (h, w))) % 200).astype(np.uint8)
    frames = []
    for k in range(n):
        idx = bg.copy()
        x, y = 40 + 25 * k, 100 + 10 * k
        idx[y:y + 160, x:x + 240] = (200 + (np.add.outer(np.arange(160), np.arange(240)) // 9 + k) % 56).astype(np.uint8)
        idx[900:1000, 1500:1800] = 200 + k % 56
        im = Image.fromarray(idx, "P")
        im.putpalette(pal.reshape(-1).tolist())
        frames.append(im)
    buf = io.BytesIO()
    frames[0].save(buf, "GIF", save_all=True, append_images=frames[1:], duration=40, loop=0)
    return buf.getvalue()


def pillow_optimized(data):
    im = Image.open(io.BytesIO(data))
    buf = io.BytesIO()
    im.save(buf, "GIF", save_all=True, optimize=True)
    return len(buf.getvalue())


def traced_decode_ms(L, data, p):
    """the host decoder's share of one call, as the library's B200_TRACE=2 line reports it (stderr captured at the descriptor)"""
    import re
    import tempfile
    with tempfile.TemporaryFile() as tmp:
        saved = os.dup(2)
        os.dup2(tmp.fileno(), 2)
        try:
            L.compress_in_memory(data, p)
        finally:
            os.dup2(saved, 2)
            os.close(saved)
        tmp.seek(0)
        m = re.search(rb"host decode ([0-9.]+) ms", tmp.read())
    return float(m.group(1)) if m else float("nan")


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--quality", type=int, default=80)
    ap.add_argument("--out", default=None)
    ap.add_argument("--gif", action="append", default=None, help="a GIF file to measure (repeatable)")
    a = ap.parse_args()
    L = E._pkg()
    assert L.lib().b200_init_device(0) == 0, "no GPU"
    assert L.set_gif(True) == 0
    p = L.default_params()
    p.gif_quality = a.quality
    inputs = []
    for path in a.gif or [os.path.join(ROOT, "tests", "golden", "g1_head.gif")]:
        with open(path, "rb") as f:
            inputs.append((os.path.basename(path), f.read()))
    inputs.append(("synthetic_1920x1080x60", synthetic()))
    gpu = card()
    rows = []
    for name, data in inputs:
        canv, delays, loop = L.gif_decode(data)
        n, h, w = canv.shape[:3]
        del canv
        out = L.compress_in_memory(data, p)           # warm-up: buffers and modules
        call = []
        for _ in range(a.reps):
            t = time.perf_counter(); out = L.compress_in_memory(data, p); call.append(time.perf_counter() - t)
        tc, td = float(np.median(call)), traced_decode_ms(L, data, p) / 1e3
        row = dict(input=name, width=w, height=h, frames=n, quality=a.quality, call_ms=round(1e3 * tc, 2),
                   mp_per_s=round(w * h * n / tc / 1e6, 1), host_decode_ms_per_frame=round(1e3 * td / n, 3),
                   rest_ms_per_frame=round(1e3 * (tc - td) / n, 3), source_bytes=len(data), output_bytes=len(out),
                   pillow_optimize_bytes=pillow_optimized(data), gpu=gpu)
        rows.append(row)
        print(json.dumps(row), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
