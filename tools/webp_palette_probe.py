"""Lossless WebP with the palette switch on the device: call time with the switch off and on (alternated, median of 5 after a
warm-up), the palette kernels' device times (a separate torch.profiler run), bytes off and on, and libwebp's bytes and CPU time
(Pillow, lossless=True, method=4, one call) for a 4K photograph, 4K flat art, a 4K 8-bit palette PNG (-> lossless WebP), a
two-colour 4K bitmap and a few-colour sprite animation.  Prints one JSON line.  Needs an H100."""
import io
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
from PIL import Image  # noqa: E402

import __graft_entry__ as G  # noqa: E402
from pngutil import pil_png, synth  # noqa: E402
from webp_palette_cases import sprite_sheet, two_colour_bitmap  # noqa: E402


def _webp(img, **kw):
    b = io.BytesIO(); img.save(b, "WEBP", **kw)
    return b.getvalue()


def _animation():
    """24 frames of 640 x 360: a 16-colour sprite sheet scrolled by 4 pixels a frame"""
    sheet = sprite_sheet(360, 736)
    return [Image.fromarray(np.ascontiguousarray(sheet[:, 4 * k:4 * k + 640]), "RGBA") for k in range(24)]


def inputs():
    """name -> (source bytes, call kind, Pillow images libwebp codes)"""
    photo = Image.fromarray(synth(2160, 3840, 3, seed=7, kind="photo"))
    flat = Image.fromarray(synth(2160, 3840, 3, seed=7, kind="flat"))
    pal = Image.fromarray(synth(2160, 3840, 3, seed=8, kind="photo")).quantize(256)
    bitmap = Image.fromarray(two_colour_bitmap(2160, 3840), "RGBA")
    frames = _animation()
    return {
        "photo_3840x2160": (_webp(photo, lossless=True, method=0), "compress", [photo]),
        "flat_3840x2160": (_webp(flat, lossless=True, method=0), "compress", [flat]),
        "palette_png_3840x2160": (pil_png(pal, compress_level=1), "convert", [pal.convert("RGBA")]),
        "bitmap_3840x2160": (_webp(bitmap, lossless=True, method=0), "compress", [bitmap]),
        "sprite_anim_640x360x24": (_webp(frames[0], save_all=True, append_images=frames[1:], lossless=True, method=0, duration=40), "compress", frames),
    }


def libwebp(images):
    t = time.perf_counter()
    if len(images) == 1:
        data = _webp(images[0], lossless=True, method=4)
    else:
        data = _webp(images[0], save_all=True, append_images=images[1:], lossless=True, method=4, duration=40)
    return len(data), (time.perf_counter() - t) * 1e3


def main():
    L = G._pkg()
    assert L.lib().b200_init_device(0) == 0, "no GPU"
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    assert L.set_webp_lossless_convert(1) == 0 and L.set_webp_anim(1) == 0
    p = L.default_params(); p.webp_lossless = 1
    call = {"compress": lambda d: L.compress_in_memory(d, p), "convert": lambda d: L.convert_in_memory(d, p, L.FMT_WEBP)}
    out = {"card": card, "inputs": {}}
    cases = inputs()
    for name, (data, kind, images) in cases.items():
        f = call[kind]
        L.set_webp_palette(0); off = f(data)
        L.set_webp_palette(1); on = f(data)
        t_off, t_on = [], []
        for _ in range(5):
            for sw, acc in ((0, t_off), (1, t_on)):
                L.set_webp_palette(sw)
                t = time.perf_counter(); f(data); acc.append((time.perf_counter() - t) * 1e3)
        lw_bytes, lw_ms = libwebp(images)
        out["inputs"][name] = {"ms_off": round(statistics.median(t_off), 2), "ms_on": round(statistics.median(t_on), 2),
                               "bytes_off": len(off), "bytes_on": len(on), "libwebp_bytes": lw_bytes, "libwebp_cpu_ms": round(lw_ms, 1)}
    import torch
    from torch.profiler import ProfilerActivity, profile
    L.set_webp_palette(1)
    for name, (data, kind, _) in cases.items():
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            call[kind](data)
            torch.cuda.synchronize()
        split, total = {}, 0.0
        for e in prof.key_averages():
            ms = e.device_time_total / 1e3
            total += ms
            short = next((t for t in e.key.replace("(", " ").replace("<", " ").replace("::", " ").split() if t.startswith("k_vp8l_palette_")), None)
            if short:
                split[short] = round(split.get(short, 0.0) + ms, 3)
        out["inputs"][name]["palette_kernels_ms"] = split
        out["inputs"][name]["all_kernels_ms"] = round(total, 3)
    L.set_webp_palette(0)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
