"""PNG `--zopfli` on the device: call time with the flag off and on (alternated, median of 5 after a warm-up), the device split of the
k_pz_* kernels (a separate torch.profiler run), and bytes off / on against zlib level 9 of the same filtered stream, for a 4096 x 4096
RGBA photograph, 1920 x 1080 flat art and a 1920 x 1080 text screenshot.  Prints one JSON line.  Needs an H100."""
import json
import os
import statistics
import subprocess
import sys
import time
import zlib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402

import __graft_entry__ as G  # noqa: E402
import png_zopfli_cases as cases  # noqa: E402
from pngutil import idat_stream, pil_png  # noqa: E402


def inputs():
    photo = np.dstack([cases.photo(4096, 4096), np.full((4096, 4096), 255, np.uint8)])
    photo[::3, ::5, 3] = 128
    return {"photo_4096_rgba": pil_png(photo, compress_level=1), "flat_1920x1080": pil_png(cases.flat(1920, 1080), compress_level=1),
            "text_1920x1080": pil_png(cases.text(1920, 1080), compress_level=1)}


def main():
    L = G._pkg()
    assert L.lib().b200_init_device(0) == 0, "no GPU"
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    L.set_png_zopfli(1)
    off_p, on_p = L.default_params(), L.default_params()
    off_p.png_optimize = on_p.png_optimize = 1                  # lossless, level 3
    on_p.png_force_zopfli = 1
    out = {"card": card, "inputs": {}}
    for name, data in inputs().items():
        off, on = L.compress_in_memory(data, off_p), L.compress_in_memory(data, on_p)      # warm-up
        t_off, t_on = [], []
        for _ in range(5):
            for p, acc in ((off_p, t_off), (on_p, t_on)):
                t = time.perf_counter(); L.compress_in_memory(data, p); acc.append((time.perf_counter() - t) * 1e3)
        filt = zlib.decompress(idat_stream(off)[1])
        out["inputs"][name] = {"stream_bytes": len(filt), "ms_off": round(statistics.median(t_off), 1), "ms_on": round(statistics.median(t_on), 1),
                               "bytes_off": len(off), "bytes_on": len(on), "zlib9_idat": len(zlib.compress(filt, 9)),
                               "idat_off": len(idat_stream(off)[1]), "idat_on": len(idat_stream(on)[1])}
    import torch
    from torch.profiler import ProfilerActivity, profile
    for name, data in inputs().items():
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            L.compress_in_memory(data, on_p)
            torch.cuda.synchronize()
        split = {}
        for e in prof.key_averages():
            k = e.key
            if "k_pz_" in k or "k_png_" in k or "DeviceRadixSort" in k:
                short = next((t for t in k.replace("(", " ").replace("<", " ").replace("::", " ").split() if t.startswith(("k_pz_", "k_png_"))), "radix_sort")
                split[short] = round(split.get(short, 0.0) + e.device_time_total / 1e3, 2)
        out["inputs"][name]["device_ms"] = split
    print(json.dumps(out))


if __name__ == "__main__":
    main()
