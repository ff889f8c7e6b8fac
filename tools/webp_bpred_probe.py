"""Lossy WebP with the B_PRED switch on against off, on the device: call time (alternated, median of 5 after a warm-up), the device
time of the VP8 kernels (k_vp8_encode vs k_vp8_encode_bpred, a separate torch.profiler run), bytes and RGB PSNR (decoded by the
project's decoder), at 1920x1080 and 3840x2160 on a synthetic photograph and on the reference sample j0.JPG, quality 75.  The card's
name and power limit are read in the same command.  Prints one JSON line.  Needs an H100."""
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
from pngutil import synth  # noqa: E402


def inputs():
    j0 = Image.open(os.path.join(ROOT, "tests", "golden", "reference_samples", "j0.JPG")).convert("RGB")
    out = {}
    for (w, h) in ((1920, 1080), (3840, 2160)):
        out[f"synth_{w}x{h}"] = synth(h, w, 3, seed=7, kind="photo")
        out[f"j0_{w}x{h}"] = np.asarray(j0.resize((w, h), Image.LANCZOS))
    return {k: np.ascontiguousarray(v.transpose(2, 0, 1)) for k, v in out.items()}


def psnr(a, b):
    mse = np.mean((a.astype(np.float64) - b.astype(np.float64)) ** 2)
    return float(10 * np.log10(255.0 ** 2 / mse)) if mse else 99.0


def kernel_ms(L, img, q):
    import torch
    from torch.profiler import ProfilerActivity, profile
    res = {}
    for on in (0, 1):
        L.set_webp_bpred(on)
        L.webp_encode_rgb(img, q)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(3):
                L.webp_encode_rgb(img, q)
            torch.cuda.synchronize()
        for e in prof.key_averages():
            if "k_vp8_encode" in e.key:
                res["bpred" if "bpred" in e.key else "i16"] = round(e.device_time_total / 3 / 1000.0, 3)
    L.set_webp_bpred(0)
    return res


def main():
    L = G._pkg()
    assert L.lib().b200_init_device(0) == 0
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    q = 75
    rows = {}
    for name, img in inputs().items():
        src = img.transpose(1, 2, 0)
        t = {0: [], 1: []}
        files = {}
        for on in (0, 1):
            L.set_webp_bpred(on); files[on] = L.webp_encode_rgb(img, q)
        for _ in range(5):
            for on in (0, 1):
                L.set_webp_bpred(on)
                a = time.perf_counter(); L.webp_encode_rgb(img, q); t[on].append((time.perf_counter() - a) * 1e3)
        L.set_webp_bpred(0)
        rows[name] = {"call_ms_off": round(statistics.median(t[0]), 2), "call_ms_on": round(statistics.median(t[1]), 2),
                      "bytes_off": len(files[0]), "bytes_on": len(files[1]),
                      "psnr_off": round(psnr(L.webp_decode(files[0]), src), 3), "psnr_on": round(psnr(L.webp_decode(files[1]), src), 3)}
        if name.startswith("synth"):
            rows[name]["kernel_ms"] = kernel_ms(L, img, q)
    print(json.dumps({"gpu": smi, "quality": q, "results": rows}))


if __name__ == "__main__":
    main()
