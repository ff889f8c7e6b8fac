"""Compression-quality gap, stated instead of hidden (round-1 verdict item 5): output bytes and PSNR of THIS pipeline (the oracle
writes the same bytes as the CUDA path -- that equality is what the GPU tests assert) next to libjpeg-turbo (Pillow, same
quality number, standard tables, optimised Huffman, progressive) and, for the WebP leg, libwebp (Pillow) at equal -q.
The reference (libcaesium -> mozjpeg with trellis quantisation, deringing and scan optimisation) is expected to produce
SMALLER files than ours at equal -q; libjpeg-turbo, its parent without those three, is the closest stand-in that exists here.
CPU only.  Writes profiles/quality.json.  usage: python tools/quality_report.py [jpeg_trellis | png_zopfli | webp_bpred]
(with a section's name, only that section is recomputed and the others are kept as they are)"""
import io
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from PIL import Image  # noqa: E402
from oracle import oracle as O  # noqa: E402
from tools.synth import synth_jpeg, synth_rgb  # noqa: E402


def psnr(a, b):
    mse = np.mean((a.astype(np.float64) - b.astype(np.float64)) ** 2)
    return 99.0 if mse == 0 else 10 * np.log10(255.0 ** 2 / mse)


def decode_rgb(data):
    im = Image.open(io.BytesIO(data)); im.load()
    return np.asarray(im.convert("RGB"))


def jpeg_rows(name, src_bytes, truth_rgb, qualities, ss_param, pil_ss):
    rows = []
    for q in qualities:
        ours = O.jpeg_lossy(src_bytes, O.params(q, ss_param, True))
        b = io.BytesIO()
        Image.fromarray(decode_rgb(src_bytes)).save(b, "JPEG", quality=q, subsampling=pil_ss, optimize=True, progressive=True)
        turbo = b.getvalue()
        rows.append({"input": name, "quality": q, "ours_bytes": len(ours), "libjpeg_turbo_bytes": len(turbo), "bytes_ratio_ours_over_turbo": round(len(ours) / len(turbo), 4),
                     "ours_psnr_vs_source_pixels": round(psnr(decode_rgb(ours), truth_rgb), 3), "libjpeg_turbo_psnr_vs_source_pixels": round(psnr(decode_rgb(turbo), truth_rgb), 3)})
    return rows


def main():
    O.lib()
    out = {"what": "bytes and PSNR at equal -q: this pipeline (Robidoux quantisation tables as mozjpeg's defaults, no trellis / deringing / scan search) vs libjpeg-turbo via Pillow "
                   "(Annex-K tables, optimised Huffman, progressive) and vs libwebp via Pillow; PSNR against the pixels the source file decodes to",
           "jpeg": [], "webp": []}
    # 4K synthetic set (BASELINE configs[1]): three seeds
    for i in range(3):
        src = synth_jpeg(3840, 2160, i)
        out["jpeg"] += jpeg_rows(f"synthetic 3840x2160 seed {i} (q90 4:2:0 source)", src, decode_rgb(src), (60, 80, 90), 420, 2)
    j0 = open(os.path.join(ROOT, "tests", "golden", "reference_samples", "j0.JPG"), "rb").read()
    sj = O.Jpeg(j0).s
    pil_ss = {(1, 1): 0, (2, 1): 1, (2, 2): 2}[(sj.hs[0], sj.vs[0])]           # "auto" keeps the source's sampling
    out["jpeg"] += jpeg_rows("reference samples/j0.JPG", j0, decode_rgb(j0), (50, 80, 95), 0, pil_ss)
    # WebP leg: 6000x4000 -> 1920 wide at -q 85 is large for a CPU report; a 1920x1280 synthetic frame and j0 at their own size
    from webputil import pil_decode  # noqa: F401
    for name, rgb in (("synthetic 1920x1280", synth_rgb(1920, 1280, 0)), ("reference samples/j0.JPG pixels", decode_rgb(j0))):
        planar = np.ascontiguousarray(rgb.transpose(2, 0, 1))
        for q in (50, 75, 85):
            ours = O.webp_encode(planar, q)[0]
            b = io.BytesIO(); Image.fromarray(rgb).save(b, "WEBP", quality=q, method=4)
            ref = b.getvalue()
            out["webp"].append({"input": name, "quality": q, "ours_bytes": len(ours), "libwebp_bytes": len(ref), "bytes_ratio_ours_over_libwebp": round(len(ours) / len(ref), 4),
                                "ours_psnr": round(psnr(decode_rgb(ours), rgb), 3), "libwebp_psnr": round(psnr(decode_rgb(ref), rgb), 3)})
    # lossy PNG (opt-in device quantiser, full-strength Floyd-Steinberg): colours and RGBA PSNR of the quantiser's palette applied to
    # its indices, next to Pillow's median cut -- dithered with Floyd-Steinberg (its palette applied again with dithering on:
    # Image.quantize ignores `dither` unless a palette is given) and, as Image.quantize(256, MEDIANCUT) returns it, undithered.
    # Pillow here has no libimagequant, so imagequant (the reference's quantiser) cannot be compared.  blur_mae: mean absolute error
    # after a 5x5 box blur, the low-frequency error (banding) that dithering removes and PSNR does not see.
    from oracle.png_quant import png_quantize

    def blur_mae(a, b, k=5):
        d = a.astype(np.float64) - b.astype(np.float64)
        c = np.cumsum(np.cumsum(np.pad(d, ((1, 0), (1, 0), (0, 0))), 0), 1)
        return float(np.abs((c[k:, k:] - c[:-k, k:] - c[k:, :-k] + c[:-k, :-k]) / (k * k)).mean())

    out["png_lossy"] = []
    for i in range(3):
        rgb = synth_rgb(1920, 1280, i)
        rgba = np.concatenate([rgb, np.full(rgb.shape[:2] + (1,), 255, np.uint8)], axis=2)
        im = Image.fromarray(rgb)
        mc = im.quantize(256, method=Image.Quantize.MEDIANCUT)
        pil = {"dithered": np.asarray(im.quantize(palette=mc, dither=Image.Dither.FLOYDSTEINBERG).convert("RGBA")), "undithered": np.asarray(mc.convert("RGBA"))}
        for q in (40, 80, 100):
            pal, idx = png_quantize(rgba, q)
            row = {"input": f"synthetic 1920x1280 seed {i}", "quality": q, "ours_colours": len(pal), "ours_psnr_rgba": round(psnr(pal[idx], rgba), 3),
                   "ours_blur_mae": round(blur_mae(pal[idx], rgba), 3)}
            for k, v in pil.items():
                row[f"pillow_mediancut_256_{k}_psnr_rgba"] = round(psnr(v, rgba), 3)
                row[f"pillow_mediancut_256_{k}_blur_mae"] = round(blur_mae(v, rgba), 3)
            out["png_lossy"].append(row)
    out["jpeg_trellis"] = jpeg_trellis()
    out["png_zopfli"] = png_zopfli()
    out["webp_bpred"] = webp_bpred()
    with open(os.path.join(ROOT, "profiles", "quality.json"), "w") as f:
        json.dump(out, f, indent=1)
    for r in out["jpeg"] + out["webp"] + out["png_lossy"] + out["jpeg_trellis"]["rows"]:
        print(r)


def jpeg_trellis():
    """Trellis quantisation (b200_set_jpeg_trellis; the oracle writes the device's bytes) against plain quantisation: bytes and RGB
    PSNR against the source's decoded pixels at q 50..90 (auto subsampling, progressive), and the BD-rate (bytes at equal PSNR) per
    image.  The lambda constants were tuned on 1280x720 images of the same synthetic generator; j0 and j1 are held out."""
    from oracle import jpeg_trellis as T
    from test_jpeg_trellis_host import bd_rate
    srcs = [(f"synthetic 3840x2160 seed {i} (q90 4:2:0 source)", synth_jpeg(3840, 2160, i)) for i in range(3)]
    srcs += [(f"reference samples/{n}", open(os.path.join(ROOT, "tests", "golden", "reference_samples", n), "rb").read()) for n in ("j0.JPG", "j1.jpg")]
    rows, bd = [], {}
    for name, data in srcs:
        truth = decode_rgb(data)
        curve = {False: ([], []), True: ([], [])}
        for q in (50, 60, 70, 80, 90):
            row = {"input": name, "quality": q}
            for t in (False, True):
                out = T.jpeg_lossy(data, O.params(q, 0, True), trellis=t)
                p = psnr(decode_rgb(out), truth)
                curve[t][0].append(len(out)); curve[t][1].append(p)
                k = "trellis" if t else "plain"
                row[f"{k}_bytes"], row[f"{k}_psnr"] = len(out), round(p, 3)
            row["bytes_ratio_trellis_over_plain"] = round(row["trellis_bytes"] / row["plain_bytes"], 4)
            rows.append(row)
        bd[name] = round(float(bd_rate(curve[False][0], curve[False][1], curve[True][0], curve[True][1])), 3)
    return {"what": "trellis vs plain quantisation, this pipeline (oracle == device); PSNR of RGB against the pixels the source decodes to; "
                    "bd_rate_percent: Bjontegaard delta of bytes at equal PSNR over q 50-90 (negative = trellis smaller)",
            "rows": rows, "bd_rate_percent": bd}


def png_zopfli():
    """PNG --zopfli (b200_set_png_zopfli; the twin's tokens are the device's, and the device's DEFLATE writer is the host writer's twin):
    zlib payload bytes of one filtered stream coded from the default greedy / lazy parse, from the optimal parse (what the device emits
    is the smaller of the two), and by zlib level 9, on the seeded flat-art and text images of the tests at two filter strategies"""
    import zlib
    import png_zopfli_cases as cases
    from oracle import png_zopfli as Z
    import __graft_entry__ as G
    L = G._pkg()
    rows = []
    for name, img in (("flat art 320x200", cases.flat(320, 200)), ("text 320x160", cases.text(320, 160)), ("photograph 256x192", cases.photo(256, 192))):
        for strategy, sname in ((0, "None"), (5, "MinSum")):
            st, bpp, stride = cases.filtered(img, strategy)
            ad = zlib.adler32(st.tobytes())
            greedy = len(L.png_deflate_tokens(O.png_lz77(st, bpp, stride)[0], ad))
            optimal = len(L.png_deflate_tokens(Z.lz77_zopfli(st, bpp, stride), ad))
            z9 = len(zlib.compress(st.tobytes(), 9))
            rows.append({"input": name, "filter": sname, "stream_bytes": int(st.size), "default_bytes": greedy, "zopfli_bytes": optimal,
                         "emitted_bytes": min(greedy, optimal), "zlib9_bytes": z9, "emitted_over_zlib9": round(min(greedy, optimal) / z9, 4),
                         "default_over_zlib9": round(greedy / z9, 4)})
    return {"what": "zlib payload bytes of one filtered stream: the default parse, the --zopfli parse, the smaller of the two (what the device "
                    "emits with the switch and flag on) and zlib level 9; CPU twin, identical to the device's bytes", "rows": rows}


def webp_bpred():
    """Lossy WebP with B_PRED (b200_set_webp_bpred; the twin writes the device's bytes) against the switch-off encoder and libwebp
    (Pillow, method 4): bytes and RGB PSNR (decoded by libwebp) at q 30..90, and the BD-rates (bytes at equal PSNR) per image.  Lambda
    is libwebp's 4x4 one, untuned; the reference samples are held out all the same."""
    from oracle import webp_bpred as B
    from test_webp_bpred_host import bd_rate
    srcs = [(f"synthetic 1280x720 seed {i}", synth_rgb(1280, 720, i)) for i in range(3)]
    for n in ("j0.JPG", "j1.jpg", "w0.webp", "w1.webp"):
        srcs.append((f"reference samples/{n}", decode_rgb(open(os.path.join(ROOT, "tests", "golden", "reference_samples", n), "rb").read())))
    rows, bd_off, bd_lib = [], {}, {}
    for name, rgb in srcs:
        planar = np.ascontiguousarray(rgb.transpose(2, 0, 1))
        curve = {"off": ([], []), "bpred": ([], []), "libwebp": ([], [])}
        for q in (30, 45, 60, 75, 90):
            b = io.BytesIO(); Image.fromarray(rgb).save(b, "WEBP", quality=q, method=4)
            files = {"off": O.webp_encode(planar, q)[0], "bpred": B.webp_bpred_encode(planar, q), "libwebp": b.getvalue()}
            row = {"input": name, "quality": q}
            for k, data in files.items():
                p = psnr(decode_rgb(data), rgb)
                curve[k][0].append(len(data)); curve[k][1].append(p)
                row[f"{k}_bytes"], row[f"{k}_psnr"] = len(data), round(p, 3)
            rows.append(row)
        # a BD-rate needs the two PSNR ranges to overlap; where they do not, there is none to state
        bd = lambda a, b: round(float(bd_rate(*curve[a], *curve[b])), 3) if max(min(curve[a][1]), min(curve[b][1])) < min(max(curve[a][1]), max(curve[b][1])) else None
        bd_off[name], bd_lib[name] = bd("off", "bpred"), bd("libwebp", "bpred")
    return {"what": "lossy WebP with B_PRED vs the switch-off encoder and vs libwebp (Pillow, method 4) at equal -q; PSNR of RGB against "
                    "the source pixels, decoded by libwebp; BD-rate: Bjontegaard delta of bytes at equal PSNR over q 30-90 (negative = B_PRED smaller), "
                    "null where the PSNR ranges do not overlap",
            "rows": rows, "bd_rate_percent_vs_switch_off": bd_off, "bd_rate_percent_vs_libwebp": bd_lib}


SECTIONS = {"jpeg_trellis": (jpeg_trellis, lambda r: r["bd_rate_percent"]), "png_zopfli": (png_zopfli, lambda r: r["rows"]),
            "webp_bpred": (webp_bpred, lambda r: [r["bd_rate_percent_vs_switch_off"], r["bd_rate_percent_vs_libwebp"]])}

if __name__ == "__main__":
    if len(sys.argv) == 2 and sys.argv[1] in SECTIONS:
        O.lib()
        fn, show = SECTIONS[sys.argv[1]]
        path = os.path.join(ROOT, "profiles", "quality.json")
        with open(path) as f:
            rep = json.load(f)
        rep[sys.argv[1]] = fn()
        with open(path, "w") as f:
            json.dump(rep, f, indent=1)
        print(json.dumps(show(rep[sys.argv[1]])))
    else:
        main()
