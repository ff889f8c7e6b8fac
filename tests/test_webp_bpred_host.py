"""The lossy WebP B_PRED twin (oracle/webp_bpred_oracle.c) on the CPU: every file it writes decodes through libwebp (Pillow) and
through the project's own VP8 decoder to exactly its own reconstruction; the cases exercise every sub-block mode, both kinds of
macroblock and a Y2 context carried across B_PRED macroblocks; the host writer rebuilds the twin's file from its stage output; a
first partition past 19 bits is refused cleanly; the switch's C header and its refusals; and the size at equal quality."""
import io
import os
import re
import subprocess

import numpy as np
import pytest

from pngutil import synth
from test_webp_host import CASES
from webputil import decode_like_libwebp, pil_decode

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "caesium-clt_b200")
BP_CASES = CASES + [(16, 40, 50, "photo"), (40, 16, 65, "noise"), (17, 33, 70, "noise"), (33, 17, 20, "flat"), (1, 1, 30, "photo"),
                    (96, 160, 40, "photo"), (64, 64, 100, "noise")]


@pytest.fixture(scope="module")
def OB(O):
    from oracle import webp_bpred
    return webp_bpred


def planar(img):
    return np.ascontiguousarray(img.transpose(2, 0, 1))


def _case(h, w, q, kind):
    return planar(synth(h, w, 3, seed=h + w + q, kind=kind))


@pytest.mark.parametrize("h,w,q,kind", BP_CASES)
def test_twin_files_decode_to_the_twin_reconstruction(L, OB, h, w, q, kind):
    st = OB.webp_bpred_stages(_case(h, w, q, kind), q)
    data = st["file"]
    assert data[:4] == b"RIFF" and data[8:16] == b"WEBPVP8 " and int.from_bytes(data[4:8], "little") == len(data) - 8
    want = decode_like_libwebp(st["Y"], st["U"], st["V"], w, h)
    assert np.array_equal(pil_decode(data), want)
    assert np.array_equal(L.webp_decode(data), want)


@pytest.mark.parametrize("q", [0, 25, 50, 75, 90, 100])
def test_twin_decodes_exactly_at_every_quality(L, OB, q):
    st = OB.webp_bpred_stages(_case(48, 80, q, "photo"), q)
    want = decode_like_libwebp(st["Y"], st["U"], st["V"], 80, 48)
    assert np.array_equal(pil_decode(st["file"]), want) and np.array_equal(L.webp_decode(st["file"]), want)


def _carried_y2(levels, modes, mbw):
    """i16 macroblocks whose Y2 context (from above or from the left) is 1 only through a B_PRED macroblock in between"""
    nmb = len(modes)
    mbh = nmb // mbw
    skip_used = modes[:, 2].any()
    flag = lambda mb: 0 if (skip_used and modes[mb, 2]) else int(levels[mb, 0].any())
    n = 0
    for mb in range(nmb):
        if modes[mb, 0] == 4 or (skip_used and modes[mb, 2]):
            continue
        y, x = divmod(mb, mbw)
        for step, lim in ((-mbw, y), (-1, x)):
            j, k = mb + step, 1
            while k <= lim and modes[j, 0] == 4:
                j += step; k += 1
            if k > 1 and k <= lim and flag(j):
                n += 1
    return n


def test_cases_exercise_bpred(OB):
    seen, nbp, ni16, carried = set(), 0, 0, 0
    for (h, w, q, kind) in BP_CASES:
        st = OB.webp_bpred_stages(_case(h, w, q, kind), q)
        m = st["modes"]
        bp = m[:, 0] == 4
        nbp += int(bp.sum()); ni16 += int((~bp).sum())
        seen |= set(st["bmodes"][bp].ravel().tolist())
        assert (st["levels"][bp, 0] == 0).all() and (st["bmodes"][~bp] == m[~bp, :1]).all()
        carried += _carried_y2(st["levels"], m, (w + 15) // 16)
    assert seen == set(range(10)) and nbp > 0 and ni16 > 0 and carried > 0, (seen, nbp, ni16, carried)


@pytest.mark.parametrize("h,w,q,kind", BP_CASES)
def test_host_writer_reproduces_the_twin_file(L, OB, h, w, q, kind):
    st = OB.webp_bpred_stages(_case(h, w, q, kind), q)
    assert L.webp_write_levels_bpred(w, h, q, st["levels"], st["modes"], st["bmodes"]) == st["file"]


def test_first_partition_overflow_is_refused(L):
    """All-B_PRED 4096x4096 frame with context-expensive sub-block modes: its modes alone need more than 2^19 bytes"""
    w = h = 4096
    nmb = (w // 16) * (h // 16)
    rng = np.random.default_rng(1)
    levels = np.zeros((nmb, 25, 16), np.int16)
    modes = np.zeros((nmb, 4), np.uint8); modes[:, 0] = 4; modes[:, 2] = 1
    bmodes = rng.integers(4, 10, (nmb, 16)).astype(np.uint8)
    with pytest.raises(L.B200Error) as e:
        L.webp_write_levels_bpred(w, h, 90, levels, modes, bmodes)
    assert e.value.code == 1
    small = L.webp_write_levels_bpred(256, 256, 90, levels[:256], modes[:256], bmodes[:256])
    assert pil_decode(small).shape == (256, 256, 3)


def test_writers_refuse_what_they_cannot_write(L, OB):
    st = OB.webp_bpred_stages(_case(32, 32, 60, "noise"), 60)
    assert (st["modes"][:, 0] == 4).any()
    with pytest.raises(L.B200Error) as e:
        L.webp_write_levels(32, 32, 60, st["levels"], st["modes"])
    assert e.value.code == 1
    bad = st["bmodes"].copy(); bad[st["modes"][:, 0] == 4, 5] = 10
    with pytest.raises(L.B200Error) as e:
        L.webp_write_levels_bpred(32, 32, 60, st["levels"], st["modes"], bad)
    assert e.value.code == 1


def test_switch_refuses_other_values(L):
    assert L.set_webp_bpred(2) != 0 and L.set_webp_bpred(-1) != 0
    assert L.set_webp_bpred(0) == 0


def test_header_is_c99_and_links(tmp_path):
    exe = str(tmp_path / "c_abi_webp_bpred_check")
    cmd = ["gcc", "-std=c99", "-pedantic", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"),
           os.path.join(ROOT, "tests", "c_abi_webp_bpred_check.c"), "-o", exe, "-L", PKG, "-lb200caesium", "-Wl,-rpath," + PKG]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0 and "webp bpred c-abi ok" in r.stdout, (r.returncode, r.stdout, r.stderr)
    hdr = open(os.path.join(ROOT, "include", "b200_caesium_webp_bpred.h")).read()
    declared = set(re.findall(r"^[a-z_0-9 ]+\b(b200_[a-z0-9_]+)\(", hdr, re.M))
    src = open(os.path.join(ROOT, "tests", "c_abi_webp_bpred_check.c")).read()
    assert declared == {"b200_set_webp_bpred", "b200_webp_encode_rgb_bpred", "b200_webp_write_levels_bpred"}
    assert all("(fn)" + f in src for f in declared)


def _psnr(a, b):
    mse = np.mean((a.astype(np.float64) - b.astype(np.float64)) ** 2)
    return 99.0 if mse == 0 else 10 * np.log10(255.0 ** 2 / mse)


def bd_rate(r1, p1, r2, p2):
    """Bjontegaard delta rate of curve 2 against curve 1 (percent; negative = smaller files at equal PSNR)"""
    l1, l2 = np.log(r1), np.log(r2)
    c1, c2 = np.polyfit(p1, l1, 3), np.polyfit(p2, l2, 3)
    lo, hi = max(min(p1), min(p2)), min(max(p1), max(p2))
    i1, i2 = np.polyint(c1), np.polyint(c2)
    a1 = np.polyval(i1, hi) - np.polyval(i1, lo); a2 = np.polyval(i2, hi) - np.polyval(i2, lo)
    return (np.exp((a2 - a1) / (hi - lo)) - 1) * 100


def rd_curves(O, OB, rgb, qs=(30, 45, 60, 75, 90)):
    """(bytes, RGB PSNR) per quality for the switch-off twin and the B_PRED twin, decoded through libwebp"""
    src = rgb.transpose(1, 2, 0)
    off, on = [], []
    for q in qs:
        a = O.webp_encode(rgb, q)[0]; b = OB.webp_bpred_encode(rgb, q)
        off.append((len(a), _psnr(pil_decode(a), src))); on.append((len(b), _psnr(pil_decode(b), src)))
    return off, on


@pytest.mark.parametrize("name", ["j0.JPG", "w0.webp"])
def test_bd_rate_against_the_switch_off_encoder_on_held_out_samples(O, OB, name):
    from PIL import Image
    path = os.path.join(ROOT, "tests", "golden", "reference_samples", name)
    if not os.path.exists(path):
        pytest.skip("reference sample not in the tree")
    im = Image.open(path).convert("RGB")
    im.thumbnail((512, 512))
    off, on = rd_curves(O, OB, np.ascontiguousarray(np.asarray(im).transpose(2, 0, 1)))
    bd = bd_rate(*map(np.array, zip(*off)), *map(np.array, zip(*on)))
    assert bd < 0, (bd, off, on)
