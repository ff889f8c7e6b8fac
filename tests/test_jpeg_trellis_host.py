"""Trellis quantisation, CPU side: the oracle's orc_quantize_trellis (oracle/jpeg_trellis_oracle.c over csrc/jpeg_trellis_core.h) against an independent brute
force and dynamic programme (tests/jt_reference.py, written from the rule in the header comment), its invariants on every block of
j0.JPG, its files, its quality against plain quantisation, and the C declarations of the opt-in header."""
import io
import os
import struct
import subprocess
import sys

import numpy as np
import pytest
from PIL import Image

import jt_reference as R
from oracle import jpeg_trellis as T

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools.synth import synth_jpeg  # noqa: E402

ZZ = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28,
               35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63])
XMAX = 8192                       # |FDCT output| <= 2^13 for 8-bit samples (test_fdct_output_bound; the DC of a black block)


def _sample(name):
    with open(os.path.join(ROOT, "tests", "golden", "reference_samples", name), "rb") as f:
        return f.read()


def trellis_zz(O, xz, qz, chroma):
    """oracle trellis on a zigzag block -> zigzag levels"""
    nat = np.zeros(64, np.int32)
    nat[ZZ] = xz
    qn = np.zeros(64, np.uint16)
    qn[ZZ] = qz
    return [int(v) for v in T.quantize_trellis(nat, qn, chroma).reshape(64)[ZZ]]


def sparse_block(rng, qz, nnz, run_long=False, last63=False):
    """|x| within the FDCT bound; nnz positions with plain level != 0, every other AC position rounds to zero"""
    xz = np.zeros(64, np.int64)
    xz[0] = rng.integers(-XMAX, XMAX + 1)
    for k in range(1, 64):                       # below half a step: plain level 0
        h = min(4 * int(qz[k]) - 1, XMAX)
        xz[k] = rng.integers(-h, h + 1)
    ks = list(rng.choice(np.arange(1, 64), nnz, replace=False)) if nnz else []
    if run_long and nnz:
        ks[0] = int(rng.integers(17, 64))        # a run of >= 16 zeros before it (ZRL)
    if last63 and nnz:
        ks[-1] = 63
    for k in ks:
        d = 8 * int(qz[k])
        top = min(XMAX // d, 40)
        if top < 1:
            continue
        lvl = int(rng.integers(1, top + 1))
        v = lvl * d + int(rng.integers(-d // 2, d // 2))
        xz[k] = min(v, XMAX) * (1 if rng.random() < 0.5 else -1)
    return xz


@pytest.mark.parametrize("q", [10, 50, 80, 95])
@pytest.mark.parametrize("chroma", [0, 1])
def test_reaches_the_brute_force_minimum(O, q, chroma):
    rng = np.random.default_rng(q * 2 + chroma)
    qz = O.quant_table(q, chroma)[ZZ].astype(np.int64)
    done = 0
    for i in range(60):
        xz = sparse_block(rng, qz, int(rng.integers(0, 6)), run_long=i % 3 == 0, last63=i % 4 == 1)
        p = [R.plain(int(xz[k]), int(qz[k])) for k in range(64)]
        if sum(1 for v in p[1:] if v) > 5:
            continue
        best, _ = R.brute_force(xz, qz, chroma)
        got = trellis_zz(O, xz, qz, chroma)
        assert R.cost(xz, qz, got, chroma) == best, (i, got)
        done += 1
    assert done >= 40


def test_brute_force_covers_zrl_and_position_63(O):
    """one hand-made block each: a lone level after a 40-zero run, and a level at 63 behind a 16-zero run"""
    qz = O.quant_table(50, 0)[ZZ].astype(np.int64)
    for ks in ([41], [5, 22, 63]):
        xz = np.zeros(64, np.int64)
        xz[0] = 300
        for j, k in enumerate(ks):
            xz[k] = (3 + j) * 8 * int(qz[k]) * (-1) ** j
        best, _ = R.brute_force(xz, qz, 0)
        got = trellis_zz(O, xz, qz, 0)
        assert R.cost(xz, qz, got, 0) == best


@pytest.mark.parametrize("q", [10, 50, 80, 95, 100])
def test_matches_an_independent_dp_on_dense_blocks(O, q):
    rng = np.random.default_rng(1000 + q)
    for chroma in (0, 1):
        qz = O.quant_table(q, chroma)[ZZ].astype(np.int64)
        for _ in range(200):
            scale = rng.choice([0.3, 1.0, 3.0])
            xz = np.clip(np.round(rng.laplace(0, scale * 8 * qz / (1 + np.arange(64) / 16))), -XMAX, XMAX).astype(np.int64)
            assert trellis_zz(O, xz, qz, chroma) == R.dp(xz, qz, chroma)


def test_fdct_output_bound(O):
    """the raw coefficients the device stores as int16 (and the core's 64-bit products) assume |x| <= 2^13"""
    q1 = np.ones(64, np.uint16)
    yy, xx = np.mgrid[:8, :8]
    blocks = [np.zeros((8, 8)), np.full((8, 8), 255), ((yy + xx) % 2) * 255, (xx < 4) * 255, (yy < 4) * 255, ((yy < 4) ^ (xx < 4)) * 255]
    for u in range(8):
        for v in range(8):
            basis = np.cos((2 * yy + 1) * u * np.pi / 16) * np.cos((2 * xx + 1) * v * np.pi / 16)
            blocks += [(basis > 0) * 255, (basis < 0) * 255]
    worst = max(int(np.abs(O.fdct_quant(b.astype(np.uint8), q1)[0]).max()) for b in blocks)
    assert 8000 < worst <= XMAX


def _standard_ac_lengths():
    """AC code lengths of the Annex K tables as libjpeg writes them into a file encoded without optimisation"""
    b = io.BytesIO()
    Image.fromarray(np.zeros((16, 16, 3), np.uint8)).save(b, "JPEG", quality=75, optimize=False)
    d, i, out = b.getvalue(), 2, {}
    while i < len(d):
        marker, length = d[i + 1], struct.unpack(">H", d[i + 2:i + 4])[0]
        if marker == 0xC4:
            j = i + 4
            while j < i + 2 + length:
                tc, th = d[j] >> 4, d[j] & 15
                counts = list(d[j + 1:j + 17])
                syms = d[j + 17:j + 17 + sum(counts)]
                if tc == 1:
                    L, s = {}, 0
                    for n, c in enumerate(counts, 1):
                        for _ in range(c):
                            L[syms[s]] = n
                            s += 1
                    out[th] = L
                j += 17 + sum(counts)
        if marker == 0xDA:
            break
        i += 2 + length
    return out


def test_annex_k_lengths():
    std = _standard_ac_lengths()
    for th in (0, 1):
        mine = R.ac_lengths(th)
        assert all(mine[s] == n for s, n in std[th].items())
        assert len(std[th]) == 162


def _blocks(j, c):
    co = j.coef(c)
    return co[: j.s.rbh[c], : j.s.rbw[c]].reshape(-1, 64)


def test_invariants_on_every_block_of_j0(O):
    src = O.Jpeg(_sample("j0.JPG")).decode_native()
    for q in (50, 80):
        plain, trel = O.forward(src, O.params(q, 0, True)), T.forward(src, O.params(q, 0, True))
        for c in range(plain.ncomp):
            p, t = _blocks(plain, c), _blocks(trel, c)
            assert np.array_equal(p[:, 0], t[:, 0])
            assert np.all((t == 0) | ((np.sign(t) == np.sign(p)) & (np.abs(t) <= np.abs(p))))
            flat = ~np.any(p[:, 1:], axis=1)
            assert np.array_equal(p[flat], t[flat])
            assert np.any(t != p)


@pytest.mark.parametrize("name", ["in_420_base_355x237.jpg", "in_422_base_355x237.jpg", "in_gray_base_355x237.jpg", "in_420_tiny_17x9.jpg"])
def test_composed_flows_are_the_oracle_flows(O, golden, name):
    """oracle/jpeg_trellis.py composes the lossy and resize flows from the oracle's stages; without the trellis they must be the
    oracle's own flows byte for byte, so the trellis files differ from the plain ones only by the quantiser"""
    data = golden(name)
    for q, ss, prog in ((80, 420, True), (60, 444, False)):
        p = O.params(q, ss, prog)
        assert T.jpeg_lossy(data, p, trellis=False) == O.jpeg_lossy(data, p)
        assert T.jpeg_lossy_resized(data, p, 100, 0, trellis=False) == O.jpeg_lossy_resized(data, p, 100, 0)


def _psnr(a, b):
    return 10 * np.log10(255.0 ** 2 / np.mean((a.astype(np.float64) - b.astype(np.float64)) ** 2))


def _rgb(data):
    im = Image.open(io.BytesIO(data))
    im.load()
    return np.asarray(im.convert("RGB"))


def bd_rate(r0, p0, r1, p1):
    """Bjontegaard delta rate (%) of curve 1 against curve 0: cubic fits of log bytes over PSNR, averaged on the overlap"""
    c0, c1 = np.polyfit(p0, np.log(r0), 3), np.polyfit(p1, np.log(r1), 3)
    lo, hi = max(min(p0), min(p1)), min(max(p0), max(p1))
    i0 = np.diff(np.polyval(np.polyint(c0), [lo, hi]))[0]
    i1 = np.diff(np.polyval(np.polyint(c1), [lo, hi]))[0]
    return (np.exp((i1 - i0) / (hi - lo)) - 1) * 100


QUALITIES = (50, 60, 70, 80, 90)
SET = [("synthetic 1280x720 seed %d" % i, lambda i=i: synth_jpeg(1280, 720, i)) for i in range(3)] + [("j1.jpg", lambda: _sample("j1.jpg"))]


@pytest.mark.parametrize("name,make", SET, ids=[n for n, _ in SET])
def test_smaller_files_and_negative_bd_rate(O, name, make):
    data = make()
    truth = _rgb(data)
    curves = {False: ([], []), True: ([], [])}
    for q in QUALITIES:
        for t in (False, True):
            out = T.jpeg_lossy(data, O.params(q, 0, True), trellis=t)
            rgb = _rgb(out)                                       # every trellis file decodes in Pillow
            assert rgb.shape == truth.shape
            curves[t][0].append(len(out))
            curves[t][1].append(_psnr(rgb, truth))
    for i, q in enumerate(QUALITIES):
        if q in (60, 80, 90):
            assert curves[True][0][i] < curves[False][0][i], (q, curves[True][0][i], curves[False][0][i])
    assert bd_rate(curves[False][0], curves[False][1], curves[True][0], curves[True][1]) < 0


def test_opt_in_header_is_c99(tmp_path):
    src = tmp_path / "jpeg_trellis_abi.c"
    src.write_text('#include "b200_caesium_jpeg_trellis.h"\n'
                   "typedef int (*fn)(int);\n"
                   "int main(void) { fn f = b200_set_jpeg_trellis; return f == 0; }\n")
    pkg = os.path.join(ROOT, "caesium-clt_b200")
    exe = str(tmp_path / "jpeg_trellis_abi")
    r = subprocess.run(["gcc", "-std=c99", "-pedantic", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", exe,
                        "-L", pkg, "-lb200caesium", "-Wl,-rpath," + pkg], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert subprocess.run([exe]).returncode == 0
