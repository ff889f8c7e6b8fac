"""PNG `--zopfli` on the CPU: the twin (oracle/png_zopfli_oracle.c over png_zopfli_core.h) against the plain-Python statement of
the rules (tests/pz_reference.py), the validity of its tokens, the size it reaches against zlib level 9, and the switch."""
import os
import re
import subprocess
import sys
import zlib

import numpy as np
import pytest

import png_zopfli_cases as cases
import pz_reference as R

ROOT = cases.ROOT
PKG = os.path.join(ROOT, "caesium-clt_b200")
from oracle import oracle as O  # noqa: E402
from oracle import png_zopfli as Z  # noqa: E402


def test_constants_are_the_documented_ones():
    assert Z.constants() == {"seg": 32768, "chain": 32, "k": 8, "region": 262144, "iters": 15, "slice": 8 << 20}


# ---- the rule against the reference ---------------------------------------------------------------------------------------
def test_cost_tables_match_the_reference():
    rng = np.random.default_rng(5)
    for trial in range(40):
        h = np.zeros(316, np.uint32)
        nz = rng.choice(316, int(rng.integers(0, 316)), replace=False)
        h[nz] = rng.integers(1, [2, 100, 10 ** 6][trial % 3], nz.size)
        assert list(Z.costs(h)) == R.costs([int(v) for v in h]), trial


@pytest.mark.parametrize("seed", range(30))
def test_front_and_pruning_match_the_reference(seed):
    rng = np.random.default_rng(seed)
    m = int(rng.integers(0, 40))
    cands = [(int(rng.integers(0, 259)), int(d)) for d in sorted(rng.choice(32768, m, replace=False) + 1)]
    if seed % 3 == 0:                                    # long fronts: every candidate longer than the one before
        cands = [(3 + k, 10 * k + 1) for k in range(m)]
    assert Z.front(cands) == R.front(cands, 8), cands


def _reference_parse(stream, bpp, stride, cost):
    s = [int(v) for v in stream]
    full = [R.exhaustive_set(s, i) for i in range(len(s))]
    twin_sets = Z.match_sets(stream, bpp, stride)
    ref_toks, ref_cost = R.shortest_path(s, full, cost)
    return s, full, twin_sets, ref_toks, ref_cost


def _hist_costs(stream, bpp, stride):
    """a realistic table: the greedy parse's statistics"""
    _, hist = O.png_lz77(np.ascontiguousarray(stream, np.uint8), bpp, stride)
    return [int(v) for v in Z.costs(hist)]


@pytest.mark.parametrize("kind", ["runs", "text", "pixels", "random", "periodic"])
def test_parse_matches_the_exhaustive_reference(kind):
    rng = np.random.default_rng(len(kind))
    n = 400
    if kind == "runs":
        st = np.repeat(rng.integers(0, 4, 40, dtype=np.uint8), rng.integers(1, 20, 40))[:n]
    elif kind == "text":
        st = np.frombuffer((b"the cost of a match is its length symbol and its distance symbol " * 8)[:n], np.uint8)
    elif kind == "pixels":
        st = cases.filtered(cases.flat(12, 10, 7))[0][:n]
    elif kind == "random":
        st = rng.integers(0, 3, n, dtype=np.uint8)
    else:
        st = np.tile(rng.integers(0, 256, 37, dtype=np.uint8), 20)[:n]
    bpp, stride = 3, 37
    cost = _hist_costs(st, bpp, stride)
    s, full, twin_sets, ref_toks, ref_cost = _reference_parse(st, bpp, stride, cost)
    twin = [int(t) for t in Z.squeeze(st, bpp, stride, np.array(cost, np.uint32))]
    assert R.parse_cost(s, twin, cost) >= ref_cost
    # where neither the chain depth nor PZ_K binds, the kept set is the full front and the parse is the reference's, token for token
    if twin_sets == full:
        assert twin == ref_toks
    # the twin's parse is the shortest path over the twin's own sets, whatever binds
    assert twin == R.shortest_path(s, twin_sets, cost)[0]
    # and every kept set is the full front pruned by the rule, or (chain depth binding) a front of a subset of the candidates
    for i, (t, f) in enumerate(zip(twin_sets, full)):
        assert all(l <= R.maxlen(i, len(s)) and 1 <= d <= min(i, 32768) for l, d in t), i
        assert all(any(fl >= l and fd <= d for fl, fd in f) for l, d in t), i


def test_small_streams_are_fully_unbound_somewhere():
    """the exact-equality branch above is exercised: on short-range data the chain depth and PZ_K never bind"""
    st = np.frombuffer((b"abcabcabdabcabcabd" * 12)[:200], np.uint8)
    s = [int(v) for v in st]
    assert Z.match_sets(st, 3, 37) == [R.exhaustive_set(s, i) for i in range(len(s))]


# ---- whole-rule outputs ----------------------------------------------------------------------------------------------------
def _check_tokens(stream, toks):
    """expands to the stream; every match reaches back no further than its position, repeats equal bytes and stays in its segment"""
    s = np.ascontiguousarray(stream, np.uint8)
    assert np.array_equal(O.png_expand(toks, s.size), s)
    p = 0
    for t in toks:
        t = int(t)
        if t & 0x80000000:
            l, d = ((t >> 16) & 0x7FFF) + 3, (t & 0xFFFF) + 1
            assert 3 <= l <= 258 and 1 <= d <= min(p, 32768)
            assert p // cases.SEG == (p + l - 1) // cases.SEG
            assert np.array_equal(s[p:p + l], s[p - d:p - d + l])
            p += l
        else:
            assert t < 256 and s[p] == t
            p += 1
    assert p == s.size


@pytest.mark.parametrize("name", ["photo", "flat", "text", "noise", "one_wide"])
def test_twin_tokens_are_valid_on_images(name):
    st, bpp, stride = cases.filtered(cases.images()[name])
    _check_tokens(st, Z.lz77_zopfli(st, bpp, stride))


@pytest.mark.parametrize("n", [0, 1, 2, 3, cases.SEG - 1, cases.SEG, cases.SEG + 1])
def test_twin_tokens_are_valid_at_boundaries(n):
    st, bpp, stride = cases.boundary_stream(n)
    toks = Z.lz77_zopfli(st, bpp, stride)
    if n == 0:
        assert toks.size == 0
    else:
        _check_tokens(st, toks)


def test_twin_tokens_are_valid_past_one_slice():
    st, bpp, stride = cases.boundary_stream(cases.SLICE + 1)
    _check_tokens(st, Z.lz77_zopfli(st, bpp, stride))


@pytest.mark.parametrize("name", ["flat", "text"])
def test_size_bar_against_zlib_9(L, name):
    """flat art and text: the twin's tokens, coded by the host writer, are no larger than zlib level 9 of the same filtered stream"""
    img = {"flat": cases.flat(320, 200), "text": cases.text(320, 160)}[name]
    st, bpp, stride = cases.filtered(img)
    z = L.png_deflate_tokens(Z.lz77_zopfli(st, bpp, stride), zlib.adler32(st.tobytes()))
    assert zlib.decompress(z) == st.tobytes()
    assert len(z) <= len(zlib.compress(st.tobytes(), 9))


# ---- the switch ------------------------------------------------------------------------------------------------------------
def test_setter_accepts_0_and_1_only(L):
    try:
        assert L.set_png_zopfli(0) == 0 and L.set_png_zopfli(1) == 0
        for bad in (2, -1, 255):
            assert L.set_png_zopfli(bad) == L.ERR_INVALID_ARGUMENT
    finally:
        L.set_png_zopfli(0)


def test_stage_entry_refuses_bad_arguments_before_the_device(L):
    for args in ((np.zeros(0, np.uint8), 1, 4), (np.zeros(8, np.uint8), 0, 4), (np.zeros(8, np.uint8), 9, 4), (np.zeros(8, np.uint8), 1, 0)):
        with pytest.raises(Exception) as e:
            L.png_lz77_zopfli(*args)
        assert getattr(e.value, "code", None) == L.ERR_INVALID_ARGUMENT


def test_switch_is_decided_in_one_place():
    """the switch goes through the OptIn table (its variable B200_PNG_ZOPFLI read once), and png_force_zopfli is combined with it in
    exactly one expression, which every PNG back-end call takes its device from"""
    src = open(os.path.join(PKG, "csrc", "api.cpp")).read()
    assert 'OptIn g_png_zopfli{"B200_PNG_ZOPFLI"}' in src
    assert len(re.findall(r"g_png_zopfli\.on\(\)", src)) == 1
    assert len(re.findall(r"p->png_force_zopfli &&", src)) == 1
    for call in ("code_unfiltered", "code_quantized", "->compress("):
        assert "s->png_dev()->" + call.lstrip("->") not in src, call


def test_header_is_c99_and_links(tmp_path):
    exe = str(tmp_path / "c_abi_png_zopfli_check")
    cmd = ["gcc", "-std=c99", "-pedantic", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"),
           os.path.join(ROOT, "tests", "c_abi_png_zopfli_check.c"), "-o", exe, "-L", PKG, "-lb200caesium", "-Wl,-rpath," + PKG]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0 and "png zopfli c-abi ok" in r.stdout, (r.returncode, r.stdout, r.stderr)
    hdr = open(os.path.join(ROOT, "include", "b200_caesium_png_zopfli.h")).read()
    declared = set(re.findall(r"^[a-z_0-9 ]+\b(b200_[a-z0-9_]+)\(", hdr, re.M))
    src = open(os.path.join(ROOT, "tests", "c_abi_png_zopfli_check.c")).read()
    assert declared == {"b200_set_png_zopfli", "b200_png_lz77_zopfli"} and all("(fn)" + f in src for f in declared)
