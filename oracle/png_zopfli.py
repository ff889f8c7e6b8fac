"""ctypes binding of the PNG `--zopfli` twin in oracle/png_zopfli_oracle.c (built into oracle/liboracle.so with the rest of the
oracle) -- TEST INFRASTRUCTURE, NOT PRODUCT CODE."""
import ctypes as C

import numpy as np

from .oracle import lib


def _stream(s):
    return np.frombuffer(bytes(s), np.uint8).copy() if isinstance(s, (bytes, bytearray)) else np.ascontiguousarray(s, np.uint8).reshape(-1)


def constants():
    """{'seg', 'chain', 'k', 'region', 'iters', 'slice'} of png_zopfli_core.h"""
    out = np.zeros(8, np.int32)
    lib().orc_pz_constants(out.ctypes.data_as(C.c_void_p))
    return dict(zip(("seg", "chain", "k", "region", "iters", "slice"), (int(v) for v in out[:6])))


def lz77_zopfli(stream, bpp, stride):
    """orc_png_lz77_zopfli: the whole rule (iterations, scoring, slices) -> uint32 tokens in b200_png_lz77's format."""
    s = _stream(stream)
    tok = np.zeros(max(s.size, 1), np.uint32)
    f = lib().orc_png_lz77_zopfli
    f.restype = C.c_size_t
    nt = f(s.ctypes.data_as(C.c_void_p), C.c_size_t(s.size), int(bpp), int(stride), tok.ctypes.data_as(C.c_void_p))
    return tok[:nt].copy()


def squeeze(stream, bpp, stride, cost):
    """one parse of every segment under one 316-entry cost table -> tokens"""
    s = _stream(stream)
    cost = np.ascontiguousarray(cost, np.uint32)
    assert cost.size == 316
    tok = np.zeros(max(s.size, 1), np.uint32)
    f = lib().orc_pz_squeeze
    f.restype = C.c_size_t
    nt = f(s.ctypes.data_as(C.c_void_p), C.c_size_t(s.size), int(bpp), int(stride), cost.ctypes.data_as(C.c_void_p), tok.ctypes.data_as(C.c_void_p))
    return tok[:nt].copy()


def match_sets(stream, bpp, stride):
    """-> [[(length, distance), ...] per position], each list by increasing distance"""
    s = _stream(stream)
    k = constants()["k"]
    ent = np.zeros((max(s.size, 1), k), np.uint32)
    cnt = np.zeros(max(s.size, 1), np.int32)
    lib().orc_pz_match_sets(s.ctypes.data_as(C.c_void_p), C.c_size_t(s.size), int(bpp), int(stride), ent.ctypes.data_as(C.c_void_p), cnt.ctypes.data_as(C.c_void_p))
    return [[(int(e >> 16) + 3, int(e & 0xFFFF) + 1) for e in ent[i, :cnt[i]]] for i in range(s.size)]


def front(cands):
    """the core's front rule over (length, distance) candidates given in increasing distance -> kept [(length, distance)]"""
    m = len(cands)
    ln = np.array([c[0] for c in cands] or [0], np.int32)
    ds = np.array([c[1] for c in cands] or [0], np.int32)
    out = np.zeros(64, np.uint32)
    k = lib().orc_pz_front(ln.ctypes.data_as(C.c_void_p), ds.ctypes.data_as(C.c_void_p), m, out.ctypes.data_as(C.c_void_p))
    return [(int(e >> 16) + 3, int(e & 0xFFFF) + 1) for e in out[:k]]


def costs(hist):
    """the 316-entry cost table of a token histogram"""
    h = np.ascontiguousarray(hist, np.uint32)
    out = np.zeros(316, np.uint32)
    lib().orc_pz_costs(h.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p))
    return out
