"""Plain restatement of the JPEG trellis quantiser's cost (caesium-clt_b200/csrc/jpeg_trellis_core.h, header comment), written
from that definition and not from the C: exact Python integers, blocks in zigzag order.  Used by tests/test_jpeg_trellis_host.py."""
import itertools

import numpy as np

A, B, RATE_SHIFT = 1 << 20, 92682, 16

# JPEG standard, Annex K: (number of codes of each length 1..16, the symbols in code order) of tables K.5 and K.6
_K5 = ([0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d],
       [0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14, 0x32,
        0x81, 0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82])
_K6 = ([0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77],
       [0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32, 0x81,
        0x08, 0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16, 0x24, 0x34,
        0xe1, 0x25, 0xf1])


def ac_lengths(chroma):
    counts, syms = _K6 if chroma else _K5
    L = [16] * 256
    i = 0
    for length, n in enumerate(counts, start=1):
        for _ in range(n):
            if i < len(syms):
                L[syms[i]] = length
            i += 1
    return L


def size(v):
    return abs(int(v)).bit_length()


def plain(x, q):
    l = (abs(x) + 4 * q) // (8 * q)
    return -l if x < 0 else l


def lam(x):
    S = sum(int(v) * int(v) for v in x[1:])
    return (63 * A * (1 << 24)) // (63 * B + S)


def dist(x, c, q, lm):
    w = (1 << 31) // (q * q)
    e = abs(x) - 8 * abs(c) * q
    return (((e * e * w) >> 20) * lm) >> 19


def candidates(p):
    """allowed magnitudes at a position whose plain level is p"""
    a = abs(p)
    if a == 0:
        return [0]
    return [0, a] + [(1 << s) - 1 for s in range(1, a.bit_length())]


def rate(levels, L):
    """bits of the AC levels under the sequential model (zigzag positions 1..63)"""
    bits, run, last = 0, 0, 0
    for k in range(1, 64):
        c = int(levels[k])
        if c == 0:
            run += 1
            continue
        s = size(c)
        bits += (run // 16) * L[0xF0] + L[((run % 16) << 4) | s] + s
        run, last = 0, k
    if last < 63:
        bits += L[0x00]
    return bits


def cost(x, q, levels, chroma):
    x = [int(v) for v in x]
    q = [int(v) for v in q]
    lm = lam(x)
    d = sum(dist(x[k], int(levels[k]), q[k], lm) for k in range(1, 64))
    return (rate(levels, ac_lengths(chroma)) << RATE_SHIFT) + d


def brute_force(x, q, chroma):
    """(minimum cost, one set of levels reaching it) over every candidate combination"""
    x = [int(v) for v in x]
    q = [int(v) for v in q]
    p = [plain(x[k], q[k]) for k in range(64)]
    nz = [k for k in range(1, 64) if p[k]]
    best = None
    for combo in itertools.product(*[candidates(p[k]) for k in nz]):
        lv = [0] * 64
        lv[0] = p[0]
        for k, m in zip(nz, combo):
            lv[k] = m if x[k] > 0 else -m
        c = cost(x, q, lv, chroma)
        if best is None or c < best[0]:
            best = (c, lv)
    return best


def dp(x, q, chroma):
    """The levels the trellis picks, by its dynamic programme and tie rule, vectorised over predecessors with numpy."""
    x = [int(v) for v in x]
    q = [int(v) for v in q]
    L = np.array(ac_lengths(chroma), dtype=np.int64)
    p = [plain(x[k], q[k]) for k in range(64)]
    out = [0] * 64
    out[0] = p[0]
    if not any(p[1:]):
        return out
    lm = lam(x)
    U = 1 << RATE_SHIFT
    pos, G, pred, sz = [0], [0], [0], [0]
    Z = 0
    for k in range(1, 64):
        d0 = dist(x[k], 0, q[k], lm)
        a = abs(p[k])
        if a:
            nb = a.bit_length()
            P = np.array(pos[::-1], dtype=np.int64)             # nearest predecessor first
            Gv = np.array(G[::-1], dtype=np.int64)
            r = k - P - 1
            best = None
            for s in range(nb, 0, -1):                           # largest magnitude first
                c = a if s == nb else (1 << s) - 1
                tot = Gv + Z + dist(x[k], c, q[k], lm) + s * U + (r // 16) * L[0xF0] * U + L[((r % 16) << 4) | s] * U
                i = int(np.argmin(tot))                          # first minimum = nearest predecessor among ties
                if best is None or tot[i] < best[0]:
                    best = (int(tot[i]), len(pos) - 1 - i, s)
            G.append(best[0] - Z - d0)
            pos.append(k)
            pred.append(best[1])
            sz.append(best[2])
        Z += d0
    ends = [G[b] + (L[0] * U if pos[b] < 63 else 0) for b in range(len(pos))]
    b = max(range(len(pos)), key=lambda i: (-ends[i], i))        # least cost, the latest among ties
    while b > 0:
        k, s = pos[b], sz[b]
        a = abs(p[k])
        c = a if s == a.bit_length() else (1 << s) - 1
        out[k] = c if x[k] > 0 else -c
        b = pred[b]
    return out
