"""Plain-Python statement of the PNG `--zopfli` rules, written from the comment at the top of png_zopfli_core.h: the cost table, the
Pareto front and its PZ_K pruning, an exhaustive match search at every distance, and the shortest path with the same tie rules.
It is slow (every distance at every position) and meant for streams of a few hundred bytes."""

SEG, WINDOW, MAXLEN = 32768, 32768, 258
LEN_BASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
LEN_EXTRA = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
DIST_BASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577]
DIST_EXTRA = [0, 0, 0, 0] + [k // 2 - 1 for k in range(4, 30)]


def len_symbol(n):
    return max(k for k in range(29) if LEN_BASE[k] <= n)


def dist_symbol(d):
    return max(k for k in range(30) if DIST_BASE[k] <= d)


def log2_q10(x):
    """1024 * log2(x), piecewise linear between powers of two"""
    x = max(int(x), 1)
    e = x.bit_length() - 1
    frac = (x >> (e - 10)) & 1023 if e >= 10 else (x << (10 - e)) & 1023
    return e * 1024 + frac


def costs(h):
    """316-entry cost table of a token histogram (1024ths of a bit, extra bits included)"""
    tl, td = sum(int(v) for v in h[:286]), sum(int(v) for v in h[286:316])
    out = []
    for x in range(316):
        t = log2_q10(tl if x < 286 else td)
        c = t - log2_q10(h[x]) if h[x] else t + 1024
        c = min(max(c, 1024), 15 * 1024)
        extra = DIST_EXTRA[x - 286] if x >= 286 else LEN_EXTRA[x - 257] if 257 <= x < 286 else 0
        out.append(c + 1024 * extra)
    return out


def front(cands, k=None):
    """the Pareto front of (length, distance) pairs with length >= 3 (no kept pair has another with a length at least as long and
    a distance at most as short), by increasing distance; with k, a front of more than k pairs keeps its k - 1 smallest distances
    and its longest pair"""
    pairs = sorted({(l, d) for l, d in cands if l >= 3}, key=lambda p: (p[1], -p[0]))
    f = [p for p in pairs if not any(q != p and q[0] >= p[0] and q[1] <= p[1] for q in pairs)]
    if k is not None and len(f) > k:
        f = f[:k - 1] + [f[-1]]
    return f


def maxlen(i, n):
    return min(MAXLEN, min(n, (i // SEG + 1) * SEG) - i)


def exhaustive_set(s, i):
    """the full front of position i over every distance 1 .. min(i, WINDOW)"""
    n, m = len(s), maxlen(i, len(s))
    if m < 3:
        return []
    c = []
    for d in range(1, min(i, WINDOW) + 1):
        l = 0
        while l < m and s[i + l] == s[i + l - d]:
            l += 1
        c.append((l, d))
    return front(c)


def shortest_path(s, sets, cost, s0=0, L=None):
    """tokens of the cheapest parse of s[s0, s0 + L) given each position's (length, distance) list (by increasing distance):
    sources in increasing order, a target changes only on a strictly smaller cost, a match edge of length l takes the cheapest entry
    at least l long (ties to the smaller distance)"""
    L = len(s) - s0 if L is None else L
    INF = 1 << 62
    c = [0] + [INF] * L
    back = [None] * (L + 1)
    for i in range(L):
        lit = c[i] + cost[s[s0 + i]]
        if lit < c[i + 1]:
            c[i + 1], back[i + 1] = lit, ("lit", s[s0 + i], 1)
        e = sets[s0 + i]
        if not e:
            continue
        for l in range(3, e[-1][0] + 1):
            best, bd = None, None
            for el, d in e:
                if el >= l:
                    dc = cost[286 + dist_symbol(d)]
                    if best is None or dc < best:
                        best, bd = dc, d
            v = c[i] + best + cost[257 + len_symbol(l)]
            if v < c[i + l]:
                c[i + l], back[i + l] = v, ("match", (l, bd), l)
    toks, t = [], L
    while t > 0:
        kind, val, step = back[t]
        toks.append(val if kind == "lit" else 0x80000000 | ((val[0] - 3) << 16) | (val[1] - 1))
        t -= step
    return toks[::-1], c[L]


def parse_cost(s, toks, cost):
    """the cost of a token list under one table"""
    total = 0
    for t in toks:
        if t & 0x80000000:
            l, d = ((t >> 16) & 0x7FFF) + 3, (t & 0xFFFF) + 1
            total += cost[257 + len_symbol(l)] + cost[286 + dist_symbol(d)]
        else:
            total += cost[t]
    return total
