/* png_quant_core.h -- the rules of the lossy PNG palette quantiser, written once for every party that has to agree on them: the
 * device kernels and their host driver (png_quant.cu) and the scalar oracle (oracle/png_quant_oracle.c, plain C -- hence no
 * namespace and no C++ in this file).  Everything that decides a palette entry or an index is integer arithmetic, so the parties
 * agree bit for bit and no atomic order can change a result.
 *
 *   colour space  a pixel is compared as alpha-premultiplied RGB plus alpha (pq_premul), so every fully transparent pixel is the
 *                 one colour (0, 0, 0, 0); distances are squared integer differences over the four channels; ties go to the
 *                 lower palette index
 *   histogram     2^20 cells of 5 bits per premultiplied channel; a cell holds its pixel count and the exact 64-bit sums of its
 *                 pixels, and stands for its rounded mean (the cell's representative) in median cut and refinement; every
 *                 rounded mean here rounds halves up
 *   median cut    boxes are ranges of cell coordinates; the splittable box with the largest weighted SSE of its representatives
 *                 (ties to the lower box) is split on its highest-variance axis (among axes with two or more occupied
 *                 coordinates; ties to the lower axis, R G B A) at the weighted median (the first coordinate t at which twice
 *                 the pixels up to t reach the box's, at most the last occupied coordinate minus one); an axis's SSE is
 *                 s2 - floor(s1^2 / n) over the box's pixel count n and the weighted sums s1, s2 of its representatives, and the
 *                 axis comparison uses that integer; stop at PQ_MAX_COLOURS boxes (one fewer with the reserved entry), when the
 *                 total SSE is at most pq_target_mse[quality] * (pixels that are not fully transparent), or when no box can be
 *                 split; an entry is the rounded mean of the box's pixels, un-premultiplied with rounding
 *   refinement    PQ_REFINE_PASSES weighted k-means passes over the occupied cells; entries left without pixels are dropped
 *                 (the others keep their order)
 *   order         the reserved transparent entry, then entries that are not opaque, then the opaque ones, each group in
 *                 refinement order
 *   transparency  fully transparent pixels (alpha 0) stay out of the histogram; when the source has any, the palette reserves
 *                 entry 0 = (0, 0, 0, 0) for them, they take it without a search and neither take nor pass dithering error, and no
 *                 other pixel may take it -- so a transparent area stays transparent and an opaque source keeps opaque entries
 *   dithering     Floyd-Steinberg at full strength (7, 3, 5, 1 sixteenths) in raster order on the premultiplied values; the
 *                 incoming error is rounded to whole units, halves away from zero, and the target clamped to 0..255 (which
 *                 bounds every error to +-255)
 *   exact path    a source with at most 256 distinct RGBA values is not quantised: its palette is those values in pq_exact_key
 *                 order (the PNG writer then takes the lossless leg's exact palette reduction) */
#ifndef PNG_QUANT_CORE_H
#define PNG_QUANT_CORE_H
#include <stdint.h>

#if defined(__CUDACC__)
#define PQ_HD static __host__ __device__ __forceinline__
#else
#define PQ_HD static inline
#endif

#ifdef __cplusplus
namespace b200 {
#endif

enum {
    PQ_CELL_BITS = 5, PQ_NCELLS = 1 << 20,      /* 5 bits per channel */
    PQ_BINS = 32,                               /* coordinates per axis */
    PQ_MAX_COLOURS = 256,
    PQ_REFINE_PASSES = 3,
    PQ_GRID = 1 << 16                           /* nearest-entry candidate grid: 4 bits per channel */
};

/* target mean squared error (summed over the four channels, 8-bit units) per quality 0..100: 2000 * ((100 - q) / 100)^3, rounded
 * (0 from q = 94 up: those qualities give the same palette) */
static const uint16_t pq_target_mse[101] = {
    2000, 1941, 1882, 1825, 1769, 1715, 1661, 1609, 1557, 1507, 1458, 1410, 1363, 1317, 1272, 1228, 1185, 1144, 1103, 1063,
    1024, 986, 949, 913, 878, 844, 810, 778, 746, 716, 686, 657, 629, 602, 575, 549, 524, 500, 477, 454,
    432, 411, 390, 370, 351, 333, 315, 298, 281, 265, 250, 235, 221, 208, 195, 182, 170, 159, 148, 138,
    128, 119, 110, 101, 93, 86, 79, 72, 66, 60, 54, 49, 44, 39, 35, 31, 28, 24, 21, 19,
    16, 14, 12, 10, 8, 7, 5, 4, 3, 3, 2, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0};

/* premultiplied value of an RGBA8 pixel */
PQ_HD void pq_premul(uint32_t rgba, int p[4])
{
    const int r = (int)(rgba & 255), g = (int)((rgba >> 8) & 255), b = (int)((rgba >> 16) & 255), a = (int)(rgba >> 24);
    p[0] = (r * a + 127) / 255; p[1] = (g * a + 127) / 255; p[2] = (b * a + 127) / 255; p[3] = a;
}
PQ_HD uint32_t pq_pack(const int p[4]) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24); }
PQ_HD uint32_t pq_cell(const int p[4]) { return ((uint32_t)(p[0] >> 3) << 15) | ((uint32_t)(p[1] >> 3) << 10) | ((uint32_t)(p[2] >> 3) << 5) | (uint32_t)(p[3] >> 3); }
PQ_HD int pq_cell_coord(uint32_t cell, int axis) { return (int)((cell >> (15 - 5 * axis)) & 31); }
PQ_HD uint32_t pq_grid(const int t[4]) { return ((uint32_t)(t[0] >> 4) << 12) | ((uint32_t)(t[1] >> 4) << 8) | ((uint32_t)(t[2] >> 4) << 4) | (uint32_t)(t[3] >> 4); }

PQ_HD int pq_dist(const int a[4], uint32_t b)
{
    int d = 0;
    for (int c = 0; c < 4; c++) { const int e = a[c] - (int)((b >> (8 * c)) & 255); d += e * e; }
    return d;
}

/* a palette entry from the exact sums of its pixels' premultiplied values: the rounded mean, un-premultiplied to RGBA8 */
PQ_HD uint32_t pq_entry_rgba(const unsigned long long s[4], unsigned long long n)
{
    int m[4];
    for (int c = 0; c < 4; c++) m[c] = (int)((s[c] + n / 2) / n);
    const int a = m[3];
    if (a == 0) return 0;
    int o[4];
    for (int c = 0; c < 3; c++) { const int v = (m[c] * 255 + a / 2) / a; o[c] = v > 255 ? 255 : v; }
    o[3] = a;
    return pq_pack(o);
}
/* the coordinates an entry is compared at: its own RGBA premultiplied again */
PQ_HD uint32_t pq_entry_coords(uint32_t rgba) { int p[4]; pq_premul(rgba, p); return pq_pack(p); }

/* Floyd-Steinberg: the error arriving at a pixel (7 left + 3 up-right + 5 up + 1 up-left, each a whole-unit error) in sixteenths,
 * rounded half away from zero */
PQ_HD int pq_fs_round(int e16) { return e16 >= 0 ? (e16 + 8) >> 4 : -((-e16 + 8) >> 4); }
PQ_HD int pq_clamp255(int v) { return v < 0 ? 0 : v > 255 ? 255 : v; }

/* exact path: the palette is the distinct values in increasing order of this key (entries that are not opaque first) */
PQ_HD unsigned long long pq_exact_key(uint32_t rgba) { return ((unsigned long long)((rgba >> 24) == 255) << 32) | rgba; }

/* nearest entry, exhaustively (ties to the lower index) */
PQ_HD int pq_nearest(const int t[4], const uint32_t *coords, int n)
{
    int best = 0, bd = 0x7FFFFFFF;
    for (int k = 0; k < n; k++) { const int d = pq_dist(t, coords[k]); if (d < bd) { bd = d; best = k; } }
    return best;
}

/* ---- median cut (host side: O(boxes) work per split) ---------------------------------------------------------------------- */
/* statistics of one box over its cells' representatives v (weights n): count, sum n v and sum n v^2 per axis, and the marginal
 * pixel counts per coordinate of each axis */
typedef struct {
    unsigned long long n, s1[4], s2[4], marg[4][PQ_BINS];
} PqBox;
#define PQ_BOX_WORDS (1 + 4 + 4 + 4 * PQ_BINS)

static inline unsigned long long pq_axis_sse(const PqBox *b, int c)
{
    if (!b->n) return 0;
    const unsigned __int128 sq = (unsigned __int128)b->s1[c] * b->s1[c];
    return b->s2[c] - (unsigned long long)(sq / b->n);
}
static inline unsigned long long pq_box_sse(const PqBox *b) { unsigned long long s = 0; for (int c = 0; c < 4; c++) s += pq_axis_sse(b, c); return s; }

/* the split of a box: axis (-1: the box cannot be split) and the last coordinate t that stays in the box */
static inline int pq_box_split(const PqBox *b, int *t_out)
{
    int axis = -1; unsigned long long best = 0;
    for (int c = 0; c < 4; c++) {
        int lo = -1, hi = -1;
        for (int k = 0; k < PQ_BINS; k++) if (b->marg[c][k]) { if (lo < 0) lo = k; hi = k; }
        if (lo == hi) continue;
        const unsigned long long v = pq_axis_sse(b, c);
        if (axis < 0 || v > best) { axis = c; best = v; }
    }
    if (axis < 0) return -1;
    int lo = -1, hi = -1;
    for (int k = 0; k < PQ_BINS; k++) if (b->marg[axis][k]) { if (lo < 0) lo = k; hi = k; }
    unsigned long long cum = 0; int t = lo;
    for (int k = lo; k <= hi; k++) { cum += b->marg[axis][k]; t = k; if (2 * cum >= b->n) break; }
    if (t >= hi) t = hi - 1;
    *t_out = t;
    return axis;
}

/* Splits box b along axis at t: cells of b with coordinate > t move to the new box k; fills the statistics of both.  axis < 0:
 * only fill *sb with the statistics of box b (the first call, box 0 = every cell). */
typedef int (*pq_split_fn)(void *ctx, int b, int axis, int t, int k, PqBox *sb, PqBox *sk);

/* the median cut proper over at most max_boxes boxes; returns the number of boxes (cells carry their box in the caller's labels)
 * or -1 when a split failed */
static inline int pq_median_cut(void *ctx, pq_split_fn split, int quality, int max_boxes, PqBox *boxes /*PQ_MAX_COLOURS*/)
{
    if (split(ctx, 0, -1, 0, 0, &boxes[0], 0)) return -1;
    const int q = quality < 0 ? 0 : quality > 100 ? 100 : quality;
    const unsigned long long limit = (unsigned long long)pq_target_mse[q] * boxes[0].n;
    int nb = 1;
    unsigned long long sse[PQ_MAX_COLOURS];
    sse[0] = pq_box_sse(&boxes[0]);
    while (nb < max_boxes) {
        unsigned long long total = 0;
        for (int i = 0; i < nb; i++) total += sse[i];
        if (total <= limit) break;
        int pick = -1, axis = -1, t = 0;
        for (int i = 0; i < nb; i++) {
            int ti = 0;
            if (pick >= 0 && sse[i] <= sse[pick]) continue;
            const int a = pq_box_split(&boxes[i], &ti);
            if (a >= 0) { pick = i; axis = a; t = ti; }
        }
        if (pick < 0) break;
        if (split(ctx, pick, axis, t, nb, &boxes[pick], &boxes[nb])) return -1;
        sse[pick] = pq_box_sse(&boxes[pick]); sse[nb] = pq_box_sse(&boxes[nb]);
        nb++;
    }
    return nb;
}

/* entries from per-entry sums (n, s[4]); entries without pixels are dropped, the rest keep their order.  Returns the count. */
static inline int pq_entries_from_sums(const unsigned long long *sums /*[k][5]*/, int k, uint32_t *rgba)
{
    int n = 0;
    for (int i = 0; i < k; i++) {
        const unsigned long long *s = sums + 5 * i;
        if (s[0]) rgba[n++] = pq_entry_rgba(s + 1, s[0]);
    }
    return n;
}

/* final order: entries that are not opaque first, each group in its given order; returns the number that are not opaque */
static inline int pq_order(uint32_t *rgba, int n)
{
    uint32_t t[PQ_MAX_COLOURS]; int m = 0;
    for (int i = 0; i < n; i++) if ((rgba[i] >> 24) != 255) t[m++] = rgba[i];
    const int ntrans = m;
    for (int i = 0; i < n; i++) if ((rgba[i] >> 24) == 255) t[m++] = rgba[i];
    for (int i = 0; i < n; i++) rgba[i] = t[i];
    return ntrans;
}

#ifdef __cplusplus
}
#endif
#endif /* PNG_QUANT_CORE_H */
