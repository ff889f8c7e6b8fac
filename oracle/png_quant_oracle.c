/* png_quant_oracle.c -- scalar twin of the lossy PNG quantiser (caesium-clt_b200/csrc/png_quant.cu) over the same rules
 * (png_quant_core.h): histogram, median cut, k-means refinement, raster Floyd-Steinberg.  TEST INFRASTRUCTURE, NOT PRODUCT CODE. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include "../caesium-clt_b200/csrc/png_quant_core.h"

typedef struct {
    const uint32_t *cells; int ncells;
    const unsigned long long *count, *sums;     /* dense: count[cell], sums[cell][4] */
    uint8_t *label;                             /* box per occupied cell */
} Ctx;

static void cell_rep(const Ctx *c, int i, int v[4])
{
    const uint32_t cell = c->cells[i];
    const unsigned long long n = c->count[cell];
    for (int k = 0; k < 4; k++) v[k] = (int)((c->sums[4 * (size_t)cell + k] + n / 2) / n);
}

static void box_add(PqBox *b, const int v[4], uint32_t cell, unsigned long long n)
{
    b->n += n;
    for (int k = 0; k < 4; k++) {
        b->s1[k] += n * (unsigned long long)v[k]; b->s2[k] += n * (unsigned long long)(v[k] * v[k]);
        b->marg[k][pq_cell_coord(cell, k)] += n;
    }
}

static int split_cb(void *ctx, int b, int axis, int t, int k, PqBox *sb, PqBox *sk)
{
    Ctx *c = (Ctx *)ctx;
    memset(sb, 0, sizeof(*sb));
    if (sk) memset(sk, 0, sizeof(*sk));
    for (int i = 0; i < c->ncells; i++) {
        if (c->label[i] != b) continue;
        const uint32_t cell = c->cells[i];
        int v[4]; cell_rep(c, i, v);
        if (axis >= 0 && pq_cell_coord(cell, axis) > t) { c->label[i] = (uint8_t)k; box_add(sk, v, cell, c->count[cell]); }
        else box_add(sb, v, cell, c->count[cell]);
    }
    return 0;
}

static int cmp_u64(const void *a, const void *b)
{
    const unsigned long long x = *(const unsigned long long *)a, y = *(const unsigned long long *)b;
    return x < y ? -1 : x > y;
}

/* rgba: w * h pixels (R, G, B, A bytes).  palette: 256 RGBA words (R in the low byte); idx: w * h indices.  Returns the palette
 * size (an image with at most 256 distinct values comes back exactly), -1 on allocation failure. */
int orc_png_quantize(const uint8_t *rgba, int w, int h, int quality, uint32_t *palette, uint8_t *idx)
{
    const size_t npix = (size_t)w * h;
    unsigned long long *count = calloc(PQ_NCELLS, 8), *sums = calloc((size_t)PQ_NCELLS * 4, 8);
    uint32_t *cells = malloc((size_t)PQ_NCELLS * 4); uint8_t *label = calloc(PQ_NCELLS, 1);
    int *err = NULL, ret = -1, clear = 0;
    PqBox *boxes = malloc(PQ_MAX_COLOURS * sizeof(PqBox));
    if (!count || !sums || !cells || !label || !boxes) goto done;
    /* distinct values (at most 257 looked for) */
    {
        uint32_t seen[257]; int ns = 0;
        for (size_t i = 0; i < npix && ns <= 256; i++) {
            uint32_t v; memcpy(&v, rgba + 4 * i, 4);
            int f = 0; for (int k = 0; k < ns; k++) if (seen[k] == v) { f = 1; break; }
            if (!f) seen[ns++] = v;
        }
        if (ns <= 256) {        /* exact: the distinct values, in pq_exact_key order */
            unsigned long long keys[256];
            for (int k = 0; k < ns; k++) keys[k] = pq_exact_key(seen[k]);
            qsort(keys, (size_t)ns, 8, cmp_u64);
            for (int k = 0; k < ns; k++) palette[k] = (uint32_t)keys[k];
            for (size_t i = 0; i < npix; i++) {
                uint32_t v; memcpy(&v, rgba + 4 * i, 4);
                for (int k = 0; k < ns; k++) if (palette[k] == v) { idx[i] = (uint8_t)k; break; }
            }
            ret = ns; goto done;
        }
    }
    for (size_t i = 0; i < npix; i++) {
        uint32_t v; memcpy(&v, rgba + 4 * i, 4);
        int p[4]; pq_premul(v, p);
        if (p[3] == 0) { clear = 1; continue; }         /* fully transparent: the reserved entry */
        const uint32_t cell = pq_cell(p);
        count[cell]++;
        for (int k = 0; k < 4; k++) sums[4 * (size_t)cell + k] += (unsigned long long)p[k];
    }
    int ncells = 0;
    for (uint32_t c = 0; c < PQ_NCELLS; c++) if (count[c]) cells[ncells++] = c;
    Ctx ctx = {cells, ncells, count, sums, label};
    const int nb = ncells ? pq_median_cut(&ctx, split_cb, quality, PQ_MAX_COLOURS - clear, boxes) : 0;
    if (nb < 0) goto done;
    /* box means, then the refinement passes */
    unsigned long long acc[PQ_MAX_COLOURS * 5];
    uint32_t ent[PQ_MAX_COLOURS], coords[PQ_MAX_COLOURS];
    memset(acc, 0, sizeof(acc));
    for (int i = 0; i < ncells; i++) {
        unsigned long long *a = acc + 5 * label[i];
        a[0] += count[cells[i]];
        for (int k = 0; k < 4; k++) a[1 + k] += sums[4 * (size_t)cells[i] + k];
    }
    int n = pq_entries_from_sums(acc, nb, ent);
    for (int pass = 0; pass < PQ_REFINE_PASSES; pass++) {
        for (int k = 0; k < n; k++) coords[k] = pq_entry_coords(ent[k]);
        memset(acc, 0, sizeof(acc));
        for (int i = 0; i < ncells; i++) {
            int v[4]; cell_rep(&ctx, i, v);
            unsigned long long *a = acc + 5 * pq_nearest(v, coords, n);
            a[0] += count[cells[i]];
            for (int k = 0; k < 4; k++) a[1 + k] += sums[4 * (size_t)cells[i] + k];
        }
        n = pq_entries_from_sums(acc, n, ent);
    }
    pq_order(ent, n);
    /* palette: the reserved transparent entry, then the quantised entries (coords[] holds only those) */
    if (clear) palette[0] = 0;
    for (int k = 0; k < n; k++) { coords[k] = pq_entry_coords(ent[k]); palette[clear + k] = ent[k]; }
    /* raster Floyd-Steinberg: err holds the whole-unit errors of the row above (cur) and of this row */
    err = calloc((size_t)(w + 2) * 8, sizeof(int));
    if (!err) goto done;
    int *up = err, *cur = err + (size_t)(w + 2) * 4;          /* index (x + 1) * 4 + c */
    for (int y = 0; y < h; y++) {
        memset(cur, 0, (size_t)(w + 2) * 4 * sizeof(int));
        for (int x = 0; x < w; x++) {
            uint32_t v; memcpy(&v, rgba + 4 * ((size_t)y * w + x), 4);
            int p[4]; pq_premul(v, p);
            if (p[3] == 0) { idx[(size_t)y * w + x] = 0; continue; }
            int t[4];
            for (int c = 0; c < 4; c++) {
                const int e16 = 7 * cur[x * 4 + c] + 3 * up[(x + 2) * 4 + c] + 5 * up[(x + 1) * 4 + c] + up[x * 4 + c];
                t[c] = pq_clamp255(p[c] + pq_fs_round(e16));
            }
            const int k = pq_nearest(t, coords, n);
            idx[(size_t)y * w + x] = (uint8_t)(clear + k);
            for (int c = 0; c < 4; c++) cur[(x + 1) * 4 + c] = t[c] - (int)((coords[k] >> (8 * c)) & 255);
        }
        int *s = up; up = cur; cur = s;
    }
    ret = clear + n;
done:
    free(count); free(sums); free(cells); free(label); free(err); free(boxes);
    return ret;
}
