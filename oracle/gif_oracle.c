/* gif_oracle.c -- scalar twin of the GIF re-encoder (caesium-clt_b200/csrc/gif_device.cu, gif_kernels.cu) over the same rules
 * (gif_core.h) and the quantiser's (png_quant_core.h): composited canvases in, the whole file out.  TEST INFRASTRUCTURE, NOT
 * PRODUCT CODE. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include "../caesium-clt_b200/csrc/gif_core.h"
#include "../caesium-clt_b200/csrc/png_quant_core.h"

int orc_png_quantize(const uint8_t *rgba, int w, int h, int quality, uint32_t *palette, uint8_t *idx);

/* ---- the quantiser without its exact path (PngQuant::quantize with allow_exact = false) ----------------------------------------
 * orc_png_quantize (png_quant_oracle.c) always answers an image of at most 256 values exactly; below quality 100 the GIF leg
 * quantises those too.  This is the same serial restatement of the median cut, refinement and dithering over the same rules. */
typedef struct {
    const uint32_t *cells; int ncells;
    const unsigned long long *count, *sums;
    uint8_t *label;
} QCtx;

static void q_cell_rep(const QCtx *c, int i, int v[4])
{
    const uint32_t cell = c->cells[i];
    const unsigned long long n = c->count[cell];
    for (int k = 0; k < 4; k++) v[k] = (int)((c->sums[4 * (size_t)cell + k] + n / 2) / n);
}

static void q_box_add(PqBox *b, const int v[4], uint32_t cell, unsigned long long n)
{
    b->n += n;
    for (int k = 0; k < 4; k++) {
        b->s1[k] += n * (unsigned long long)v[k]; b->s2[k] += n * (unsigned long long)(v[k] * v[k]);
        b->marg[k][pq_cell_coord(cell, k)] += n;
    }
}

static int q_split(void *ctx, int b, int axis, int t, int k, PqBox *sb, PqBox *sk)
{
    QCtx *c = (QCtx *)ctx;
    memset(sb, 0, sizeof(*sb));
    if (sk) memset(sk, 0, sizeof(*sk));
    for (int i = 0; i < c->ncells; i++) {
        if (c->label[i] != b) continue;
        const uint32_t cell = c->cells[i];
        int v[4]; q_cell_rep(c, i, v);
        if (axis >= 0 && pq_cell_coord(cell, axis) > t) { c->label[i] = (uint8_t)k; q_box_add(sk, v, cell, c->count[cell]); }
        else q_box_add(sb, v, cell, c->count[cell]);
    }
    return 0;
}

/* as orc_png_quantize, never taking the exact path: returns the palette size, -1 on allocation failure */
int orc_gif_quantize(const uint8_t *rgba, int w, int h, int quality, uint32_t *palette, uint8_t *idx)
{
    const size_t npix = (size_t)w * h;
    unsigned long long *count = calloc(PQ_NCELLS, 8), *sums = calloc((size_t)PQ_NCELLS * 4, 8);
    uint32_t *cells = malloc((size_t)PQ_NCELLS * 4); uint8_t *label = calloc(PQ_NCELLS, 1);
    int *err = NULL, ret = -1, clear = 0;
    PqBox *boxes = malloc(PQ_MAX_COLOURS * sizeof(PqBox));
    if (!count || !sums || !cells || !label || !boxes) goto done;
    for (size_t i = 0; i < npix; i++) {
        uint32_t v; memcpy(&v, rgba + 4 * i, 4);
        int p[4]; pq_premul(v, p);
        if (p[3] == 0) { clear = 1; continue; }
        const uint32_t cell = pq_cell(p);
        count[cell]++;
        for (int k = 0; k < 4; k++) sums[4 * (size_t)cell + k] += (unsigned long long)p[k];
    }
    int ncells = 0;
    for (uint32_t c = 0; c < PQ_NCELLS; c++) if (count[c]) cells[ncells++] = c;
    QCtx ctx = {cells, ncells, count, sums, label};
    const int nb = ncells ? pq_median_cut(&ctx, q_split, quality, PQ_MAX_COLOURS - clear, boxes) : 0;
    if (nb < 0) goto done;
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
            int v[4]; q_cell_rep(&ctx, i, v);
            unsigned long long *a = acc + 5 * pq_nearest(v, coords, n);
            a[0] += count[cells[i]];
            for (int k = 0; k < 4; k++) a[1 + k] += sums[4 * (size_t)cells[i] + k];
        }
        n = pq_entries_from_sums(acc, n, ent);
    }
    pq_order(ent, n);
    if (clear) palette[0] = 0;
    for (int k = 0; k < n; k++) { coords[k] = pq_entry_coords(ent[k]); palette[clear + k] = ent[k]; }
    err = calloc((size_t)(w + 2) * 8, sizeof(int));
    if (!err) goto done;
    int *up = err, *cur = err + (size_t)(w + 2) * 4;
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

typedef struct { uint8_t *p; size_t n, cap; int bad; } Out;

static void put(Out *o, const uint8_t *b, size_t n)
{
    if (o->bad || n > o->cap - o->n) { o->bad = 1; return; }
    memcpy(o->p + o->n, b, n); o->n += n;
}

/* LZW of n indices at minimum code size m, sub-blocked with its terminator; 0 or -1 (allocation, room) */
static int lzw(const uint8_t *idx, size_t n, int m, Out *o)
{
    const size_t nseg = n ? (n + GIF_SEG - 1) / GIF_SEG : 1;
    uint32_t *table = malloc(GIF_HASH * 4);
    uint16_t *codes = malloc(GIF_SEG_CODES * 2);
    uint8_t *bytes = calloc(nseg * GIF_SEG_CODES * 12 / 8 + 8, 1);
    int ret = -1;
    if (!table || !codes || !bytes) goto done;
    unsigned long long bit = 0;
    for (size_t s = 0; s < nseg; s++) {
        const size_t at = s * GIF_SEG, len = n - at < GIF_SEG ? n - at : GIF_SEG;
        unsigned b = 0;
        const int nc = gif_lzw_segment(idx + at, (int)len, m, s == 0, s == nseg - 1, table, codes, &b);
        for (int k = 0; k < nc; k++) {
            const int w = codes[k] >> 12;
            const uint32_t c = codes[k] & 4095u;
            for (int j = 0; j < w; j++, bit++) bytes[bit >> 3] |= (uint8_t)(((c >> j) & 1) << (bit & 7));
        }
    }
    const size_t nbytes = (size_t)((bit + 7) / 8), total = gif_blocks_size(nbytes);
    for (size_t i = 0; i < total; i++) { const uint8_t v = gif_blocks_byte(bytes, nbytes, i); put(o, &v, 1); }
    ret = o->bad ? -1 : 0;
done:
    free(table); free(codes); free(bytes);
    return ret;
}

/* the GIF LZW coder alone: returns the sub-blocked size written to out, -1 when it does not fit or allocation fails */
long long orc_gif_lzw(const uint8_t *idx, size_t n, int m, uint8_t *out, size_t cap)
{
    Out o = {out, 0, cap, 0};
    return lzw(idx, n, m, &o) ? -1 : (long long)o.n;
}

static GifRect diff_box(const uint32_t *a, const uint32_t *b, int w, int h, int clears_only)
{
    GifRect r = {0, 0, 0, 0};
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            const uint32_t pa = a[(size_t)y * w + x], pb = b[(size_t)y * w + x];
            if (pa == pb || (clears_only && !((pa >> 24) && !(pb >> 24)))) continue;
            const GifRect p = {x, y, x + 1, y + 1};
            r = gif_union(r, p);
        }
    return r;
}

/* canvases: n composited frames of w * h RGBA words (R in the low byte), delays in 1/100 s, loop -1 for none.  Returns the file
 * size written to out, -1 when it does not fit or allocation fails. */
long long orc_gif_encode(const uint32_t *canvases, const int *delays, int n, int w, int h, int loop, int quality, uint8_t *out, size_t cap)
{
    Out o = {out, 0, cap, 0};
    const size_t npix = (size_t)w * h;
    const GifRect whole = {0, 0, w, h}, none = {0, 0, 0, 0};
    uint8_t buf[8 + 10 + 768 + 1];
    put(&o, buf, (size_t)gif_put_header(buf, w, h, loop));
    uint32_t *crop = malloc(npix * 4 + 4), pal[256];
    uint8_t *idx = malloc(npix + 1);
    long long ret = -1;
    if (!crop || !idx) goto done;
    /* the kept canvases in order: a canvas equal to the last kept one only lengthens its delay */
    int *keep = malloc(sizeof(int) * (size_t)(n + 1)), *delay = malloc(sizeof(int) * (size_t)(n + 1)), nk = 0;
    if (!keep || !delay) { free(keep); free(delay); goto done; }
    for (int i = 0; i < n; i++) {
        if (nk && !memcmp(canvases + npix * keep[nk - 1], canvases + npix * i, npix * 4)) {
            const int d = delay[nk - 1] + delays[i];
            delay[nk - 1] = d > GIF_MAX_DELAY ? GIF_MAX_DELAY : d;
            continue;
        }
        keep[nk] = i; delay[nk] = delays[i]; nk++;
    }
    GifRect redraw = none;
    for (int j = 0; j < nk; j++) {
        const uint32_t *cur = canvases + npix * keep[j], *prev = j ? canvases + npix * keep[j - 1] : cur;
        const GifRect clears = j + 1 < nk ? diff_box(cur, canvases + npix * keep[j + 1], w, h, 1) : none;
        const GifRect r = j ? gif_union(gif_union(diff_box(prev, cur, w, h, 0), clears), redraw) : whole;
        const GifRect drawn = j ? redraw : whole;
        const int disposal = gif_rect_empty(clears) ? 1 : 2, rw = r.x1 - r.x0, rh = r.y1 - r.y0;
        for (int y = r.y0; y < r.y1; y++)
            for (int x = r.x0; x < r.x1; x++)
                crop[(size_t)(y - r.y0) * rw + (x - r.x0)] = gif_out_pixel(prev[(size_t)y * w + x], cur[(size_t)y * w + x], gif_in_rect(drawn, x, y));
        const int np = quality == 100 ? orc_png_quantize((const uint8_t *)crop, rw, rh, quality, pal, idx)
                                      : orc_gif_quantize((const uint8_t *)crop, rw, rh, quality, pal, idx);
        if (np <= 0) { free(keep); free(delay); goto done; }
        put(&o, buf, (size_t)gif_put_frame_head(buf, delay[j], disposal, r, pal, np));
        if (lzw(idx, (size_t)rw * rh, gif_min_code_size(np), &o)) { free(keep); free(delay); goto done; }
        redraw = disposal == 2 ? r : none;
    }
    free(keep); free(delay);
    {
        const uint8_t t = 0x3B;
        put(&o, &t, 1);
    }
    ret = o.bad ? -1 : (long long)o.n;
done:
    free(crop); free(idx);
    return ret;
}
