/* jpeg_trellis_oracle.c -- scalar twin of the JPEG encoder's opt-in trellis quantiser (k_jpeg_trellis in
 * caesium-clt_b200/csrc/jpeg_kernels.cu) over the same rule (jpeg_trellis_core.h).  TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * PARITY NOTE: this is the project's own rate-distortion quantiser, modelled on mozjpeg's per-block AC trellis (JCP_MAX_COMPRESSION)
 * but not pinned to mozjpeg's output: Annex K rates, 1/Q^2 weights, tuned lambda, no DC trellis, no EOB-run optimisation, no
 * Huffman-rate feedback.  What it is pinned to is the device: both include jpeg_trellis_core.h, and tests/test_jpeg_trellis_host.py
 * checks this twin against an exhaustive search and an independent dynamic programme written from the header comment. */
#include <stdlib.h>
#include <string.h>
#include "jpeg_oracle.h"
#include "../caesium-clt_b200/csrc/jpeg_trellis_core.h"

static const uint8_t ZZ[64] = { /* zigzag index k -> natural (row-major) position */
     0,  1,  8, 16,  9,  2,  3, 10, 17, 24, 32, 25, 18, 11,  4,  5,
    12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13,  6,  7, 14, 21, 28,
    35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
    58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63 };

/* one block, natural order in and out; chroma = 0 costs symbols with the Annex K.5 AC lengths (component 0), 1 with K.6 */
void orc_quantize_trellis(const int32_t dct[64], const uint16_t q[64], int chroma, int16_t out[64])
{
    uint16_t qz[64]; int16_t xz[64];
    for (int k = 0; k < 64; k++) { qz[k] = q[ZZ[k]]; xz[k] = (int16_t)dct[ZZ[k]]; }
    JtTable t; jt_make_table(qz, chroma, &t);
    long long G[64]; uint8_t pos[64], pred[64], size[64];
    jt_trellis_block(xz, &t, xz, G, pos, pred, size, 1);
    for (int k = 0; k < 64; k++) out[ZZ[k]] = xz[k];
}

/* orc_jpeg_forward with the trellis in place of plain quantisation: the plain forward path gives the geometry, the tables and the
 * dummy blocks (AC 0, DC of a neighbouring real block -- the trellis keeps every DC), then every real block is transformed again
 * from the same downsampled plane and quantised by the trellis. */
int orc_jpeg_forward_trellis(const uint8_t *const planes[ORC_MAX_COMP], int width, int height, int ncomp,
                             const orc_jpeg_params *p, orc_jpeg *o, char err[256])
{
    if (orc_jpeg_forward(planes, width, height, ncomp, p, o, err)) return -1;
    for (int c = 0; c < o->ncomp; c++) {
        const int pw = o->rbw[c] * 8, ph = o->rbh[c] * 8;
        uint8_t *ds = (uint8_t *)malloc((size_t)pw * ph);
        if (!ds) { orc_jpeg_free(o); if (err) strcpy(err, "out of memory"); return -1; }
        orc_downsample(planes[c], width, height, width, o->hmax / o->hs[c], o->vmax / o->vs[c], ds, pw, ph);
        uint8_t px[64]; int32_t dct[64];
        for (int by = 0; by < o->rbh[c]; by++) for (int bx = 0; bx < o->rbw[c]; bx++) {
            for (int y = 0; y < 8; y++) memcpy(px + 8 * y, ds + (size_t)(by * 8 + y) * pw + bx * 8, 8);
            orc_fdct_islow(px, dct);
            orc_quantize_trellis(dct, o->qt[o->tq[c]], c != 0, o->coef[c] + ((size_t)by * o->bw[c] + bx) * 64);
        }
        free(ds);
    }
    return 0;
}
