/*
 * oracle/jpeg_oracle.h -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * CPU restatement of the JPEG half of the hot path that caesiumclt reaches through
 * `caesium::compress_in_memory` (caesium-clt's src/compressor.rs:305) and, for
 * `--lossless`, the coefficient-domain transcode selected by
 * `parameters.jpeg.optimize` (caesium-clt's src/compressor.rs:427).
 *
 * The arithmetic itself is NOT in the caesium-clt sources: it lives in libcaesium 0.20.3
 * (Cargo.lock:892) -> mozjpeg-sys 2.2.1 (Cargo.lock:1035) -> mozjpeg 4.x, whose
 * sources are not vendored.  This file restates the *published* IJG/libjpeg-turbo
 * algorithms those crates execute (names of the upstream routines are cited at each
 * function) and is pinned empirically against libjpeg-turbo 3.1 (via Pillow) and
 * the DQT/scan-script known-answer vectors of the reference's own fixtures
 * (samples/j0.JPG, samples/level_1_0/j1.jpg) -- see tests/test_oracle_jpeg.py.
 *
 * PARITY STATUS: "pinned to sibling implementation + fixture KATs"; the true
 * reference binary cannot be built here (no cargo/rustc), so trellis quantisation,
 * overshoot deringing and optimize_scans of mozjpeg are NOT restated (DESIGN.md §3).
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl
 * reference legs may load this library.
 */
#ifndef JPEG_ORACLE_H
#define JPEG_ORACLE_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ORC_MAX_COMP 4

typedef struct {
    int width, height, ncomp;
    int progressive;               /* SOF2 */
    int hs[ORC_MAX_COMP], vs[ORC_MAX_COMP], tq[ORC_MAX_COMP], cid[ORC_MAX_COMP];
    int hmax, vmax;
    int mcux, mcuy;                /* MCUs across / down (interleaved geometry) */
    int bw[ORC_MAX_COMP], bh[ORC_MAX_COMP];   /* allocated blocks (padded to MCU) */
    int rbw[ORC_MAX_COMP], rbh[ORC_MAX_COMP]; /* real blocks: ceil(cw/8), ceil(ch/8) */
    int cw[ORC_MAX_COMP], ch[ORC_MAX_COMP];   /* component sample dims */
    uint16_t qt[4][64];            /* natural (row-major) order */
    int qt_present[4];
    int16_t *coef[ORC_MAX_COMP];   /* [bh][bw][64], natural order, quantised */
    int restart_interval;
    int nscans;
    int scan_script[64][8];        /* ncomp_in_scan, Ss, Se, Ah, Al, comp0, comp1|-1, comp2|-1 */
    int jfif, adobe, adobe_transform;
    /* carried markers (APPn / COM), verbatim including FF xx LL LL */
    uint8_t *markers; size_t markers_len;
    uint8_t *icc_markers; size_t icc_len;      /* APP2 "ICC_PROFILE" segments only */
} orc_jpeg;

typedef struct {
    int quality;             /* 0..100 */
    int subsampling;         /* 444,422,420,411, 0=auto(420 for 3 comps) */
    int progressive;         /* 1 = SOF2 multi-scan, 0 = SOF0 single interleaved scan */
    int keep_metadata;       /* copy APPn/COM */
    int preserve_icc;        /* copy ICC APP2 even when !keep_metadata */
} orc_jpeg_params;

/* ---- building blocks (each independently callable from the tests) ---- */
void orc_quant_table(int quality, int which /*0 luma,1 chroma*/, uint16_t out[64]);        /* mozjpeg jcparam.c: table idx 3 + jpeg_set_quality(force_baseline=FALSE) */
void orc_idct_islow(const int16_t coef[64], const uint16_t q[64], uint8_t out[64]);         /* jidctint.c jpeg_idct_islow */
void orc_fdct_islow(const uint8_t px[64], int32_t out[64]);                                 /* jfdctint.c jpeg_fdct_islow (+convsamp) */
void orc_quantize(const int32_t dct[64], const uint16_t q[64], int16_t out[64]);            /* jcdctmgr.c quantize (non-trellis) */
void orc_upsample_h2v2_fancy(const uint8_t *in, int cw, int ch, int stride, uint8_t *out, int ow, int oh, int ostride); /* jdsample.c */
void orc_upsample_h2v1_fancy(const uint8_t *in, int cw, int ch, int stride, uint8_t *out, int ow, int oh, int ostride);
void orc_upsample_h1v2_fancy(const uint8_t *in, int cw, int ch, int stride, uint8_t *out, int ow, int oh, int ostride);
void orc_upsample_box(const uint8_t *in, int cw, int ch, int stride, int hx, int vx, uint8_t *out, int ow, int oh, int ostride);
/* downsample W x H full-res plane into a (pw x ph) padded plane, jcsample.c + jcprepct.c edge rules */
void orc_downsample(const uint8_t *in, int w, int h, int stride, int hx, int vx, uint8_t *out, int pw, int ph);

/* ---- whole stages ---- */
int  orc_jpeg_read(const uint8_t *data, size_t len, orc_jpeg *j, char err[256]);  /* markers + Huffman (baseline/progressive) -> coefficients */
void orc_jpeg_free(orc_jpeg *j);
/* dequant + IDCT every block of component c into a (bw*8 x bh*8) plane */
void orc_jpeg_idct_component(const orc_jpeg *j, int c, uint8_t *plane);
/* decoder output in the file's native colour space, planar, each plane width x height
 * (what jpeg_read_scanlines yields with out_color_space = jpeg_color_space) */
int  orc_jpeg_decode_native(const orc_jpeg *j, uint8_t *planes[ORC_MAX_COMP], char err[256]);
/* forward path: planar full-res native-space image -> quantised coefficients of a new orc_jpeg */
int  orc_jpeg_forward(const uint8_t *const planes[ORC_MAX_COMP], int width, int height, int ncomp,
                      const orc_jpeg_params *p, orc_jpeg *out, char err[256]);
/* entropy-code an orc_jpeg (coefficients + tables) into a file */
int  orc_jpeg_write(const orc_jpeg *j, const orc_jpeg_params *p, const orc_jpeg *meta_src,
                    uint8_t **out, size_t *out_len, char err[256]);

/* libcaesium jpeg::lossy (compress_in_memory with jpeg.optimize == false) */
int  orc_jpeg_lossy(const uint8_t *data, size_t len, const orc_jpeg_params *p,
                    uint8_t **out, size_t *out_len, char err[256]);
/* libcaesium jpeg::lossless (jpegtran-style; jpeg.optimize == true) */
int  orc_jpeg_lossless(const uint8_t *data, size_t len, const orc_jpeg_params *p,
                       uint8_t **out, size_t *out_len, char err[256]);
void orc_free(void *p);

#ifdef __cplusplus
}
#endif
#endif
