/* b200_caesium_webp_bpred.h -- 4x4 intra prediction (B_PRED) for lossy WebP (opt-in).  With the switch on, every lossy WebP output --
 * WebP re-compression, JPEG / PNG / GIF -> WebP, the VP8 chunk of files with alpha, the lossy frames of animated WebP and every try of a
 * `--max-size` search on WebP -- lets each macroblock take the sixteen 4x4 sub-block predictors instead of one 16x16 predictor when
 * that scores lower in 256 * squared error + lambda * estimated bits.  A frame whose first partition would outgrow VP8's 19-bit size
 * field is coded 16x16-only, exactly as with the switch off.  Declared apart from b200_caesium.h while the leg is opt-in. */
#ifndef B200_CAESIUM_WEBP_BPRED_H
#define B200_CAESIUM_WEBP_BPRED_H
#include "b200_caesium.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Process-wide switch: 1 = lossy WebP outputs may use B_PRED; 0 = they never do, as before.  While never set, the environment variable
 * B200_WEBP_BPRED=gpu turns it on (read once).  Default off.  Returns B200_OK or B200_ERR_INVALID_ARGUMENT. */
int b200_set_webp_bpred(int on);

/* Stage view of the B_PRED encoder (used whatever the switch says): planar RGB [3][h][w] -> .webp file, and optionally the levels
 * ([mbh*mbw][25][16] int16, zigzag; a B_PRED macroblock has zero Y2 levels and keeps each luma block's DC at index 0), the modes
 * ([mbh*mbw][4] = ymode, uvmode, skip, 0; ymode 4 = B_PRED) and the sub-block modes ([mbh*mbw][16], raster order; 0 DC, 1 TM, 2 VE,
 * 3 HE, 4 RD, 5 VR, 6 LD, 7 VL, 8 HD, 9 HU; a 16x16 macroblock repeats its ymode).  Any of the three may be NULL. */
b200_status b200_webp_encode_rgb_bpred(const uint8_t *rgb, int w, int h, int quality, uint8_t **out, size_t *out_len,
                                       int16_t *levels, uint8_t *modes, uint8_t *bmodes);
/* host only: boolean-code levels + modes + sub-block modes (layout above) into a .webp file.  B200_ERR_INVALID_ARGUMENT for a sub-block
 * mode past 9 or a first partition that does not fit in 19 bits. */
b200_status b200_webp_write_levels_bpred(int w, int h, int quality, const int16_t *levels, const uint8_t *modes, const uint8_t *bmodes,
                                         uint8_t **out, size_t *out_len);

#ifdef __cplusplus
}
#endif
#endif /* B200_CAESIUM_WEBP_BPRED_H */
