/* b200_caesium_png_lossy.h -- lossy PNG on the device (opt-in): palette quantisation with Floyd-Steinberg dithering for PNG outputs
 * with png_optimize == 0, what libcaesium hands to imagequant.  The quantiser is the project's own (median cut over a 5-bit
 * histogram, k-means refinement, raster-order error diffusion; DESIGN.md §4.9) and does not produce imagequant's bytes, so it is
 * off until the integrator turns it on: with the switch off every call answers exactly as before (B200_ERR_UNSUPPORTED for lossy
 * PNG).  Declared apart from b200_caesium.h while the leg is opt-in. */
#ifndef B200_CAESIUM_PNG_LOSSY_H
#define B200_CAESIUM_PNG_LOSSY_H
#include "b200_caesium.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Process-wide switch: 1 = b200_compress_in_memory / b200_convert_in_memory (JPEG and WebP sources) / b200_compress_batch with
 * png_optimize == 0, and b200_compress_to_size_in_memory on PNG sources (bisecting png_quality), run the device quantiser; 0 =
 * they answer B200_ERR_UNSUPPORTED.  While never set, the environment variable B200_PNG_LOSSY=gpu turns it on (read once).
 * Default off.  Returns B200_OK or B200_ERR_INVALID_ARGUMENT. */
int b200_set_png_lossy(int on);

/* The quantiser alone on the current device (independent of the switch): rgba = width * height pixels as R, G, B, A bytes;
 * quality 0..100.  palette_rgba (caller-allocated, 1024 bytes) receives *npalette entries as R, G, B, A (entries that are not
 * opaque first); indices (caller-allocated, width * height) the entry of every pixel.  An image with at most 256 distinct values
 * comes back exactly: its values, not opaque first, each group in increasing order of R | G << 8 | B << 16 | A << 24. */
b200_status b200_png_quantize(const uint8_t *rgba, int width, int height, int quality, uint8_t *palette_rgba, int *npalette, uint8_t *indices);

#ifdef __cplusplus
}
#endif
#endif /* B200_CAESIUM_PNG_LOSSY_H */
