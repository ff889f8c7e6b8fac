/* b200_caesium_gif.h -- GIF on the device (opt-in): still and animated GIFs re-encoded frame by frame with the palette quantiser
 * of the lossy PNG leg and a segmented LZW coder (DESIGN.md §4.11).  libcaesium re-encodes GIFs through gifski, whose bytes this
 * leg does not reproduce, so it is off until the integrator turns it on: with the switch off every call answers exactly as before
 * (B200_ERR_UNSUPPORTED for GIF).  Declared apart from b200_caesium.h while the leg is opt-in. */
#ifndef B200_CAESIUM_GIF_H
#define B200_CAESIUM_GIF_H
#include "b200_caesium.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Process-wide switch: 1 = b200_compress_in_memory and b200_compress_batch on GIF sources run the device leg at gif_quality
 * (100: every frame whose changed area has at most 256 values keeps them exactly); 0 = they answer B200_ERR_UNSUPPORTED.  While
 * never set, the environment variable B200_GIF=gpu turns it on (read once).  Default off.  Resizing (width / height), conversions
 * to or from GIF and compress_to_size on a GIF answer B200_ERR_UNSUPPORTED either way, as does a file with a frame that extends
 * past its logical screen.  Returns B200_OK or B200_ERR_INVALID_ARGUMENT. */
int b200_set_gif(int on);

/* The host decoder alone (independent of the switch, no device needed): the displayed canvas of every frame after compositing
 * (*nframes frames of width * height pixels as R, G, B, A bytes, alpha 0 or 255, a clear pixel all zero) in *rgba, each frame's
 * delay in 1/100 s in *delays, the NETSCAPE2.0 loop count in *loop (-1: none).  *rgba and *delays are released with b200_free.
 * Truncated or inconsistent data answers B200_ERR_CORRUPT_INPUT. */
b200_status b200_gif_decode(const uint8_t *in, size_t in_len, int *width, int *height, int *nframes, int *loop, uint8_t **rgba, int **delays);

/* The device LZW coder alone on the current device (independent of the switch): n palette indices, each below 2^min_code_size
 * (2..8), in raster order -> GIF image data as it follows the minimum code size byte (255-byte sub-blocks, each after its length,
 * and the 0 terminator) in *out, released with b200_free. */
b200_status b200_gif_lzw(const uint8_t *indices, size_t n, int min_code_size, uint8_t **out, size_t *out_len);

#ifdef __cplusplus
}
#endif
#endif /* B200_CAESIUM_GIF_H */
