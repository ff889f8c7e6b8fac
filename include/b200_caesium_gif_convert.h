/* b200_caesium_gif_convert.h -- conversions to and from GIF on the device (opt-in): what libcaesium's convert does for
 * `caesiumclt --format gif` on JPEG, PNG and WebP sources, and for `--format jpeg|png|webp` on GIF sources (DESIGN.md §4.14).
 * libcaesium writes GIFs through gifski, whose bytes this project does not reproduce: a converted GIF is the one-frame file the GIF
 * leg (b200_caesium_gif.h) writes for the source's pixels, so the conversions are off until the integrator turns them on.  Declared
 * apart from b200_caesium.h while they are opt-in. */
#ifndef B200_CAESIUM_GIF_CONVERT_H
#define B200_CAESIUM_GIF_CONVERT_H
#include "b200_caesium.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Process-wide switch, independent of b200_set_gif.  1 = b200_convert_in_memory runs these on the device:
 *   - fmt = B200_FMT_GIF on JPEG, PNG and WebP sources: every pixel with alpha 0 becomes clear, every other one opaque, and the
 *     image is written as one whole-canvas frame (delay 0, no loop count) quantised at gif_quality.  width / height answer
 *     B200_ERR_UNSUPPORTED.
 *   - GIF sources to B200_FMT_JPEG, B200_FMT_PNG and lossy B200_FMT_WEBP: frame 0 only (as b200_gif_first_frame gives it), resized
 *     with Lanczos3 when width / height are set; a JPEG drops the alpha, a PNG or WebP keeps it when some pixel is clear.
 *     webp_lossless answers B200_ERR_UNSUPPORTED.
 * 0 = all of these answer B200_ERR_UNSUPPORTED as before.  While never set, the environment variable B200_GIF_CONVERT=gpu turns it
 * on (read once).  Default off.  Returns B200_OK or B200_ERR_INVALID_ARGUMENT. */
int b200_set_gif_convert(int on);

/* The frame-0 decoder alone (independent of the switch, no device needed): frame 0 of a GIF as the conversions read it, in *rgba as
 * *width * *height pixels of R, G, B, A bytes (released with b200_free).  Inside frame 0's rectangle a pixel is its palette colour,
 * with alpha 0 for the transparent index and 255 otherwise; outside it all four bytes are 0.  The file is checked only up to the
 * end of frame 0's image data.  A frame 0 past the logical screen answers B200_ERR_UNSUPPORTED; a truncated or inconsistent
 * frame 0 answers B200_ERR_CORRUPT_INPUT. */
b200_status b200_gif_first_frame(const uint8_t *in, size_t in_len, int *width, int *height, uint8_t **rgba);

#ifdef __cplusplus
}
#endif
#endif /* B200_CAESIUM_GIF_CONVERT_H */
