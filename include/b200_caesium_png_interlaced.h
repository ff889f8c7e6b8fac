/* b200_caesium_png_interlaced.h -- Adam7-interlaced PNG input (opt-in).  With the switch on, every leg that takes a PNG source accepts
 * interlace method 1: lossless and lossy compression, resize, compress_to_size, conversion to WebP (lossless and lossy) and to JPEG,
 * b200_compress_batch, b200_png_resize_samples, b200_png_decode and b200_png_decode_reduced.  The device legs un-filter the seven
 * passes in one wavefront launch and gather the full rows from them; the host decoder does the same on the CPU.  Output is never
 * interlaced: an Adam7 file gives the bytes its non-interlaced twin (the same pixels and chunks) gives.  Declared apart from
 * b200_caesium.h while the input is opt-in. */
#ifndef B200_CAESIUM_PNG_INTERLACED_H
#define B200_CAESIUM_PNG_INTERLACED_H
#include "b200_caesium.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Process-wide switch: 1 = Adam7 PNG sources are decoded; 0 = they answer B200_ERR_UNSUPPORTED with "interlaced PNG is not supported
 * on the GPU path", as before.  Interlace methods other than 0 and 1 answer that way whatever the switch says.  While never set,
 * the environment variable B200_PNG_INTERLACED=gpu turns it on (read once).  Default off.  Returns B200_OK or
 * B200_ERR_INVALID_ARGUMENT. */
int b200_set_png_interlaced(int on);

#ifdef __cplusplus
}
#endif
#endif /* B200_CAESIUM_PNG_INTERLACED_H */
