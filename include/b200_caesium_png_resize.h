/* b200_caesium_png_resize.h -- PNG -> PNG with a target size on the device (opt-in): what libcaesium does for a PNG with width /
 * height set (decode to the image crate's type, Lanczos3 resize_exact, then oxipng or imagequant).  The samples are expanded to the
 * decoded type (every channel kept, 16 bits stay 16 bits; palette -> RGB(A)8, a tRNS colour key adds alpha), resized with the
 * library's Lanczos3 kernels and handed to the lossless or lossy PNG back end.  The resized file carries none of the source's
 * ancillary chunks, whatever keep_metadata says.  Declared apart from b200_caesium.h while the leg is opt-in. */
#ifndef B200_CAESIUM_PNG_RESIZE_H
#define B200_CAESIUM_PNG_RESIZE_H
#include "b200_caesium.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Process-wide switch: 1 = b200_compress_in_memory and b200_compress_batch on PNG sources with width or height set resize on the
 * device (lossless with png_optimize; lossy additionally needs b200_set_png_lossy), and so does b200_compress_to_size_in_memory
 * (which needs both switches); 0 = those calls answer B200_ERR_UNSUPPORTED as before.  While never set, the environment variable
 * B200_PNG_RESIZE=gpu turns it on (read once).  Default off.  Returns B200_OK or B200_ERR_INVALID_ARGUMENT. */
int b200_set_png_resize(int on);

/* The expansion and resize alone on the current device (independent of the switch): width / height as in b200_params (both 0: the
 * expanded image at the source's size).  *raw (released with b200_free) receives info->height rows of info->row_bytes bytes in PNG
 * byte order (interleaved, 16-bit samples big-endian); info describes the decoded type at the target size.  Corrupt input answers
 * B200_ERR_CORRUPT_INPUT, interlaced input B200_ERR_UNSUPPORTED. */
b200_status b200_png_resize_samples(const uint8_t *in, size_t in_len, uint32_t width, uint32_t height, b200_png_info *info, uint8_t **raw);

#ifdef __cplusplus
}
#endif
#endif /* B200_CAESIUM_PNG_RESIZE_H */
