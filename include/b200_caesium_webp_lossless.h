/* b200_caesium_webp_lossless.h -- JPEG / PNG -> lossless WebP on the device (opt-in): what libcaesium's convert does with
 * webp.lossless set (caesiumclt --lossless --format webp).  The source is decoded on the device (JPEG: entropy decode, IDCT, upsampling,
 * YCbCr -> RGB; PNG: inflate on the host, un-filter on the device), resized with Lanczos3 when width / height are set, and coded by the
 * project's own VP8L encoder -- its bytes are not libwebp's: 16-25 % larger than libwebp's on photographs and several times larger on
 * flat art, which libwebp codes with a colour-indexing transform.  No metadata is written.  Declared apart from b200_caesium.h while the
 * leg is opt-in. */
#ifndef B200_CAESIUM_WEBP_LOSSLESS_H
#define B200_CAESIUM_WEBP_LOSSLESS_H
#include "b200_caesium.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Process-wide switch: 1 = b200_convert_in_memory(fmt = B200_FMT_WEBP) with webp_lossless set converts JPEG and PNG sources on the
 * device; 0 = those calls answer B200_ERR_UNSUPPORTED as before.  b200_compress_to_size_in_memory with webp_lossless answers
 * B200_ERR_UNSUPPORTED either way: a caller that converts first and then sizes (caesiumclt --max-size --format webp --lossless) gets
 * the conversion from the device and hands only the sizing to libcaesium.  While never set, the environment variable
 * B200_WEBP_LOSSLESS_CONVERT=gpu turns it on (read once).  Default off.  Returns B200_OK or B200_ERR_INVALID_ARGUMENT. */
int b200_set_webp_lossless_convert(int on);

#ifdef __cplusplus
}
#endif
#endif /* B200_CAESIUM_WEBP_LOSSLESS_H */
