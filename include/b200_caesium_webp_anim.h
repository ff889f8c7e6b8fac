/* b200_caesium_webp_anim.h -- animated WebP on the device (opt-in): every frame is composited the way libwebp's WebPAnimDecoder
 * does, the changed box of each new canvas is re-encoded with the lossy VP8 encoder (webp_quality) or, with webp_lossless, the
 * lossless VP8L encoder, and the host writes the container (DESIGN.md §4.15).  libcaesium re-encodes animations through libwebp's
 * WebPAnimEncoder, whose blend, dispose and keyframe search this leg does not reproduce, so it is off until the integrator turns
 * it on: with the switch off every call answers exactly as before (B200_ERR_UNSUPPORTED for an animated WebP).  Declared apart
 * from b200_caesium.h while the leg is opt-in. */
#ifndef B200_CAESIUM_WEBP_ANIM_H
#define B200_CAESIUM_WEBP_ANIM_H
#include "b200_caesium.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Process-wide switch: 1 = b200_compress_in_memory and b200_compress_batch on animated WebP sources run the device leg; 0 = they
 * answer B200_ERR_UNSUPPORTED.  While never set, the environment variable B200_WEBP_ANIM=gpu turns it on (read once).  Default
 * off.  Resizing (width / height), compress_to_size and every conversion from an animated WebP answer B200_ERR_UNSUPPORTED either
 * way, and b200_webp_decode / b200_webp_decode_rgba keep refusing animations.  Returns B200_OK or B200_ERR_INVALID_ARGUMENT. */
int b200_set_webp_anim(int on);

/* The host decoder alone (independent of the switch, no device needed): the composited canvas of every frame (*nframes frames of
 * width * height pixels as R, G, B, A bytes) in *rgba, each frame's duration in ms in *durations, the ANIM loop count in *loop
 * (0: forever) and its background colour bytes, as stored, in bg.  *rgba and *durations are released with b200_free.  Truncated
 * or inconsistent data, a frame outside the canvas and a canvas side above 16383 answer B200_ERR_CORRUPT_INPUT. */
b200_status b200_webp_anim_decode(const uint8_t *in, size_t in_len, int *width, int *height, int *nframes, int *loop, uint8_t bg[4], uint8_t **rgba,
                                  int **durations);

#ifdef __cplusplus
}
#endif
#endif /* B200_CAESIUM_WEBP_ANIM_H */
