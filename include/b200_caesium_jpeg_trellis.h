/* b200_caesium_jpeg_trellis.h -- rate-distortion ("trellis") quantisation of lossy JPEG output on the device (opt-in).  Per 8x8
 * block, every AC level may drop to zero or to a smaller magnitude where the bits it saves outweigh the error it adds, weighed
 * the way mozjpeg's trellis does (DESIGN.md §4).  Smaller files at the same quality setting, but not the bytes of plain
 * quantisation, so it is off until the integrator turns it on: with the switch off every call answers exactly as before.
 * Declared apart from b200_caesium.h while the leg is opt-in. */
#ifndef B200_CAESIUM_JPEG_TRELLIS_H
#define B200_CAESIUM_JPEG_TRELLIS_H
#include "b200_caesium.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Process-wide switch: 1 = every lossy JPEG output -- b200_compress_in_memory and b200_compress_batch (JPEG re-encode, resize
 * included), b200_convert_in_memory to JPEG, each try of b200_compress_to_size_in_memory on a JPEG, and b200_jpeg_pipe_* (read
 * at create) -- is quantised by the trellis; 0 = plain round-to-nearest quantisation.  The lossless transcode (jpeg_optimize)
 * never quantises and is not affected.  While never set, the environment variable B200_JPEG_TRELLIS=1 turns it on (read once).
 * Default off.  Returns B200_OK or B200_ERR_INVALID_ARGUMENT. */
int b200_set_jpeg_trellis(int on);

#ifdef __cplusplus
}
#endif
#endif /* B200_CAESIUM_JPEG_TRELLIS_H */
