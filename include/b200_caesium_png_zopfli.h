/* b200_caesium_png_zopfli.h -- `--zopfli` on the device (opt-in).  With the switch on, png_force_zopfli = 1 makes every PNG output
 * (lossless and lossy, PNG -> PNG resize, Adam7 sources, the palette-reduced path, JPEG / WebP / GIF -> PNG and every
 * compress_to_size try) also code the chosen filtered stream from an iterated optimal LZ77 parse -- zopfli's method: a shortest path
 * over every match a position offers, re-run 15 times with symbol costs from the previous parse -- and emit the smaller of that and
 * the default zlib payload (the default on a tie).  The filter choice does not move, and a file is never larger than without the
 * flag.  Declared apart from b200_caesium.h while the leg is opt-in. */
#ifndef B200_CAESIUM_PNG_ZOPFLI_H
#define B200_CAESIUM_PNG_ZOPFLI_H
#include "b200_caesium.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Process-wide switch: 1 = png_force_zopfli takes the optimal parse; 0 = png_force_zopfli is accepted and ignored, as before.  While
 * never set, the environment variable B200_PNG_ZOPFLI=gpu turns it on (read once).  Default off.  Returns B200_OK or
 * B200_ERR_INVALID_ARGUMENT. */
int b200_set_png_zopfli(int on);

/* The optimal parse of a filtered stream (filter distance bpp 1..8, row stride in bytes), whatever the switch says: *tokens
 * (library-allocated, free with b200_free) in b200_png_lz77's format, *ntokens their number. */
b200_status b200_png_lz77_zopfli(const uint8_t *filtered, size_t n, int bpp, int stride, uint32_t **tokens, size_t *ntokens);

#ifdef __cplusplus
}
#endif
#endif /* B200_CAESIUM_PNG_ZOPFLI_H */
