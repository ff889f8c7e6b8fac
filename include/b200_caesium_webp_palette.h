/* b200_caesium_webp_palette.h -- the colour-indexing (palette) transform for lossless WebP (opt-in).  With the switch on, every
 * lossless WebP output -- `--lossless` on WebP sources, JPEG / PNG -> lossless WebP and the lossless frames of animated WebP -- also
 * codes an image of at most 256 distinct ARGB colours through a palette (ascending by ARGB value, indices bundled 2, 4 or 8 to a
 * pixel when there are at most 16, 4 or 2 colours) and keeps the smaller file, the one without the palette on a tie.  So a file is
 * never larger than with the switch off; images of more colours are coded exactly as before.  Declared apart from b200_caesium.h
 * while the leg is opt-in. */
#ifndef B200_CAESIUM_WEBP_PALETTE_H
#define B200_CAESIUM_WEBP_PALETTE_H
#include "b200_caesium.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Process-wide switch: 1 = lossless WebP outputs also try the palette; 0 = they never do, as before.  While never set, the
 * environment variable B200_WEBP_PALETTE=gpu turns it on (read once).  Default off.  Returns B200_OK or B200_ERR_INVALID_ARGUMENT. */
int b200_set_webp_palette(int on);

#ifdef __cplusplus
}
#endif
#endif /* B200_CAESIUM_WEBP_PALETTE_H */
