/* Compiled by tests/test_c_abi_gif.py with `gcc -std=c99 -pedantic -Wall -Wextra -Werror`: include/b200_caesium_gif.h must be
 * plain C, its entry points must link against libb200caesium.so, and the calls that need no device must behave. */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "b200_caesium_gif.h"

typedef void (*fn)(void);

int main(void)
{
    fn all[] = {(fn)b200_set_gif, (fn)b200_gif_decode, (fn)b200_gif_lzw};
    /* a 2x1 GIF: no global table, one frame with a 2-entry local table, LZW at minimum code size 2 (CLEAR 0 1 EOI) */
    static const unsigned char gif[] = {'G', 'I', 'F', '8', '9', 'a', 2, 0, 1, 0, 0, 0, 0,
                                        0x2C, 0, 0, 0, 0, 2, 0, 1, 0, 0x80, 10, 20, 30, 40, 50, 60,
                                        2, 2, 0x44, 0x0A, 0, 0x3B};
    size_t i, n = sizeof(all) / sizeof(all[0]);
    int w = 0, h = 0, frames = 0, loop = 0, *delays = NULL;
    uint8_t *rgba = NULL;
    b200_status st;

    for (i = 0; i < n; i++) if (!all[i]) return 1;
    if (b200_set_gif(2) != B200_ERR_INVALID_ARGUMENT || b200_set_gif(0) != B200_OK) return 2;
    st = b200_gif_decode(gif, sizeof(gif), &w, &h, &frames, &loop, &rgba, &delays);
    if (st.code != B200_OK || w != 2 || h != 1 || frames != 1 || loop != -1 || !rgba || !delays) return 3;
    if (rgba[0] != 10 || rgba[1] != 20 || rgba[2] != 30 || rgba[3] != 255 || rgba[4] != 40 || rgba[7] != 255 || delays[0] != 0) return 4;
    b200_free(rgba); b200_free(delays);
    /* truncated: corrupt input, nothing handed out, a library-allocated message */
    rgba = NULL; delays = NULL;
    st = b200_gif_decode(gif, sizeof(gif) - 3, &w, &h, &frames, &loop, &rgba, &delays);
    if (st.code != B200_ERR_CORRUPT_INPUT || !st.message || rgba || delays) return 5;
    b200_free(st.message);
    printf("gif c-abi ok: %u entry points\n", (unsigned)n);
    return 0;
}
