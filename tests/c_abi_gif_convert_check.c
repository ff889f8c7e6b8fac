/* Compiled by tests/test_gif_convert_host.py with `gcc -std=c99 -pedantic -Wall -Wextra -Werror`: include/b200_caesium_gif_convert.h
 * must be plain C, its entry points must link against libb200caesium.so, and the calls that need no device must behave. */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "b200_caesium_gif_convert.h"

typedef void (*fn)(void);

int main(void)
{
    fn all[] = {(fn)b200_set_gif_convert, (fn)b200_gif_first_frame};
    /* a 3x2 screen; frame 0 is 2x1 at (1, 1) with a 2-entry local table, index 1 transparent (its colour 40 50 60 is kept), LZW at
     * minimum code size 2 (CLEAR 0 1 EOI); then a second frame cut short -- never read */
    static const unsigned char gif[] = {'G', 'I', 'F', '8', '9', 'a', 3, 0, 2, 0, 0, 0, 0,
                                        0x21, 0xF9, 4, 1, 0, 0, 1, 0,
                                        0x2C, 1, 0, 1, 0, 2, 0, 1, 0, 0x80, 10, 20, 30, 40, 50, 60,
                                        2, 2, 0x44, 0x0A, 0,
                                        0x2C, 0, 0};
    size_t i, n = sizeof(all) / sizeof(all[0]);
    int w = 0, h = 0;
    uint8_t *rgba = NULL;
    static const uint8_t want[24] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 10, 20, 30, 255, 40, 50, 60, 0};
    b200_status st;

    for (i = 0; i < n; i++) if (!all[i]) return 1;
    if (b200_set_gif_convert(2) != B200_ERR_INVALID_ARGUMENT || b200_set_gif_convert(-1) != B200_ERR_INVALID_ARGUMENT || b200_set_gif_convert(0) != B200_OK) return 2;
    st = b200_gif_first_frame(gif, sizeof(gif), &w, &h, &rgba);
    if (st.code != B200_OK || w != 3 || h != 2 || !rgba) return 3;
    if (memcmp(rgba, want, sizeof(want))) return 4;
    b200_free(rgba);
    /* cut inside frame 0's image data: corrupt input, nothing handed out, a library-allocated message */
    rgba = NULL;
    st = b200_gif_first_frame(gif, 38, &w, &h, &rgba);
    if (st.code != B200_ERR_CORRUPT_INPUT || !st.message || rgba) return 5;
    b200_free(st.message);
    printf("gif convert c-abi ok: %u entry points\n", (unsigned)n);
    return 0;
}
