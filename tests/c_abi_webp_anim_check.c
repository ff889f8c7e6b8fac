/* Compiled by tests/test_c_abi_webp_anim.py with `gcc -std=c99 -pedantic -Wall -Wextra -Werror`: include/b200_caesium_webp_anim.h
 * must be plain C, its entry points must link against libb200caesium.so, and the calls that need no device must behave.  The file
 * to decode is the first argument. */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "b200_caesium_webp_anim.h"

typedef void (*fn)(void);

int main(int argc, char **argv)
{
    fn all[] = {(fn)b200_set_webp_anim, (fn)b200_webp_anim_decode};
    size_t i, n = sizeof(all) / sizeof(all[0]), len;
    int w = 0, h = 0, frames = 0, loop = -1, *durations = NULL;
    uint8_t bg[4], *rgba = NULL;
    unsigned char *data;
    b200_status st;
    FILE *f;

    for (i = 0; i < n; i++) if (!all[i]) return 1;
    if (b200_set_webp_anim(2) != B200_ERR_INVALID_ARGUMENT || b200_set_webp_anim(0) != B200_OK) return 2;
    if (argc < 2 || !(f = fopen(argv[1], "rb"))) return 3;
    data = (unsigned char *)malloc(1 << 20);
    len = fread(data, 1, 1 << 20, f);
    fclose(f);
    st = b200_webp_anim_decode(data, len, &w, &h, &frames, &loop, bg, &rgba, &durations);
    if (st.code != B200_OK || w != 17 || h != 13 || frames != 4 || loop != 65535 || !rgba || !durations) return 4;
    if (bg[0] != 0x10 || bg[3] != 0x40 || durations[0] != 5) return 5;
    /* the first frame is one pixel at (4, 2); everything else on the canvas is clear */
    for (i = 0; i < (size_t)(w * h); i++) if (i != (size_t)(2 * w + 4) && (rgba[4 * i] | rgba[4 * i + 1] | rgba[4 * i + 2] | rgba[4 * i + 3])) return 6;
    b200_free(rgba); b200_free(durations);
    /* truncated: corrupt input, nothing handed out, a library-allocated message */
    rgba = NULL; durations = NULL;
    st = b200_webp_anim_decode(data, len - 5, &w, &h, &frames, &loop, bg, &rgba, &durations);
    if (st.code != B200_ERR_CORRUPT_INPUT || !st.message || rgba || durations) return 7;
    b200_free(st.message);
    free(data);
    printf("webp anim c-abi ok: %u entry points\n", (unsigned)n);
    return 0;
}
