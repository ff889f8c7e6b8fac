/* Compiled by tests/test_png_zopfli_host.py with `gcc -std=c99 -pedantic -Wall -Wextra -Werror`:
 * include/b200_caesium_png_zopfli.h must be plain C, its entry points must link against libb200caesium.so, the switch must refuse
 * values other than 0 and 1, and the stage entry point must refuse null arguments before it looks for a device. */
#include <stdio.h>
#include "b200_caesium_png_zopfli.h"

typedef void (*fn)(void);

int main(void)
{
    fn all[] = {(fn)b200_set_png_zopfli, (fn)b200_png_lz77_zopfli};
    size_t i, n = sizeof(all) / sizeof(all[0]), nt = 0;
    uint32_t *tok = NULL;
    for (i = 0; i < n; i++) if (!all[i]) return 1;
    if (b200_set_png_zopfli(2) != B200_ERR_INVALID_ARGUMENT || b200_set_png_zopfli(-1) != B200_ERR_INVALID_ARGUMENT) return 2;
    if (b200_set_png_zopfli(1) != B200_OK || b200_set_png_zopfli(0) != B200_OK) return 3;
    if (b200_png_lz77_zopfli(NULL, 4, 1, 4, &tok, &nt).code != B200_ERR_INVALID_ARGUMENT) return 4;
    printf("png zopfli c-abi ok\n");
    return 0;
}
