/* Compiled by tests/test_webp_palette_host.py with `gcc -std=c99 -pedantic -Wall -Wextra -Werror`:
 * include/b200_caesium_webp_palette.h must be plain C, its entry point must link against libb200caesium.so, and the switch must
 * refuse values other than 0 and 1. */
#include <stdio.h>
#include "b200_caesium_webp_palette.h"

typedef void (*fn)(void);

int main(void)
{
    fn all[] = {(fn)b200_set_webp_palette};
    size_t i, n = sizeof(all) / sizeof(all[0]);
    for (i = 0; i < n; i++) if (!all[i]) return 1;
    if (b200_set_webp_palette(2) != B200_ERR_INVALID_ARGUMENT || b200_set_webp_palette(-1) != B200_ERR_INVALID_ARGUMENT) return 2;
    if (b200_set_webp_palette(1) != B200_OK || b200_set_webp_palette(0) != B200_OK) return 3;
    printf("webp palette c-abi ok\n");
    return 0;
}
