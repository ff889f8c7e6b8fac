/* Compiled by tests/test_webp_bpred_host.py with `gcc -std=c99 -pedantic -Wall -Wextra -Werror`:
 * include/b200_caesium_webp_bpred.h must be plain C, its entry points must link against libb200caesium.so, the switch must refuse
 * values other than 0 and 1, and the host writer must refuse a sub-block mode past 9. */
#include <stdio.h>
#include <string.h>
#include "b200_caesium_webp_bpred.h"

typedef void (*fn)(void);

int main(void)
{
    fn all[] = {(fn)b200_set_webp_bpred, (fn)b200_webp_encode_rgb_bpred, (fn)b200_webp_write_levels_bpred};
    size_t i, n = sizeof(all) / sizeof(all[0]);
    int16_t levels[400];
    uint8_t modes[4] = {4, 0, 1, 0}, bmodes[16];
    uint8_t *out = NULL;
    size_t out_len = 0;
    b200_status st;
    for (i = 0; i < n; i++) if (!all[i]) return 1;
    if (b200_set_webp_bpred(2) != B200_ERR_INVALID_ARGUMENT || b200_set_webp_bpred(-1) != B200_ERR_INVALID_ARGUMENT) return 2;
    if (b200_set_webp_bpred(1) != B200_OK || b200_set_webp_bpred(0) != B200_OK) return 3;
    memset(levels, 0, sizeof(levels));
    memset(bmodes, 10, sizeof(bmodes));
    st = b200_webp_write_levels_bpred(16, 16, 75, levels, modes, bmodes, &out, &out_len);
    if (st.code != B200_ERR_INVALID_ARGUMENT) return 4;
    b200_free(st.message);
    memset(bmodes, 9, sizeof(bmodes));
    st = b200_webp_write_levels_bpred(16, 16, 75, levels, modes, bmodes, &out, &out_len);
    if (st.code != B200_OK || !out || out_len < 30) return 5;
    b200_free(out);
    printf("webp bpred c-abi ok\n");
    return 0;
}
