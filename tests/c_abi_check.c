/* Compiled by tests/test_c_abi.py with `gcc -std=c99 -pedantic -Wall -Wextra -Werror`: include/b200_caesium.h must be plain C,
 * every declared entry point must link against libb200caesium.so, and the calls that need no device must behave. */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "b200_caesium.h"

typedef void (*fn)(void);

int main(void)
{
    /* taking the address of every declared function makes the linker resolve all of them */
    fn all[] = {
        (fn)b200_params_default, (fn)b200_init, (fn)b200_init_device, (fn)b200_shutdown, (fn)b200_device_count, (fn)b200_version, (fn)b200_free,
        (fn)b200_set_entropy_mode, (fn)b200_compress_in_memory, (fn)b200_convert_in_memory, (fn)b200_compress_to_size_in_memory, (fn)b200_compress_batch,
        (fn)b200_sniff_format, (fn)b200_jpeg_decode_coefficients, (fn)b200_jpeg_output_layout, (fn)b200_jpeg_requantize, (fn)b200_jpeg_encode_coefficients,
        (fn)b200_jpeg_encode_coefficients_device, (fn)b200_jpeg_decode_planes, (fn)b200_jpeg_quant_table,
        (fn)b200_png_decode, (fn)b200_png_decode_reduced, (fn)b200_png_filter, (fn)b200_png_lz77, (fn)b200_png_deflate_tokens, (fn)b200_png_level_strategies,
        (fn)b200_webp_encode_rgb, (fn)b200_webp_write_levels, (fn)b200_webp_qindex,
        (fn)b200_jpeg_pipe_create, (fn)b200_jpeg_pipe_run, (fn)b200_jpeg_pipe_finish, (fn)b200_jpeg_pipe_fetch, (fn)b200_jpeg_pipe_kernel_times, (fn)b200_jpeg_pipe_destroy, (fn)b200_device_jobs, (fn)b200_device_numa_node, (fn)b200_png_device_times, (fn)b200_webp_decode, (fn)b200_webp_alpha_chunk, (fn)b200_webp_wrap_alpha, (fn)b200_webp_decode_rgba, (fn)b200_webp_alpha_filter, (fn)b200_webp_d2h_bytes,
    };
    size_t i, n = sizeof(all) / sizeof(all[0]);
    b200_params p;
    static const unsigned char png_sig[8] = {0x89, 'P', 'N', 'G', '\r', '\n', 0x1a, '\n'};
    static const unsigned char jpg_sig[4] = {0xff, 0xd8, 0xff, 0xe0};
    static const unsigned char webp_sig[12] = {'R', 'I', 'F', 'F', 0, 0, 0, 0, 'W', 'E', 'B', 'P'};
    uint16_t qt[64];
    int f[6];
    b200_status st;
    uint8_t *out = NULL;
    size_t out_len = 0;

    for (i = 0; i < n; i++) if (!all[i]) return 1;
    b200_params_default(&p);
    if (p.jpeg_quality != 80 || p.png_optimization_level != 3 || !p.jpeg_progressive) return 2;
    if (b200_sniff_format(png_sig, 8) != B200_FMT_PNG || b200_sniff_format(jpg_sig, 4) != B200_FMT_JPEG || b200_sniff_format(webp_sig, 12) != B200_FMT_WEBP ||
        b200_sniff_format((const uint8_t *)"nope", 4) != B200_FMT_UNKNOWN) return 3;
    if (!b200_version() || !strstr(b200_version(), "sm_90a")) return 4;
    b200_jpeg_quant_table(80, 0, qt);
    if (qt[0] == 0 || qt[63] == 0) return 5;
    if (b200_webp_qindex(100, f) != 0 || f[0] != 4 || b200_webp_qindex(0, f) != 127 || f[1] != 284) return 6;
    /* an unknown format is refused without touching the device; the status message is library-allocated */
    st = b200_compress_in_memory((const uint8_t *)"not an image", 12, &p, &out, &out_len);
    if (st.code != B200_ERR_UNKNOWN_FORMAT || !st.message || out) return 7;
    b200_free(st.message);
    st = b200_convert_in_memory(jpg_sig, 4, &p, B200_FMT_JPEG, &out, &out_len);
    if (st.code != B200_ERR_SAME_FORMAT) return 8;
    b200_free(st.message);
    printf("c-abi ok: %u entry points, %s\n", (unsigned)n, b200_version());
    return 0;
}
