/* gif_core.h -- the rules of the GIF re-encoder, written once for every party that has to agree on them: the device kernels and
 * their host driver (gif_kernels.cu, gif_device.cu) and the scalar oracle (oracle/gif_oracle.c, plain C -- hence no namespace and
 * no C++ in this file).
 *
 *   frames        each source frame is composited to a full RGBA canvas (alpha 0 or 255, a clear pixel is 0x00000000); a canvas
 *                 equal to the previous one is dropped and its delay added to the previous output frame (at most 65535)
 *   rectangle     output frame i covers the bounding box of the pixels that differ from canvas i-1 (D), of the pixels that the
 *                 next kept canvas turns from opaque to clear (K), and, when frame i-1 is disposed to background, frame i-1's own
 *                 rectangle (R); frame 0 covers the whole canvas
 *   pixels        inside its rectangle a frame draws canvas i where the pixel lies in R or differs from canvas i-1, and is
 *                 transparent elsewhere (the viewer keeps what it showed, so dither noise does not flicker); frame 0 draws canvas 0
 *   disposal      2 (restore to background) when K is not empty -- the viewer clears the rectangle, which covers K, before the next
 *                 frame draws it again -- else 1 (leave in place).  A frame cannot clear a pixel by drawing it, hence K.
 *   colours       every frame has its own local colour table from the palette quantiser (png_quant_core.h) at gif_quality, with
 *                 the exact path only at quality 100; a palette whose entry 0 is clear makes 0 the transparent index
 *   LZW           the indices in raster order are cut into segments of GIF_SEG pixels; each segment follows a CLEAR code and is
 *                 greedy GIF LZW on its own (widths m + 1 .. 12, a width grows when the decoder's next code reaches 2^width, no
 *                 early change; CLEAR when the dictionary fills); one EOI ends the stream.  Codes are packed LSB first without
 *                 a break at segment boundaries, so any GIF decoder reads the stream. */
#ifndef GIF_CORE_H
#define GIF_CORE_H
#include <stddef.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define GIF_HD static __host__ __device__ __forceinline__
#else
#define GIF_HD static inline
#endif

#ifdef __cplusplus
namespace b200 {
#endif

enum {
    GIF_SEG = 16384,                                  /* pixels per LZW segment (DESIGN.md §4.11 has the table it was chosen from) */
    GIF_SEG_CODES = GIF_SEG + GIF_SEG / 1024 + 4,     /* codes one segment can emit: data codes, dictionary-full CLEARs, the ends */
    GIF_HASH = 8192,                                  /* dictionary hash slots of one walker (32 KiB): load factor at most 1/2 */
    GIF_MAX_DELAY = 65535
};

/* a rectangle [x0, x1) x [y0, y1); empty when x1 <= x0 */
typedef struct { int x0, y0, x1, y1; } GifRect;

GIF_HD int gif_rect_empty(GifRect r) { return r.x1 <= r.x0 || r.y1 <= r.y0; }
GIF_HD int gif_in_rect(GifRect r, int x, int y) { return x >= r.x0 && x < r.x1 && y >= r.y0 && y < r.y1; }
GIF_HD GifRect gif_union(GifRect a, GifRect b)
{
    if (gif_rect_empty(a)) return b;
    if (gif_rect_empty(b)) return a;
    GifRect r = {a.x0 < b.x0 ? a.x0 : b.x0, a.y0 < b.y0 ? a.y0 : b.y0, a.x1 > b.x1 ? a.x1 : b.x1, a.y1 > b.y1 ? a.y1 : b.y1};
    return r;
}

/* the pixel a frame draws at a position inside its rectangle (redraw: the position lies in R, or this is frame 0) */
GIF_HD uint32_t gif_out_pixel(uint32_t prev, uint32_t cur, int redraw) { return redraw || prev != cur ? cur : 0u; }

/* the canvas pixel of a converted source pixel: clear (0x00000000) where alpha is 0, else opaque -- the gif crate's
 * Frame::from_rgba_speed makes every other alpha 255 */
GIF_HD uint32_t gif_canvas_pixel(uint32_t r, uint32_t g, uint32_t b, uint32_t a) { return a ? (r | g << 8 | b << 16 | 0xFF000000u) : 0u; }

/* colour table size field s (2^(s+1) entries hold n) and the LZW minimum code size */
GIF_HD int gif_table_bits(int n) { int s = 0; while ((1 << (s + 1)) < n) s++; return s; }
GIF_HD int gif_min_code_size(int n) { const int s = gif_table_bits(n) + 1; return s < 2 ? 2 : s; }

/* Greedy LZW of one segment: idx[0, n) at minimum code size m, after a CLEAR (`first`: this segment also emits the stream's
 * opening CLEAR; `last`: it ends with EOI, otherwise with the CLEAR that opens the next segment).  Codes go to `codes` as
 * code | width << 12; returns their count and sets *bits to the sum of their widths.  table: GIF_HASH words of scratch, a slot
 * holding (prefix << 8 | byte) << 12 | code (empty: all ones -- prefix 4095 never extends, the dictionary is cleared when 4095
 * is assigned). */
GIF_HD int gif_lzw_segment(const uint8_t *idx, int n, int m, int first, int last, uint32_t *table, uint16_t *codes, unsigned *bits)
{
    const uint32_t clear = 1u << m, first_code = clear + 2;
    int nc = 0, w = m + 1, fresh = 1;
    unsigned b = 0;
    uint32_t next = first_code, dn = first_code;      /* the encoder's next code, and the decoder's (one entry behind) */
    for (int i = 0; i < GIF_HASH; i++) table[i] = 0xFFFFFFFFu;
    if (first) { codes[nc++] = (uint16_t)(clear | (uint32_t)w << 12); b += (unsigned)w; }
    if (n > 0) {
        uint32_t cur = idx[0];
        for (int i = 1; i <= n; i++) {
            uint32_t h = 0, key = 0;
            if (i < n) {
                key = cur << 8 | idx[i];
                h = (key * 2654435761u) >> 19;
                uint32_t e;
                while ((e = table[h]) != 0xFFFFFFFFu && (e >> 12) != key) h = (h + 1) & (GIF_HASH - 1);
                if (e != 0xFFFFFFFFu) { cur = e & 4095u; continue; }
            }
            codes[nc++] = (uint16_t)(cur | (uint32_t)w << 12); b += (unsigned)w;
            if (!fresh) { dn++; if (dn == (1u << w) && w < 12) w++; }
            fresh = 0;
            if (i == n) break;
            table[h] = key << 12 | next;
            if (++next == 4096) {
                codes[nc++] = (uint16_t)(clear | (uint32_t)w << 12); b += (unsigned)w;
                for (int k = 0; k < GIF_HASH; k++) table[k] = 0xFFFFFFFFu;
                w = m + 1; next = dn = first_code; fresh = 1;
            }
            cur = idx[i];
        }
    }
    codes[nc++] = (uint16_t)((last ? clear + 1 : clear) | (uint32_t)w << 12); b += (unsigned)w;
    *bits = b;
    return nc;
}

/* sub-blocked image data of nbytes LZW bytes: 255-byte blocks, each after its length, then the 0 terminator */
GIF_HD size_t gif_blocks_size(size_t nbytes) { return nbytes + (nbytes + 254) / 255 + 1; }
GIF_HD uint8_t gif_blocks_byte(const uint8_t *data, size_t nbytes, size_t i)
{
    const size_t blk = i / 256, r = i % 256, at = blk * 255;
    if (at >= nbytes) return 0;
    const size_t len = nbytes - at < 255 ? nbytes - at : 255;
    if (r == 0) return (uint8_t)len;
    return r > len ? 0 : data[at + r - 1];
}

/* ---- container (host side) ----------------------------------------------------------------------------------------------------- */
static inline uint8_t *gif_put16(uint8_t *o, int v) { o[0] = (uint8_t)v; o[1] = (uint8_t)(v >> 8); return o + 2; }

/* GIF89a header, a logical screen without a global table, and NETSCAPE2.0 when loop >= 0; returns bytes written (at most 32) */
static inline int gif_put_header(uint8_t *o, int w, int h, int loop)
{
    uint8_t *p = o;
    const char *sig = "GIF89a";
    for (int i = 0; i < 6; i++) *p++ = (uint8_t)sig[i];
    p = gif_put16(p, w); p = gif_put16(p, h);
    *p++ = 0; *p++ = 0; *p++ = 0;
    if (loop >= 0) {
        const char *app = "NETSCAPE2.0";
        *p++ = 0x21; *p++ = 0xFF; *p++ = 11;
        for (int i = 0; i < 11; i++) *p++ = (uint8_t)app[i];
        *p++ = 3; *p++ = 1; p = gif_put16(p, loop); *p++ = 0;
    }
    return (int)(p - o);
}

/* graphic control extension, image descriptor with a local table of palette[0, n) (RGBA words, R in the low byte) and the
 * minimum code size byte; returns bytes written (at most 8 + 10 + 768 + 1) */
static inline int gif_put_frame_head(uint8_t *o, int delay, int disposal, GifRect r, const uint32_t *palette, int n)
{
    uint8_t *p = o;
    const int transparent = n > 0 && (palette[0] >> 24) == 0, s = gif_table_bits(n);
    *p++ = 0x21; *p++ = 0xF9; *p++ = 4;
    *p++ = (uint8_t)(disposal << 2 | transparent);
    p = gif_put16(p, delay);
    *p++ = 0; *p++ = 0;
    *p++ = 0x2C;
    p = gif_put16(p, r.x0); p = gif_put16(p, r.y0); p = gif_put16(p, r.x1 - r.x0); p = gif_put16(p, r.y1 - r.y0);
    *p++ = (uint8_t)(0x80 | s);
    for (int k = 0; k < (2 << s); k++) {
        const uint32_t c = k < n ? palette[k] : 0;
        *p++ = (uint8_t)c; *p++ = (uint8_t)(c >> 8); *p++ = (uint8_t)(c >> 16);
    }
    *p++ = (uint8_t)gif_min_code_size(n);
    return (int)(p - o);
}

#ifdef __cplusplus
}
#endif
#endif /* GIF_CORE_H */
