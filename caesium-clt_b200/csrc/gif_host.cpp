// gif_host.cpp -- GIF decoding on the calling thread (gif_host.h).  Every length and code is checked against what remains of the
// input and of the frame, so truncated or inconsistent data is refused and nothing is read out of bounds.
#include "gif_host.h"
#include <cstring>

namespace b200 {

namespace {

uint32_t rd16(const uint8_t *p) { return (uint32_t)p[0] | (uint32_t)p[1] << 8; }

// skips the sub-blocks at pos up to and including the terminator; false when the data ends first
bool skip_blocks(const uint8_t *d, size_t n, size_t &pos)
{
    for (;;) {
        if (pos >= n) return false;
        const size_t len = d[pos++];
        if (!len) return true;
        if (len > n - pos) return false;
        pos += len;
    }
}

void read_table(const uint8_t *p, int count, uint32_t *t)
{
    for (int i = 0; i < count; i++) t[i] = (uint32_t)p[3 * i] | (uint32_t)p[3 * i + 1] << 8 | (uint32_t)p[3 * i + 2] << 16 | 0xFF000000u;
}

// LZW image data (already joined from its sub-blocks) -> npix indices; false on a bad code or too little data
bool lzw_decode(const uint8_t *data, size_t n, int m, uint8_t *out, size_t npix, std::string &err)
{
    static thread_local uint16_t prefix[4096];
    static thread_local uint8_t suffix[4096], firstc[4096], stack[4097];
    const int clear = 1 << m, eoi = clear + 1;
    for (int i = 0; i < clear; i++) { suffix[i] = firstc[i] = (uint8_t)i; prefix[i] = 0xFFFF; }
    int w = m + 1, next = clear + 2, prev = -1;
    size_t pos = 0, bitpos = 0;
    const size_t nbits = n * 8;
    while (pos < npix) {
        if (bitpos + (size_t)w > nbits) break;
        int code = 0;
        for (int k = 0; k < w; k++, bitpos++) code |= ((data[bitpos >> 3] >> (bitpos & 7)) & 1) << k;
        if (code == clear) { w = m + 1; next = clear + 2; prev = -1; continue; }
        if (code == eoi) break;
        if (prev < 0) {
            if (code >= clear) { err = "GIF LZW: a code refers to no dictionary entry"; return false; }
            out[pos++] = (uint8_t)code; prev = code;
            continue;
        }
        if (code > next || (code == next && next >= 4096)) { err = "GIF LZW: a code refers to no dictionary entry"; return false; }
        int sp = 0, c = code;
        if (code == next) { stack[sp++] = firstc[prev]; c = prev; }
        while (c >= clear) { stack[sp++] = suffix[c]; c = prefix[c]; }
        stack[sp++] = (uint8_t)c;
        while (sp > 0 && pos < npix) out[pos++] = stack[--sp];
        if (next < 4096) {
            prefix[next] = (uint16_t)prev; suffix[next] = (uint8_t)c; firstc[next] = firstc[prev];
            next++;
            if (next == (1 << w) && w < 12) w++;
        }
        prev = code;
    }
    if (pos < npix) { err = "GIF image data too short"; return false; }
    return true;
}

// row k of the image data of a frame fh rows high -> its row in the frame (interlaced: the four passes of rows 8k, 8k + 4, 4k + 2, 2k + 1)
int frame_row(int k, int fh, bool interlaced)
{
    if (!interlaced) return k;
    const int p1 = (fh + 7) / 8, p2 = (fh + 3) / 8, p3 = (fh + 1) / 4;
    return k < p1 ? 8 * k : k < p1 + p2 ? 8 * (k - p1) + 4 : k < p1 + p2 + p3 ? 4 * (k - p1 - p2) + 2 : 2 * (k - p1 - p2 - p3) + 1;
}

} // namespace

bool GifReader::read_screen(const uint8_t *d, size_t n, std::string &err)
{
    d_ = d; n_ = n; frames = 0; loop = -1; unsupported = false;
    if (n < 13 || (memcmp(d, "GIF87a", 6) && memcmp(d, "GIF89a", 6))) { err = "not a GIF"; return false; }
    width = (int)rd16(d + 6); height = (int)rd16(d + 8);
    if (!width || !height) { err = "GIF logical screen is empty"; return false; }
    size_t pos = 13;
    gct_n_ = 0;
    if (d[10] & 0x80) {
        gct_n_ = 2 << (d[10] & 7);
        if ((size_t)gct_n_ * 3 > n - pos) { err = "GIF global colour table truncated"; return false; }
        read_table(d + pos, gct_n_, gct_);
        pos += (size_t)gct_n_ * 3;
    }
    first_block_ = pos;
    return true;
}

bool GifReader::walk_block(size_t &pos, uint8_t &kind, std::string &err)
{
    const uint8_t *d = d_;
    const size_t n = n_;
    if (pos >= n) { err = "GIF truncated (no trailer)"; return false; }
    const uint8_t b = kind = d[pos++];
    if (b == 0x3B) return true;
    if (b == 0x21) {
        if (pos >= n) { err = "GIF extension truncated"; return false; }
        const uint8_t label = d[pos++];
        if (label == 0xFF && pos + 12 <= n && d[pos] == 11 && !memcmp(d + pos + 1, "NETSCAPE2.0", 11)) {
            const size_t q = pos + 12;
            if (q + 4 <= n && d[q] == 3 && d[q + 1] == 1) loop = (int)rd16(d + q + 2);
        }
        if (label == 0xF9 && (pos >= n || d[pos] < 4)) { err = "GIF graphic control extension too short"; return false; }
        if (!skip_blocks(d, n, pos)) { err = "GIF extension truncated"; return false; }
        return true;
    }
    if (b != 0x2C) { err = "GIF block of unknown type"; return false; }
    if (n - pos < 9) { err = "GIF image descriptor truncated"; return false; }
    const uint32_t x = rd16(d + pos), y = rd16(d + pos + 2), w = rd16(d + pos + 4), h = rd16(d + pos + 6);
    const uint8_t f = d[pos + 8];
    pos += 9;
    if (x + w > (uint32_t)width || y + h > (uint32_t)height) { unsupported = true; err = "a GIF frame extends past the logical screen"; return false; }
    if (f & 0x80) {
        const size_t t = (size_t)(2 << (f & 7)) * 3;
        if (t > n - pos) { err = "GIF local colour table truncated"; return false; }
        pos += t;
    } else if (!gct_n_) { err = "GIF frame without a colour table"; return false; }
    if (pos >= n) { err = "GIF image data truncated"; return false; }
    if (d[pos] < 2 || d[pos] > 8) { err = "GIF LZW minimum code size out of range"; return false; }
    pos++;
    if (!skip_blocks(d, n, pos)) { err = "GIF image data truncated"; return false; }
    return true;
}

bool GifReader::read_image(Image &im, std::string &err)
{
    const uint8_t *d = d_;
    im.x = (int)rd16(d + pos_); im.y = (int)rd16(d + pos_ + 2); im.w = (int)rd16(d + pos_ + 4); im.h = (int)rd16(d + pos_ + 6);
    const uint8_t f = d[pos_ + 8];
    pos_ += 9;
    im.interlaced = (f & 0x40) != 0;
    im.table = gct_; im.tn = gct_n_;
    if (f & 0x80) { im.tn = 2 << (f & 7); read_table(d + pos_, im.tn, im.lct); im.table = im.lct; pos_ += (size_t)im.tn * 3; }
    const int m = d[pos_++];
    lzw_.clear();
    for (;;) {
        const size_t len = d[pos_++];
        if (!len) break;
        lzw_.insert(lzw_.end(), d + pos_, d + pos_ + len);
        pos_ += len;
    }
    const size_t npix = (size_t)im.w * im.h;
    idx_.resize(npix);
    if (!lzw_decode(lzw_.data(), lzw_.size(), m, idx_.data(), npix, err)) return false;
    for (size_t i = 0; i < npix; i++) if (idx_[i] >= im.tn) { err = "GIF pixel index past its colour table"; return false; }
    return true;
}

bool GifReader::open(const uint8_t *d, size_t n, std::string &err)
{
    if (!read_screen(d, n, err)) return false;
    size_t pos = first_block_;
    for (;;) {
        uint8_t kind;
        if (!walk_block(pos, kind, err)) return false;
        if (kind == 0x3B) break;
        if (kind == 0x2C) frames++;
    }
    if (!frames) { err = "GIF without frames"; return false; }
    pos_ = first_block_;
    canvas_.assign((size_t)width * height, 0u);
    saved_.clear();
    prev_disposal_ = 0;
    return true;
}

bool GifReader::next(uint32_t *canvas, int &delay, std::string &err)
{
    err.clear();
    const uint8_t *d = d_;
    int disposal = 0, tindex = -1;
    delay = 0;
    for (;;) {
        // open() has checked every length up to the trailer
        const uint8_t b = d[pos_++];
        if (b == 0x3B) { pos_--; return false; }
        if (b == 0x21) {
            const uint8_t label = d[pos_++];
            if (label == 0xF9) {
                const uint8_t f = d[pos_ + 1];
                disposal = (f >> 2) & 7; if (disposal > 3) disposal = 0;
                delay = (int)rd16(d + pos_ + 2);
                tindex = (f & 1) ? d[pos_ + 4] : -1;
            }
            skip_blocks(d, n_, pos_);
            continue;
        }
        // 0x2C
        Image im;
        if (!read_image(im, err)) return false;
        // the previous frame's disposal, then this frame's save for disposal 3
        if (prev_disposal_ == 2) {
            for (int r = 0; r < prev_h_; r++) memset(&canvas_[(size_t)(prev_y_ + r) * width + prev_x_], 0, (size_t)prev_w_ * 4);
        } else if (prev_disposal_ == 3 && !saved_.empty()) canvas_.swap(saved_);
        if (disposal == 3) saved_ = canvas_;
        for (int k = 0; k < im.h; k++) {
            uint32_t *dst = &canvas_[(size_t)(im.y + frame_row(k, im.h, im.interlaced)) * width + im.x];
            const uint8_t *src = &idx_[(size_t)k * im.w];
            for (int i = 0; i < im.w; i++) if (src[i] != tindex) dst[i] = im.table[src[i]];
        }
        prev_disposal_ = disposal; prev_x_ = im.x; prev_y_ = im.y; prev_w_ = im.w; prev_h_ = im.h;
        memcpy(canvas, canvas_.data(), canvas_.size() * 4);
        return true;
    }
}

bool GifReader::first_frame(const uint8_t *d, size_t n, std::vector<uint32_t> &canvas, std::string &err)
{
    if (!read_screen(d, n, err)) return false;
    size_t pos = first_block_;
    int tindex = -1;
    for (;;) {
        const size_t at = pos;
        uint8_t kind;
        if (!walk_block(pos, kind, err)) return false;
        if (kind == 0x3B) { err = "GIF without frames"; return false; }
        if (kind == 0x21 && d[at + 1] == 0xF9) tindex = (d[at + 3] & 1) ? d[at + 6] : -1;      // checked: its block holds 4 bytes or more
        if (kind == 0x2C) { pos_ = at + 1; break; }
    }
    frames = 1;
    Image im;
    if (!read_image(im, err)) return false;
    canvas.assign((size_t)width * height, 0u);
    for (int k = 0; k < im.h; k++) {
        uint32_t *dst = &canvas[(size_t)(im.y + frame_row(k, im.h, im.interlaced)) * width + im.x];
        const uint8_t *src = &idx_[(size_t)k * im.w];
        for (int i = 0; i < im.w; i++) dst[i] = src[i] == tindex ? im.table[src[i]] & 0x00FFFFFFu : im.table[src[i]];
    }
    return true;
}

} // namespace b200
