// webp_anim_host.cpp -- see webp_anim_host.h.
#include <cstring>
#include "webp_anim_host.h"
#include "vp8_decode.h"

namespace b200 {

namespace {
inline uint32_t rd24(const uint8_t *p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16); }
inline uint32_t rd32(const uint8_t *p) { return rd24(p) | ((uint32_t)p[3] << 24); }
} // namespace

// the sub-chunks of one ANMF payload (after its 16-byte frame header): an optional ALPH, then 'VP8 ' or VP8L; unknown chunks after
// the image are skipped
bool WebpAnimReader::frame_ref(const uint8_t *p, size_t n, Ref &r, std::string &err)
{
    r.alph = r.vp8 = r.vp8l = nullptr;
    r.alph_len = r.vp8_len = r.vp8l_len = 0;
    size_t i = 0;
    while (i + 8 <= n) {
        const uint8_t *tag = p + i;
        const size_t sz = rd32(p + i + 4);
        if (sz > n - i - 8) { err = "truncated WebP chunk"; return false; }
        const bool image = r.vp8 || r.vp8l;
        if (!image && !memcmp(tag, "ALPH", 4)) {
            if (r.alph) { err = "animated WebP frame with two ALPH chunks"; return false; }
            r.alph = p + i + 8; r.alph_len = sz;
        } else if (!image && !memcmp(tag, "VP8 ", 4)) { r.vp8 = p + i + 8; r.vp8_len = sz; }
        else if (!image && !memcmp(tag, "VP8L", 4)) { r.vp8l = p + i + 8; r.vp8l_len = sz; }
        else if (!image) { err = "animated WebP frame without an image chunk"; return false; }
        i += 8 + sz + (sz & 1);
    }
    if (!r.vp8 && !r.vp8l) { err = "animated WebP frame without an image chunk"; return false; }
    if (r.vp8l && r.alph) { err = "animated WebP frame with an ALPH chunk before VP8L"; return false; }
    int bw, bh;
    if (r.vp8) {
        const uint8_t *f = r.vp8;
        if (r.vp8_len < 10 || f[3] != 0x9d || f[4] != 0x01 || f[5] != 0x2a) { err = "bad VP8 frame header in animated WebP"; return false; }
        bw = (f[6] | (f[7] << 8)) & 0x3fff; bh = (f[8] | (f[9] << 8)) & 0x3fff;
        r.has_alpha = r.alph != nullptr;
    } else {
        const uint8_t *f = r.vp8l;
        if (r.vp8l_len < 5 || f[0] != 0x2f) { err = "bad VP8L frame header in animated WebP"; return false; }
        const uint32_t v = rd32(f + 1);
        bw = 1 + (int)(v & 0x3fff); bh = 1 + (int)((v >> 14) & 0x3fff);
        r.has_alpha = (v >> 28) & 1;
    }
    if (bw != r.rect.w || bh != r.rect.h) { err = "animated WebP frame bitstream size differs from its ANMF size"; return false; }
    return true;
}

bool WebpAnimReader::open(const uint8_t *d, size_t n, std::string &err)
{
    refs_.clear(); next_ = 0; frames = 0;
    if (n < 12 || memcmp(d, "RIFF", 4) || memcmp(d + 8, "WEBP", 4)) { err = "not a WebP file"; return false; }
    const size_t riff = rd32(d + 4);
    if (riff < 4 || riff > n - 8) { err = "truncated WebP file"; return false; }
    const size_t end = 8 + riff;
    size_t i = 12;
    bool vp8x = false, anim = false;
    while (i + 8 <= end) {
        const uint8_t *tag = d + i;
        const size_t sz = rd32(d + i + 4);
        if (sz > end - i - 8) { err = "truncated WebP chunk"; return false; }
        const uint8_t *p = d + i + 8;
        if (!memcmp(tag, "VP8X", 4)) {
            if (i != 12 || sz < 10) { err = "bad VP8X chunk in animated WebP"; return false; }
            width = 1 + (int)rd24(p + 4); height = 1 + (int)rd24(p + 7);
            if (width > WA_MAX_SIDE || height > WA_MAX_SIDE) { err = "animated WebP canvas side over 16383"; return false; }
            vp8x = true;
        } else if (!memcmp(tag, "ANIM", 4)) {
            if (!vp8x || anim || sz < 6) { err = "bad ANIM chunk in animated WebP"; return false; }
            memcpy(bg, p, 4); loop = p[4] | (p[5] << 8);
            anim = true;
        } else if (!memcmp(tag, "ANMF", 4)) {
            if (!anim || sz < 16) { err = "bad ANMF chunk in animated WebP"; return false; }
            Ref r;
            r.rect.x = 2 * (int)rd24(p); r.rect.y = 2 * (int)rd24(p + 3);
            r.rect.w = 1 + (int)rd24(p + 6); r.rect.h = 1 + (int)rd24(p + 9);
            r.duration = rd24(p + 12);
            r.flags = p[15] & (WA_DISPOSE_BG | WA_NO_BLEND);
            if (r.rect.x + r.rect.w > width || r.rect.y + r.rect.h > height) { err = "animated WebP frame outside the canvas"; return false; }
            if (!frame_ref(p + 16, sz - 16, r, err)) return false;
            refs_.push_back(r);
        } else if (!memcmp(tag, "VP8 ", 4) || !memcmp(tag, "VP8L", 4) || !memcmp(tag, "ALPH", 4)) {
            err = "image chunk outside ANMF in animated WebP"; return false;
        }
        i += 8 + sz + (sz & 1);
    }
    if (!anim || refs_.empty()) { err = "animated WebP without ANIM or ANMF chunks"; return false; }
    frames = (int)refs_.size();
    return true;
}

bool WebpAnimReader::next(WebpAnimFrame &f, std::string &err)
{
    err.clear();
    if (next_ >= refs_.size()) return false;
    const Ref &r = refs_[next_++];
    WebpInfo info;
    info.lossless = r.vp8l != nullptr;
    info.has_alpha = r.alph != nullptr;
    std::vector<uint8_t> rgb, alpha;
    if (webp_decode_chunks(r.vp8, r.vp8_len, r.alph, r.alph_len, r.vp8l, r.vp8l_len, info, rgb, err, &alpha)) {
        if (err.empty()) err = "corrupt animated WebP frame";
        return false;
    }
    f.rect = r.rect; f.flags = r.flags; f.duration = r.duration; f.has_alpha = r.has_alpha;
    const size_t np = (size_t)r.rect.w * r.rect.h;
    f.rgba.resize(np);
    for (size_t k = 0; k < np; k++)
        f.rgba[k] = rgb[k] | (uint32_t)rgb[np + k] << 8 | (uint32_t)rgb[2 * np + k] << 16 | (uint32_t)(alpha.empty() ? 255u : alpha[k]) << 24;
    return true;
}

bool webp_anim_decode_all(const uint8_t *data, size_t n, WebpAnimReader &rd, std::vector<uint32_t> &canvases, std::vector<uint32_t> &durations, std::string &err)
{
    if (!rd.open(data, n, err)) return false;
    const int W = rd.width, H = rd.height;
    const size_t np = (size_t)W * H;
    std::vector<uint32_t> canvas(np, 0u);
    canvases.clear(); durations.clear();
    canvases.reserve(np * rd.frames);
    WebpAnimFrame f;
    WaRect prev{0, 0, 0, 0};
    int prev_flags = 0, prev_key = 0;
    for (int k = 0; rd.next(f, err); k++) {
        const WaStep s = webp_anim_step(k, f.rect, f.has_alpha, f.flags, prev, prev_flags, prev_key, W, H);
        for (int y = 0; y < H; y++)
            for (int x = 0; x < W; x++) {
                const size_t at = (size_t)y * W + x;
                const uint32_t src = wa_in_rect(f.rect, x, y) ? f.rgba[(size_t)(y - f.rect.y) * f.rect.w + (x - f.rect.x)] : 0u;
                canvas[at] = webp_anim_pixel(&s, x, y, canvas[at], src);
            }
        canvases.insert(canvases.end(), canvas.begin(), canvas.end());
        durations.push_back(f.duration);
        prev = f.rect; prev_flags = f.flags; prev_key = s.keyframe;
    }
    return err.empty();
}

} // namespace b200
