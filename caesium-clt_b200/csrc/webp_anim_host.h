// webp_anim_host.h -- the animated WebP reader of the animated WebP leg, on the calling thread (webp_anim_host.cpp): RIFF / VP8X /
// ANIM / ANMF, and each frame's ALPH + 'VP8 ' or VP8L payload decoded with the still-image decoders (vp8_decode.h).
#pragma once
#include <cstddef>
#include <cstdint>
#include <string>
#include <vector>
#include "webp_anim_core.h"

namespace b200 {

// one decoded frame: its rectangle on the canvas, its ANMF flags (WA_DISPOSE_BG, WA_NO_BLEND) and duration in ms, whether its
// bitstream declares alpha (an ALPH chunk, or the VP8L header's alpha bit: libwebp's keyframe rule asks for that, not for the
// pixels), and its pixels as RGBA words (rect.w * rect.h, R in the low byte)
struct WebpAnimFrame {
    WaRect rect{0, 0, 0, 0};
    int flags = 0;
    uint32_t duration = 0;
    bool has_alpha = false;
    std::vector<uint32_t> rgba;
};

// Reads one animated WebP frame by frame.  open() walks and checks the whole container without decoding: a canvas side above
// WA_MAX_SIDE, a frame outside the canvas, a frame whose bitstream size differs from its ANMF size, a missing or misplaced chunk
// and a truncated chunk are all refused there, before any device work.  next() then decodes the frames in order; the reader
// holds one frame's pixels at a time.
class WebpAnimReader {
public:
    int width = 0, height = 0;
    int loop = 0;                   // ANIM loop count (0 = forever)
    uint8_t bg[4] = {0, 0, 0, 0};   // ANIM background colour bytes, as stored
    int frames = 0;

    bool open(const uint8_t *data, size_t n, std::string &err);
    // the next frame; false at the end (err empty) or on corrupt data (err says why)
    bool next(WebpAnimFrame &f, std::string &err);

private:
    struct Ref {
        WaRect rect;
        int flags;
        uint32_t duration;
        bool has_alpha;
        const uint8_t *alph, *vp8, *vp8l;
        size_t alph_len, vp8_len, vp8l_len;
    };
    bool frame_ref(const uint8_t *p, size_t n, Ref &r, std::string &err);
    std::vector<Ref> refs_;
    size_t next_ = 0;
};

// The composited canvas of every frame (rule of webp_anim_core.h) on the host, for the decoder hook and its tests: frames *
// width * height RGBA words in canvases, each frame's duration in durations.
bool webp_anim_decode_all(const uint8_t *data, size_t n, WebpAnimReader &rd, std::vector<uint32_t> &canvases, std::vector<uint32_t> &durations,
                          std::string &err);

} // namespace b200
