// gif_host.h -- the GIF decoder of the GIF leg, on the calling thread (gif_host.cpp): container, LZW and compositing to one RGBA
// canvas per frame.
#pragma once
#include <cstddef>
#include <cstdint>
#include <string>
#include <vector>

namespace b200 {

// Reads one GIF frame by frame.  open() walks the whole block structure once without decoding (so a truncated file is refused
// before any device work, and the loop count is known before the first frame is written); next() then decodes and composites the
// frames in order.  Comment, plain-text and application extensions other than NETSCAPE2.0 are skipped.
//
// Compositing follows gif-dispose: the canvas starts fully transparent, a transparent index leaves the canvas pixel as it is,
// disposal 2 clears the frame's rectangle to transparent and disposal 3 restores the canvas from before the frame, both before the
// next frame is drawn.  A canvas pixel is 0x00000000 (clear) or opaque, R in the low byte.  The reader holds the current canvas
// and, for disposal 3, the one before it.
class GifReader {
public:
    int width = 0, height = 0;
    int loop = -1;              // NETSCAPE2.0 loop count (0 = forever), -1 when the file has none
    int frames = 0;
    bool unsupported = false;   // after a refusal: a frame extends past the logical screen (else the file is corrupt)

    bool open(const uint8_t *data, size_t n, std::string &err);
    // the displayed canvas of the next frame (width * height words) and its delay in 1/100 s; false at the end (err empty) or on
    // corrupt data (err says why)
    bool next(uint32_t *canvas, int &delay, std::string &err);

private:
    const uint8_t *d_ = nullptr;
    size_t n_ = 0, pos_ = 0, first_block_ = 0;
    uint32_t gct_[256] = {};
    int gct_n_ = 0;
    std::vector<uint32_t> canvas_, saved_;
    std::vector<uint8_t> idx_, lzw_;
    int prev_disposal_ = 0, prev_x_ = 0, prev_y_ = 0, prev_w_ = 0, prev_h_ = 0;
};

} // namespace b200
