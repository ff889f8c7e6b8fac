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

    // Instead of open() / next(): frame 0 alone as the image crate decodes a GIF for a conversion -- width * height words, R in the
    // low byte; inside the frame's rectangle every pixel is its palette colour, with alpha 0 for the transparent index and 255
    // otherwise; outside it 0x00000000.  The blocks are checked up to the end of frame 0's image data only, so damage after it is
    // never seen.  Refusals as open(): `unsupported` for a frame past the logical screen, otherwise the file is corrupt.
    bool first_frame(const uint8_t *data, size_t n, std::vector<uint32_t> &canvas, std::string &err);

private:
    struct Image {                          // one frame's descriptor and colour table; its indices are in idx_
        int x, y, w, h, tn;
        bool interlaced;
        const uint32_t *table;
        uint32_t lct[256];
    };
    // the header and global colour table
    bool read_screen(const uint8_t *data, size_t n, std::string &err);
    // the block at pos checked against the input and skipped; kind = its introducer (0x21, 0x2C or the trailer 0x3B)
    bool walk_block(size_t &pos, uint8_t &kind, std::string &err);
    // the image at pos_ (after its 0x2C, its block checked by walk_block): descriptor, colour table and indices in stream order
    bool read_image(Image &im, std::string &err);

    const uint8_t *d_ = nullptr;
    size_t n_ = 0, pos_ = 0, first_block_ = 0;
    uint32_t gct_[256] = {};
    int gct_n_ = 0;
    std::vector<uint32_t> canvas_, saved_;
    std::vector<uint8_t> idx_, lzw_;
    int prev_disposal_ = 0, prev_x_ = 0, prev_y_ = 0, prev_w_ = 0, prev_h_ = 0;
};

} // namespace b200
