// jpeg_host.h -- host half of the JPEG path: marker parsing, Huffman decode to zigzag coefficient
// buffers, and Huffman encode from them (entropy coding stays on the host per BASELINE.json's north_star;
// it is what mozjpeg's jdhuff.c/jdphuff.c/jchuff.c/jcphuff.c do below caesium::compress_in_memory,
// caesium-clt's src/compressor.rs:305).  Written for throughput: 64-bit bit buffers, lookahead tables,
// token streams shared by the statistics and emission passes.
#pragma once
#include <cstdint>
#include <cstddef>
#include <string>
#include <vector>

namespace b200 {

struct JpegGeom {
    int width = 0, height = 0, ncomp = 0;
    bool progressive = false;
    int cid[4] = {1, 2, 3, 4};
    int hs[4] = {1, 1, 1, 1}, vs[4] = {1, 1, 1, 1}, tq[4] = {0, 1, 1, 1};
    int hmax = 1, vmax = 1, mcux = 0, mcuy = 0;
    int bw[4] = {0}, bh[4] = {0};     // allocated blocks (whole MCUs)
    int rbw[4] = {0}, rbh[4] = {0};   // real blocks
    int cw[4] = {0}, ch[4] = {0};     // component sample dims
    int64_t comp_offset[4] = {0};     // int16 units
    int64_t total_coefs = 0;
    uint16_t qt[4][64] = {{0}};       // per QUANT SLOT, zigzag order
    bool qt_present[4] = {false, false, false, false};
    void finalize();                  // derive everything from width/height/ncomp/hs/vs
    int64_t blocks(int c) const { return (int64_t)bw[c] * bh[c]; }
};

struct JpegMeta {
    bool jfif = false;
    uint8_t jfif_body[9] = {1, 1, 0, 0, 1, 0, 1, 0, 0};  // version, units, densities, thumbnail dims
    std::vector<uint8_t> app_markers;   // APPn/COM verbatim (FF xx len ...), excluding JFIF APP0, Adobe APP14, ICC APP2
    std::vector<uint8_t> icc_markers;   // APP2 ICC_PROFILE chunks verbatim
    bool adobe = false; int adobe_transform = 1;   // APP14 "Adobe": transform 0 = components are RGB (or CMYK), 1 = YCbCr
};

// Stateful reader: read_header() walks the markers up to the first SOS (tables + frame), decode() entropy-decodes
// every scan into a caller-supplied buffer (so the buffer can be pinned memory).
class JpegReader {
public:
    JpegReader(const uint8_t *data, size_t len) : d_(data), n_(len) {}
    bool read_header(std::string &err);
    bool decode(int16_t *coefs, std::string &err);   // coefs: geom().total_coefs int16, fully overwritten
    const JpegGeom &geom() const { return g_; }
    const JpegMeta &meta() const { return m_; }
    // After read_header(): is this file decodable by the device entropy decoder?  (baseline process, exactly one scan
    // that carries every component, no restart interval.)  Fills the scan's table selectors and the byte range of its
    // entropy-coded segment; on true, the reader is positioned after the scan so later markers are still parsed by
    // finish_after_device_decode().
    // verified = the host walked the entropy-coded segment (stuffed zeros counted, no marker inside, EOI right behind it).
    // scan_on_device: skip that walk -- the segment is taken to end at the file's last EOI and the device decoder counts the stuffed
    // bytes and looks for markers itself while it un-stuffs (a marker inside sends the image to the host decoder).
    struct DeviceScan { int ns; int ci[4], td[4], ta[4]; size_t ecs_begin, ecs_end, stuffed; bool verified; };
    bool device_decodable(DeviceScan &ds, bool scan_on_device = false);
    const uint8_t *dht_bits(int kind, int id) const { return kind ? ac_[id].bits : dc_[id].bits; }
    const uint8_t *dht_vals(int kind, int id) const { return kind ? ac_[id].vals : dc_[id].vals; }
    bool dht_present(int kind, int id) const { return kind ? ac_[id].present : dc_[id].present; }
    const uint8_t *data() const { return d_; }
    struct Huff {
        uint8_t bits[17]; uint8_t vals[256]; bool present = false;
        // decode acceleration
        uint16_t look[1 << 10];      // (len << 8) | symbol for codes <= 10 bits, 0 otherwise
        int32_t maxcode[18]; int32_t valoff[18];
        void build();
    };
private:
    bool parse_segment(unsigned marker, const uint8_t *seg, size_t sl, std::string &err);
    bool decode_scan(const uint8_t *seg, size_t sl, const uint8_t *ecs, const uint8_t **next, int16_t *coefs, std::string &err);
    const uint8_t *d_; size_t n_; size_t pos_ = 0;
    JpegGeom g_; JpegMeta m_;
    Huff dc_[4], ac_[4];
    int restart_interval_ = 0;
    bool have_sof_ = false;
    bool zeroed_ = false;
};

struct JpegWriteOptions {
    bool progressive = true;
    bool keep_metadata = false;
    bool preserve_icc = true;
    bool copy_jfif = false;      // lossless transcode keeps the source's JFIF density (jpeg_copy_critical_parameters)
};

// AC = 0 / DC = previous-block rule for the blocks an MCU has beyond the component's real extent
// (jccoefct.c compress_first_pass, jctrans.c compress_output)
void jpeg_fill_dummy_blocks(const JpegGeom &g, int16_t *coefs);

// Entropy-code `coefs` (geometry g, zigzag order) into a complete JFIF file.
bool jpeg_write(const JpegGeom &g, const int16_t *coefs, const JpegWriteOptions &opt, const JpegMeta *meta,
                std::vector<uint8_t> &out, std::string &err);

// The scan script both encoders (host writer, GPU entropy encoder) follow: sequential = one interleaved scan;
// progressive = the 8-scan script mozjpeg's optimize_scans settled on for samples/j0.JPG (SURVEY.md KAT-3).
struct ScanDef { int ns, ci[3], Ss, Se, Ah, Al; };
int jpeg_scan_script(const JpegGeom &g, bool progressive, ScanDef out[16]);
// which of the four tables [kind 0 DC / 1 AC][tbl 0 luma / 1 chroma] a scan defines (emitted as DHT before its SOS)
void jpeg_scan_tables_needed(const JpegGeom &g, bool progressive, const ScanDef &s, bool need[2][2]);

// A scan whose entropy-coded segment was produced elsewhere (the GPU encoder): DHT payloads + stuffed bytes.
struct EncodedScan {
    ScanDef def;
    bool has_tab[2][2];
    uint8_t bits[2][2][17]; uint8_t vals[2][2][256]; int nvals[2][2];
    const uint8_t *data; size_t len;
};
// Same file layout as jpeg_write (SOI, JFIF, carried markers, DQT, SOF, then per scan DHT* + SOS + data, EOI).
bool jpeg_assemble(const JpegGeom &g, const JpegWriteOptions &opt, const JpegMeta *meta, const EncodedScan *scans, int nscans,
                   std::vector<uint8_t> &out, std::string &err);

// length of the file jpeg_assemble would write (scan data is not read)
size_t jpeg_assembled_size(const JpegGeom &g, const JpegWriteOptions &opt, const JpegMeta *meta, const EncodedScan *scans, int nscans);

bool jpeg_assemble_malloc(const JpegGeom &g, const JpegWriteOptions &opt, const JpegMeta *meta, const EncodedScan *scans, int nscans,
                          uint8_t **out, size_t *out_len, std::string &err);

// mozjpeg base table idx 3 scaled by jpeg_set_quality(q, force_baseline = FALSE); natural order
void jpeg_quant_table(int quality, int which, uint16_t out_natural[64]);
extern const uint8_t kZigzag[64];   // zigzag index -> natural position

// geometry the encoder side of compress_in_memory produces for an input + CSParameters.jpeg.*
bool jpeg_output_geom(const JpegGeom &in, int quality, int subsampling, JpegGeom &out, std::string &err);

} // namespace b200
