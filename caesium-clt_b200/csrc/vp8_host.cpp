// vp8_host.cpp -- see vp8_host.h.  Entropy coding of the WebP leg stays on the host (north_star: "VP8 bool-coder on the host").
#include "vp8_host.h"
#include <cmath>
#include <cstring>
#include "vp8_tables.h"
#include "vp8_tokens_core.h"
#include "vp8_bpred_core.h"

namespace b200 {

int vp8_qindex(int quality)
{   // libwebp: c = quality / 100; linearised, cube root, scaled to the 0..127 index range (segment alpha 0)
    const double c = quality / 100.0, lin = c < 0.75 ? c * (2.0 / 3.0) : 2.0 * c - 1.0;
    const int q = (int)(127.0 * (1.0 - std::pow(lin, 1.0 / 3.0)));
    return q < 0 ? 0 : q > 127 ? 127 : q;
}

int vp8_filter_level(int qindex) { const int l = qindex / 2; return l > 63 ? 63 : l; }

void vp8_quant_factors(int q, int f[6])
{
    f[0] = VP8_DC_Q[q]; f[1] = VP8_AC_Q[q];
    f[2] = 2 * VP8_DC_Q[q]; f[3] = VP8_AC_Q[q] * 155 / 100; if (f[3] < 8) f[3] = 8;
    f[4] = VP8_DC_Q[q > 117 ? 117 : q]; f[5] = VP8_AC_Q[q];
}

namespace {

// RFC 6386 section 7.3 arithmetic encoder: 8-bit probabilities, range kept in [128, 255], carries propagated into the bytes
// already written.
class BoolWriter {
public:
    // `low_` is the RFC's 32-bit `bottom` kept in 64 bits so that a whole renormalisation (1..7 bit positions) is one shift: the byte that
    // completes sits above bit 24 + k with its carry on top (k = positions shifted past the byte boundary), exactly where the bit-by-bit
    // loop of the RFC would have found them.  Output goes through a raw pointer into a buffer sized up front (reserve()): one decision
    // yields at most 8 bits.
    explicit BoolWriter(size_t decisions = 4096) { buf_.resize(decisions + 16); p_ = buf_.data(); }
    void reserve_more(size_t decisions) { const size_t used = size(); if (used + decisions + 16 > buf_.size()) { buf_.resize(used + decisions + 16 + buf_.size() / 2); p_ = buf_.data() + used; } }
    size_t size() const { return (size_t)(p_ - buf_.data()); }
    const uint8_t *data() const { return buf_.data(); }
    inline void put(int bit, int prob)
    {
        const uint32_t split = 1 + (((range_ - 1) * (uint32_t)prob) >> 8);
        const uint32_t m = 0u - (uint32_t)(bit & 1);                  // the decision is data: no branch on it
        low_ += split & m;
        range_ = split ^ ((split ^ (range_ - split)) & m);
        const int shift = __builtin_clz(range_) - 24;                  // 0 when the range is still >= 128
        range_ <<= shift; low_ <<= shift; count_ -= shift;
        if (count_ <= 0) {
            const int k = -count_;
            const uint32_t v = (uint32_t)(low_ >> (24 + k));
            if (v & 0x100u) carry();
            *p_++ = (uint8_t)v;
            low_ &= (1ull << (24 + k)) - 1ull;
            count_ += 8;
        }
    }
    void literal(int value, int nbits) { reserve_more((size_t)nbits); for (int i = nbits - 1; i >= 0; i--) put((value >> i) & 1, 128); }
    void finish()
    {
        reserve_more(8);
        int c = count_; uint32_t v = (uint32_t)low_;
        if (low_ & (1ull << (32 - c))) carry();
        v <<= c & 7;
        for (c >>= 3; c > 0; c--) v <<= 8;
        for (int i = 0; i < 4; i++, v <<= 8) *p_++ = (uint8_t)(v >> 24);
    }
private:
    std::vector<uint8_t> buf_; uint8_t *p_;
    uint32_t range_ = 255; uint64_t low_ = 0; int count_ = 24;
    void carry() { uint8_t *q = p_; while (q > buf_.data() && q[-1] == 0xFF) *--q = 0; if (q > buf_.data()) q[-1]++; }
};

using vt::kNumProbs;

// host side of the token pass (the device runs k_vp8_tokens instead): every decision is tallied and appended to a list; the writer
// replays the list against the probabilities chosen from the tallies
struct TokenRecorder {
    uint32_t (*count)[2]; std::vector<uint16_t> &list; uint16_t *q = nullptr;
    // room for one macroblock's worth of decisions is made before the macroblock is walked
    void begin_mb() { const size_t used = q ? (size_t)(q - list.data()) : 0; if (used + vt::kMaxDecisionsPerMb > list.size()) list.resize(list.size() * 2 + (size_t)vt::kMaxDecisionsPerMb * 64); q = list.data() + used; }
    size_t size() const { return q ? (size_t)(q - list.data()) : 0; }
    void node(int s, bool bit) { count[s][bit ? 1 : 0]++; *q++ = vt::rec_node(s, bit); }
    void fixed(bool bit, int prob) { *q++ = vt::rec_fixed(bit, prob); }
};

// the frame's decisions from its levels: masks of every macroblock first (a skipped one counts as empty), then one independent walk
// per macroblock -- the same two steps the device takes (k_vp8_mbmask, k_vp8_tokens)
void host_tokens(int mbw, int mbh, bool use_skip, const int16_t *levels, const uint8_t *modes, uint32_t *cnt /*[kNumProbs][2]*/, std::vector<uint16_t> &tokens)
{
    const size_t nmb = (size_t)mbw * mbh;
    std::vector<uint32_t> mask(nmb);
    std::vector<uint8_t> y2top(nmb), y2left(nmb);
    for (size_t mb = 0; mb < nmb; mb++) mask[mb] = (use_skip && modes[4 * mb + 2]) ? 0u : vt::mb_mask(levels + mb * 400, modes[4 * mb] == 4);
    for (int x = 0; x < mbw; x++) vt::y2_carry_col(mask.data(), modes, mbw, mbh, x, y2top.data());
    for (int y = 0; y < mbh; y++) vt::y2_carry_row(mask.data(), modes, mbw, y, y2left.data());
    tokens.resize(nmb * 128 + vt::kMaxDecisionsPerMb);
    TokenRecorder tc{reinterpret_cast<uint32_t (*)[2]>(cnt), tokens};
    for (int my = 0; my < mbh; my++)
        for (int mx = 0; mx < mbw; mx++) {
            const size_t mb = (size_t)my * mbw + mx;
            if (use_skip && modes[4 * mb + 2]) continue;
            tc.begin_mb();
            vt::walk_mb(tc, levels + mb * 400, vt::with_y2(my ? mask[mb - mbw] : 0u, y2top[mb]), vt::with_y2(mx ? mask[mb - 1] : 0u, y2left[mb]), modes[4 * mb] == 4);
        }
    tokens.resize(tc.size());
}

// price of one decision coded with probability-of-zero p/256, in 1/256 bit
inline int bit_cost(int p) { return p <= 0 ? 1 << 20 : (int)(-std::log2(p / 256.0) * 256.0 + 0.5); }

void put_le(std::vector<uint8_t> &o, uint32_t v, int nbytes) { for (int i = 0; i < nbytes; i++) o.push_back((uint8_t)(v >> (8 * i))); }

} // namespace

bool vp8_frame_uses_skip(int width, int height, const uint8_t *modes)
{
    const int nmb = ((width + 15) >> 4) * ((height + 15) >> 4);
    for (int i = 0; i < nmb; i++) if (modes[4 * i + 2]) return true;
    return false;
}

bool vp8_write_file(int width, int height, int qindex, const int16_t *levels, const uint8_t *modes, std::vector<uint8_t> &out, const uint8_t *bmodes)
{
    if (width < 1 || height < 1 || width > 16383 || height > 16383) return false;
    const int mbw = (width + 15) >> 4, mbh = (height + 15) >> 4;
    for (int i = 0; i < mbw * mbh; i++) {                            // modes index the sub-block mode probabilities: refuse any out of range
        if (modes[4 * i] > 4 || modes[4 * i + 1] > 3) return false;
        if (modes[4 * i] == 4) { if (!bmodes) return false; for (int k = 0; k < 16; k++) if (bmodes[16 * i + k] > 9) return false; }
    }
    std::vector<uint32_t> cnt((size_t)kNumProbs * 2, 0);
    std::vector<uint16_t> tokens;
    host_tokens(mbw, mbh, vp8_frame_uses_skip(width, height, modes), levels, modes, cnt.data(), tokens);
    return vp8_write_file_tokens(width, height, qindex, modes, cnt.data(), tokens.data(), tokens.size(), out, bmodes);
}

bool vp8_write_file_tokens(int width, int height, int qindex, const uint8_t *modes, const uint32_t *cnt, const uint16_t *tokens, size_t ntokens, std::vector<uint8_t> &out,
                           const uint8_t *bmodes)
{
    const int mbw = (width + 15) >> 4, mbh = (height + 15) >> 4, nmb = mbw * mbh;
    if (width < 1 || height < 1 || width > 16383 || height > 16383) return false;
    int nskip = 0, nbpred = 0;
    for (int i = 0; i < nmb; i++) { nskip += modes[4 * i + 2]; nbpred += modes[4 * i] == 4; }
    if (nbpred && !bmodes) return false;
    const bool use_skip = nskip > 0;
    int skip_p = (int)(((long long)(nmb - nskip) * 255) / nmb); if (skip_p < 1) skip_p = 1; if (skip_p > 255) skip_p = 255;
    // ---- token probabilities (13.4): from the tallies of this frame's tree decisions, replace a default wherever the frame's
    //      own estimate (libwebp's 255 - ones * 255 / total) saves more than the flag + 8-bit update costs
    std::vector<uint8_t> probs(VP8_COEF_PROBS, VP8_COEF_PROBS + kNumProbs), updated(kNumProbs, 0);
    for (int i = 0; i < kNumProbs; i++) {
        const uint64_t c0 = cnt[2 * i], c1 = cnt[2 * i + 1], total = c0 + c1;
        if (!total) continue;
        const int oldp = probs[i], u = VP8_COEF_UPDATE_PROBS[i];
        int newp = 255 - (int)(c1 * 255 / total); if (newp < 1) newp = 1;
        const uint64_t keep = c0 * bit_cost(oldp) + c1 * bit_cost(256 - oldp) + bit_cost(u);
        const uint64_t change = c0 * bit_cost(newp) + c1 * bit_cost(256 - newp) + bit_cost(256 - u) + 8 * 256;
        if (newp != oldp && change < keep) { probs[i] = (uint8_t)newp; updated[i] = 1; }
    }
    // ---- first partition: frame header (RFC 6386 9.2-9.11, 19.2) and the per-macroblock modes (19.3)
    // decisions: a 16x16 macroblock takes at most 8, a B_PRED one at most 3 + 16 * 7 (sub-block modes HD and HU are 7 deep) + 3
    BoolWriter hd((size_t)kNumProbs * 9 + (size_t)nmb * 8 + (size_t)nbpred * 120 + 256);
    hd.literal(0, 1);                   // color_space
    hd.literal(0, 1);                   // clamping_type
    hd.literal(0, 1);                   // segmentation_enabled
    hd.literal(1, 1);                   // filter_type: simple (luma edges only)
    hd.literal(vp8_filter_level(qindex), 6);   // loop_filter_level: a decoder-side post-filter; prediction in K8 uses unfiltered samples, as the format defines
    hd.literal(0, 3);                   // sharpness_level
    hd.literal(0, 1);                   // loop_filter_adj_enable
    hd.literal(0, 2);                   // log2_nbr_of_dct_partitions
    hd.literal(qindex, 7);              // y_ac_qi
    hd.literal(0, 5);                   // five delta-present flags, all clear
    hd.literal(0, 1);                   // refresh_entropy_probs
    for (int i = 0; i < kNumProbs; i++) { hd.put(updated[i], VP8_COEF_UPDATE_PROBS[i]); if (updated[i]) hd.literal(probs[i], 8); }
    hd.literal(use_skip, 1);            // mb_no_coeff_skip
    if (use_skip) hd.literal(skip_p, 8);
    // sub-block mode contexts (11.3): the modes above / to the left, a 16x16 macroblock's luma mode standing for all its sub-blocks,
    // DC beyond the frame's edges
    std::vector<uint8_t> top_modes((size_t)mbw * 4, 0);
    uint8_t left_modes[4] = {0, 0, 0, 0};
    for (int i = 0; i < nmb; i++) {
        const int ym = modes[4 * i], uvm = modes[4 * i + 1];
        uint8_t *tm = &top_modes[(size_t)(i % mbw) * 4];
        if (i % mbw == 0) memset(left_modes, 0, 4);
        if (use_skip) hd.put(modes[4 * i + 2], skip_p);
        if (ym == 4) {
            hd.put(0, 145);                                                             // B_PRED
            const uint8_t *bm = bmodes + (size_t)i * 16;
            for (int k = 0; k < 16; k++) {
                uint8_t p[8], b[8];
                const int n = vp8bp_bmode_bits(tm[k & 3], left_modes[k >> 2], bm[k], p, b);
                for (int j = 0; j < n; j++) hd.put(b[j], p[j]);
                tm[k & 3] = left_modes[k >> 2] = bm[k];
            }
        } else {
            hd.put(1, 145);                                                             // a 16x16 mode, not B_PRED
            const bool tm_or_h = ym == 1 || ym == 3;
            hd.put(tm_or_h, 156);
            if (tm_or_h) hd.put(ym == 1, 128); else hd.put(ym == 2, 163);
            memset(tm, ym, 4); memset(left_modes, ym, 4);
        }
        hd.put(uvm != 0, 142);
        if (uvm != 0) { hd.put(uvm != 2, 114); if (uvm != 2) hd.put(uvm != 3, 183); }
    }
    hd.finish();
    if (hd.size() >= (1u << 19)) return false;
    // ---- token partition, coded with the table chosen above
    BoolWriter tk(ntokens + 64);
    for (size_t k = 0; k < ntokens; k++) { const uint16_t t = tokens[k]; tk.put(t & 1, (t & 0x8000u) ? (t >> 1) & 0xFF : probs[t >> 1]); }
    tk.finish();
    // ---- RIFF container (WebP simple lossy format)
    const size_t vp8_size = 10 + hd.size() + tk.size(), riff_payload = 4 + 8 + vp8_size + (vp8_size & 1);
    out.clear(); out.reserve(8 + riff_payload);
    out.insert(out.end(), {'R', 'I', 'F', 'F'}); put_le(out, (uint32_t)riff_payload, 4);
    out.insert(out.end(), {'W', 'E', 'B', 'P', 'V', 'P', '8', ' '}); put_le(out, (uint32_t)vp8_size, 4);
    put_le(out, (1u << 4) | ((uint32_t)hd.size() << 5), 3);      // key frame (bit 0 clear), version 0, show_frame, first partition size
    out.insert(out.end(), {0x9d, 0x01, 0x2a}); put_le(out, (uint32_t)width, 2); put_le(out, (uint32_t)height, 2);
    out.insert(out.end(), hd.data(), hd.data() + hd.size());
    out.insert(out.end(), tk.data(), tk.data() + tk.size());
    if (vp8_size & 1) out.push_back(0);
    return true;
}

} // namespace b200
