// tests/emul/gpuenc_stats_emul.cpp -- TEST INFRASTRUCTURE.  Checks, on the CPU, the two shortcuts the device encoder
// (caesium-clt_b200/csrc/jpeg_gpuenc.cu) takes over the plain block-parallel formulation that gpuenc_emul.cpp runs:
//   1. the statistics: inline symbols counted in the classify pass (gen_block with no group) plus one EOBn symbol per group
//      counted where k_ge_groups records it must equal the histogram of every symbol of every block;
//   2. the bit writer: every completed word of a block after its first is written with a plain store, not an OR; the words
//      must equal the ones written with OR only, whatever order the blocks are written in.
// Not linked into the product library.
#include <cstring>
#include <string>
#include <vector>
#include "../../caesium-clt_b200/csrc/jpeg_gpuenc_plan.h"

using namespace b200;

// 0: both hold; 1 / 2: the input does not parse / decode; 3: the histograms differ; 4: the bit buffers differ
extern "C" int emul_stats_check(const uint8_t *jpeg, size_t len, int progressive)
{
    std::string err;
    JpegReader rd(jpeg, len);
    if (!rd.read_header(err)) return 1;
    const JpegGeom &g = rd.geom();
    std::vector<int16_t> coefs((size_t)g.total_coefs);
    if (!rd.decode(coefs.data(), err)) return 2;
    jpeg_fill_dummy_blocks(g, coefs.data());
    GpuEncPlan plan;
    const int16_t *base = coefs.data();
    gpuenc_plan(g, progressive != 0, &base, 1, plan);
    const long long U = plan.total_units;
    std::vector<uint32_t> meta(U), gcount(U, 0), tsum(U), bitlen(U);
    std::vector<long long> evkey(U), prev_ev(U);
    std::vector<unsigned long long> bitoff(U);
    const size_t NH = plan.scans.size() * 4 * 256;
    std::vector<uint32_t> hist(NH, 0), hist_all(NH, 0);
    // classify + inline symbols, in the device's pass order
    for (const ge::Scan &s : plan.scans) for (int u = 0; u < s.nblocks; u++) {
        const ge::BlockRef b = ge::locate(s, u);
        const uint32_t m = ge::classify(s, b.blk);
        meta[s.unit_base + u] = m;
        evkey[s.unit_base + u] = ge::meta_event(m) ? s.unit_base + u : -1;
        uint32_t *h = hist.data() + (size_t)s.tab_base * 256;
        auto add = [h](int idx) { h[idx]++; };
        ge::HistSink<decltype(add)> sk(add);
        ge::gen_block(s, b, 0, sk);
    }
    { long long run = -1; for (long long i = 0; i < U; i++) { prev_ev[i] = run; if (evkey[i] > run) run = evkey[i]; } }
    { uint32_t run = 0; for (long long i = 0; i < U; i++) { tsum[i] = run; run += (uint32_t)ge::meta_tail(meta[i]); } }
    // groups + their EOBn symbols (AC table of the scan's one component)
    for (const ge::Scan &s : plan.scans) {
        if (s.mode != ge::MODE_AC_FIRST && s.mode != ge::MODE_AC_REFINE) continue;
        uint32_t *h = hist.data() + ((size_t)s.tab_base + 2 + s.tbl[0]) * 256;
        auto counted = [h](uint32_t c) { h[ge::eob_symbol(c)]++; };
        int prev = -1;
        for (int b = 0; b <= s.nblocks; b++) {
            if (b < s.nblocks && !ge::meta_event(meta[s.unit_base + b])) continue;
            ge::assign_groups(meta.data() + s.unit_base, tsum.data() + s.unit_base, s.nblocks, prev, b, gcount.data() + s.unit_base, counted);
            prev = b;
        }
    }
    // every symbol of every block, groups included
    for (const ge::Scan &s : plan.scans) for (int u = 0; u < s.nblocks; u++) {
        uint32_t *h = hist_all.data() + (size_t)s.tab_base * 256;
        auto add = [h](int idx) { h[idx]++; };
        ge::HistSink<decltype(add)> sk(add);
        ge::gen_block(s, ge::locate(s, u), gcount[s.unit_base + u], sk);
    }
    if (hist != hist_all) return 3;
    // tables, lengths, offsets; then the bit buffer written twice
    std::vector<ge::Table> tabs(plan.scans.size() * 4);
    std::vector<int> cs(257), oth(257); std::vector<long long> fr(257);
    for (size_t t = 0; t < tabs.size(); t++) ge::build_table(hist.data() + t * 256, tabs[t], cs.data(), oth.data(), fr.data());
    for (const ge::Scan &s : plan.scans) for (int u = 0; u < s.nblocks; u++) {
        ge::LenSink sk; sk.tabs = tabs.data() + s.tab_base;
        ge::gen_block(s, ge::locate(s, u), gcount[s.unit_base + u], sk);
        bitlen[s.unit_base + u] = (uint32_t)sk.bits;
    }
    { unsigned long long run = 0; for (long long i = 0; i < U; i++) { bitoff[i] = run; run += bitlen[i]; } }
    // the plain-store buffer is written twice, blocks in scan order and in reverse: a plain store into a word a neighbour also
    // writes loses that neighbour's bits in one of the two orders
    std::vector<uint32_t> w_or((size_t)plan.total_words, 0), w_fwd((size_t)plan.total_words, 0), w_rev((size_t)plan.total_words, 0);
    for (const ge::Scan &s : plan.scans) {
        const unsigned long long total = s.nblocks ? bitoff[s.unit_base + s.nblocks - 1] + bitlen[s.unit_base + s.nblocks - 1] - bitoff[s.unit_base] : 0;
        if ((long long)((total + 31) / 32) > s.word_cap) return 4;
        auto emit = [&](int u, uint32_t *w, bool plain) {
            const unsigned long long off = bitoff[s.unit_base + u] - bitoff[s.unit_base];
            auto orw = [w](long long i, uint32_t v) { w[i] |= v; };
            auto stw = [w, plain](long long i, uint32_t v) { if (plain) w[i] = v; else w[i] |= v; };
            ge::EmitSink<decltype(orw), decltype(stw)> sk(tabs.data() + s.tab_base, orw, stw, s.word_base, off);
            ge::gen_block(s, ge::locate(s, u), gcount[s.unit_base + u], sk);
            sk.finish();
        };
        for (int u = 0; u < s.nblocks; u++) { emit(u, w_or.data(), false); emit(u, w_fwd.data(), true); }
        for (int u = s.nblocks - 1; u >= 0; u--) emit(u, w_rev.data(), true);
    }
    return w_or == w_fwd && w_or == w_rev ? 0 : 4;
}
