// tests/emul/gpuenc_blockmajor_emul.cpp -- TEST INFRASTRUCTURE.  Runs the block-major view of the device encoder's classify,
// length and emit passes (caesium-clt_b200/csrc/jpeg_gpuenc.cu) on the CPU and compares it with the scan-major formulation:
//   - every block of every component, through the visit records of jpeg_gpuenc_plan.h, reaches each unit of each scan exactly
//     once (enc_unit_of) with the block ge::locate gives, and the DC predecessor enc_dc_prev names is ge::locate's;
//   - symbols counted into, and code words looked up in, the on-chip table layout (ENC_TAB_ENTRIES, enc_entry_table, KindTabs)
//     give the scan-major histograms, per-unit bit lengths and bit buffer.
// Not linked into the product library.
#include <cstring>
#include <string>
#include <vector>
#include "../../caesium-clt_b200/csrc/jpeg_gpuenc_plan.h"

using namespace b200;

namespace {
struct TabHist {                // k_geb_classify's counters, without the atomics
    ge::KindTabs<uint32_t> h;
    void sym(int kind, int, int symbol, int, unsigned) { (kind ? h.ac : h.dc)[symbol]++; }
    void raw64(int, unsigned long long) {}
};
template <class T>
ge::KindTabs<T> kind_tabs(T *tab, const EncVisit &v) { return ge::KindTabs<T>{tab + ENC_DC_ENTRY, tab + v.ac_entry}; }
}

// 0: all agree; 1 / 2: the input does not parse / decode; 3: histograms; 4: bit buffers; 5: unit -> block; 6: DC predecessor;
// 7: classification; 8: bit lengths; 9: a unit not reached exactly once; 10: the script does not fit the on-chip slots
extern "C" int emul_blockmajor_check(const uint8_t *jpeg, size_t len, int progressive)
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
    if (!plan.on_chip) return 10;
    const long long U = plan.total_units;
    std::vector<uint32_t> meta(U), gcount(U, 0), tsum(U), bitlen(U), bitlen_bm(U), reached(U, 0);
    std::vector<long long> evkey(U), prev_ev(U);
    std::vector<unsigned long long> bitoff(U);
    const size_t NH = plan.scans.size() * 4 * 256;
    std::vector<uint32_t> hist(NH, 0), hist_bm(NH, 0);
    // scan-major: classify, inline symbols, groups, tables, lengths, offsets, bit buffer
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
    std::vector<uint32_t> hist_inline = hist;
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
    std::vector<ge::Table> tabs(plan.scans.size() * 4);
    std::vector<int> cs(257), oth(257); std::vector<long long> fr(257);
    for (size_t t = 0; t < tabs.size(); t++) ge::build_table(hist.data() + t * 256, tabs[t], cs.data(), oth.data(), fr.data());
    for (const ge::Scan &s : plan.scans) for (int u = 0; u < s.nblocks; u++) {
        ge::LenSink sk; sk.tabs = tabs.data() + s.tab_base;
        ge::gen_block(s, ge::locate(s, u), gcount[s.unit_base + u], sk);
        bitlen[s.unit_base + u] = (uint32_t)sk.bits;
    }
    { unsigned long long run = 0; for (long long i = 0; i < U; i++) { bitoff[i] = run; run += bitlen[i]; } }
    std::vector<uint32_t> w_ref((size_t)plan.total_words, 0), w_bm((size_t)plan.total_words, 0);
    for (const ge::Scan &s : plan.scans) for (int u = 0; u < s.nblocks; u++) {
        auto orw = [&](long long i, uint32_t v) { w_ref[i] |= v; };
        ge::EmitSink<decltype(orw)> sk(tabs.data() + s.tab_base, orw, s.word_base, bitoff[s.unit_base + u] - bitoff[s.unit_base]);
        ge::gen_block(s, ge::locate(s, u), gcount[s.unit_base + u], sk);
        sk.finish();
    }
    // block-major, one component at a time as a CTA row of the device passes sees it
    for (const BlockComp &bc : plan.comps) {
        uint32_t h[ENC_TAB_ENTRIES] = {}, tc[ENC_TAB_ENTRIES] = {};
        uint8_t tl[ENC_TAB_ENTRIES] = {};
        for (int k = 0; k < ENC_TAB_ENTRIES; k++) {
            int symbol; const int t = enc_entry_table(bc, k, symbol);
            if (t >= 0) { tc[k] = tabs[t].code_len[symbol]; tl[k] = (uint8_t)tc[k]; }
        }
        const int16_t *cb = bc.coef + bc.comp_off;
        for (int row = 0; row < bc.bh; row++) for (int col = 0; col < bc.bw; col++) {
            const int16_t *blk = cb + ((long long)row * bc.bw + col) * 64;
            const ge::Masks3 M = ge::make_masks3(blk);
            for (int j = 0; j < bc.nscan; j++) {
                const EncVisit &v = bc.visit[j];
                const ge::Scan &s = plan.scans[v.scan];
                const int u = enc_unit_of(bc, v.ns, row, col);
                if (u < 0) continue;
                if (u >= s.nblocks) return 5;
                const ge::BlockRef want = ge::locate(s, u);
                if (want.blk != blk) return 5;
                const long long gi = v.unit_base + u;
                reached[gi]++;
                ge::BlockRef b; b.blk = blk; b.prev = nullptr; b.slot = 0;
                if (v.mode == ge::MODE_SEQ || v.mode == ge::MODE_DC_FIRST) {
                    const int p = enc_dc_prev(bc, v.ns, row, col);
                    b.prev = p < 0 ? nullptr : cb + (long long)p * 64;
                    if (b.prev != want.prev) return 6;
                }
                if (ge::classify_m(v, M) != meta[gi]) return 7;
                TabHist hk{kind_tabs(h, v)};
                ge::gen_block_m(v, v.tbl, b, M, 0, hk);
                ge::LenSinkT<ge::KindTabs<const uint8_t>> lk{kind_tabs<const uint8_t>(tl, v)};
                ge::gen_block_m(v, v.tbl, b, M, gcount[gi], lk);
                bitlen_bm[gi] = (uint32_t)lk.bits;
                auto orw = [&](long long i, uint32_t x) { w_bm[i] |= x; };
                ge::EmitSink<decltype(orw), decltype(orw), ge::KindTabs<const uint32_t>> ek(kind_tabs<const uint32_t>(tc, v), orw, orw, s.word_base,
                                                                                             bitoff[gi] - bitoff[v.unit_base]);
                ge::gen_block_m(v, v.tbl, b, M, gcount[gi], ek);
                ek.finish();
            }
        }
        for (int k = 0; k < ENC_TAB_ENTRIES; k++) {
            int symbol; const int t = enc_entry_table(bc, k, symbol);
            if (h[k]) { if (t < 0) return 3; hist_bm[(size_t)t * 256 + symbol] += h[k]; }
        }
    }
    for (long long i = 0; i < U; i++) if (reached[i] != 1) return 9;
    if (hist_bm != hist_inline) return 3;
    if (bitlen_bm != bitlen) return 8;
    return w_bm == w_ref ? 0 : 4;
}
