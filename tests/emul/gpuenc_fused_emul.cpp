// tests/emul/gpuenc_fused_emul.cpp -- TEST INFRASTRUCTURE.  Runs the device encoder's size and emit scheme
// (caesium-clt_b200/csrc/jpeg_gpuenc.cu: k_geb_classify's correction-bit counts, k_ge_tables' bits per table, k_ge_scanout, k_geb_len
// over the interleaved scans, k_geb_emit's per-thread slots and CTA runs, k_ge_place) on the CPU and compares it with the scan-major
// formulation:
//   - each scan's size from its histograms (count * (code length + sym_extra_bits)) plus its correction bits equals the sum of the
//     per-unit bit lengths;
//   - the bit buffer built from slots, runs in a staging arena and their placement is the scan-major bit buffer, bit for bit, for
//     any slot capacity (a small one sends units down the overflow path: coded a second time, straight to their place).
// The CTAs of a component are run last to first, so the runs land in the arena in another order than the scan's.
// Not linked into the product library.
#include <cstring>
#include <string>
#include <vector>
#include "../../caesium-clt_b200/csrc/jpeg_gpuenc_plan.h"

using namespace b200;

namespace {
template <class T>
ge::KindTabs<T> kind_tabs(T *tab, const EncVisit &v) { return ge::KindTabs<T>{tab + ENC_DC_ENTRY, tab + v.ac_entry}; }
}

// 0: all agree; 1 / 2: the input does not parse / decode; 3: a scan size; 4: bit buffers; 5: a run outgrew the scan's part of
// the arena; 10: the script does not fit the on-chip slots.  *overflowed = units that did not fit their slot.
extern "C" int emul_fused_check(const uint8_t *jpeg, size_t len, int progressive, int slot_words, long long *overflowed)
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
    const int NS = (int)plan.scans.size();
    std::vector<uint32_t> meta(U), gcount(U, 0), tsum(U), bitlen(U);
    std::vector<long long> evkey(U);
    std::vector<unsigned long long> bitoff(U);
    std::vector<uint32_t> hist((size_t)NS * 4 * 256, 0);
    // scan-major reference: classify, histograms, groups, tables, lengths, offsets, bit buffer
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
    { uint32_t run = 0; for (long long i = 0; i < U; i++) { tsum[i] = run; run += (uint32_t)ge::meta_tail(meta[i]); } }
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
    std::vector<ge::Table> tabs((size_t)NS * 4);
    std::vector<int> cs(257), oth(257); std::vector<long long> fr(257);
    for (size_t t = 0; t < tabs.size(); t++) ge::build_table(hist.data() + t * 256, tabs[t], cs.data(), oth.data(), fr.data());
    for (const ge::Scan &s : plan.scans) for (int u = 0; u < s.nblocks; u++) {
        ge::LenSink sk; sk.tabs = tabs.data() + s.tab_base;
        ge::gen_block(s, ge::locate(s, u), gcount[s.unit_base + u], sk);
        bitlen[s.unit_base + u] = (uint32_t)sk.bits;
    }
    { unsigned long long run = 0; for (long long i = 0; i < U; i++) { bitoff[i] = run; run += bitlen[i]; } }
    std::vector<uint32_t> w_ref((size_t)plan.total_words, 0), w_dev((size_t)plan.total_words, 0);
    for (const ge::Scan &s : plan.scans) for (int u = 0; u < s.nblocks; u++) {
        auto orw = [&](long long i, uint32_t v) { w_ref[i] |= v; };
        ge::EmitSink<decltype(orw)> sk(tabs.data() + s.tab_base, orw, s.word_base, bitoff[s.unit_base + u] - bitoff[s.unit_base]);
        ge::gen_block(s, ge::locate(s, u), gcount[s.unit_base + u], sk);
        sk.finish();
    }

    // ---- scan sizes: correction bits counted block-major (k_geb_classify), bits per table (k_ge_tables), totals (k_ge_scanout)
    std::vector<uint32_t> corr(NS, 0), total(NS, 0), arena_base(NS, 0);
    for (const BlockComp &bc : plan.comps) {
        const int16_t *cb = bc.coef + bc.comp_off;
        for (int row = 0; row < bc.bh; row++) for (int col = 0; col < bc.bw; col++) {
            const ge::Masks3 M = ge::make_masks3(cb + ((long long)row * bc.bw + col) * 64);
            for (int j = 0; j < bc.nscan; j++) if (enc_unit_of(bc, bc.visit[j].ns, row, col) >= 0) corr[bc.visit[j].scan] += (uint32_t)ge::corr_bits_m(bc.visit[j], M);
        }
    }
    uint32_t abase = 0;
    for (int si = 0; si < NS; si++) {
        unsigned long long tb = corr[si];
        for (int t = 0; t < 4; t++) for (int sym = 0; sym < 256; sym++) {
            const uint32_t f = hist[((size_t)si * 4 + t) * 256 + sym];
            if (f) tb += (unsigned long long)f * ((tabs[(size_t)si * 4 + t].code_len[sym] & 0xFFu) + (unsigned)ge::sym_extra_bits(t >> 1, sym));
        }
        const ge::Scan &s = plan.scans[si];
        unsigned long long want = 0;
        for (int u = 0; u < s.nblocks; u++) want += bitlen[s.unit_base + u];
        if (tb != want) return 3;
        total[si] = (uint32_t)tb;
        arena_base[si] = abase;
        if (s.nruns) abase += (total[si] + 31) / 32 + (uint32_t)s.nruns;
    }

    // ---- interleaved scans: lengths over their units only (k_geb_len), offsets
    std::vector<uint32_t> lbitlen((size_t)std::max(plan.total_lunits, 1ll));
    std::vector<uint32_t> lbitoff(lbitlen.size());
    for (const ge::Scan &s : plan.scans) if (s.ns > 1) for (int u = 0; u < s.nblocks; u++) lbitlen[s.lu_base + u] = bitlen[s.unit_base + u];
    { uint32_t run = 0; for (size_t i = 0; i < lbitlen.size(); i++) { lbitoff[i] = run; run += lbitlen[i]; } }

    // ---- emit (k_geb_emit), CTA by CTA, last CTA first
    std::vector<uint32_t> arena((size_t)abase + 1, 0), cursor(NS, 0), runlen((size_t)std::max(plan.total_runs, 1)), runpos(runlen.size());
    std::vector<uint32_t> slot((size_t)std::max(slot_words, 1) * ENC_THREADS);
    long long nover = 0;
    for (const BlockComp &bc : plan.comps) {
        uint32_t tc[ENC_TAB_ENTRIES] = {};
        for (int k = 0; k < ENC_TAB_ENTRIES; k++) { int symbol; const int t = enc_entry_table(bc, k, symbol); if (t >= 0) tc[k] = tabs[t].code_len[symbol]; }
        const int16_t *cb = bc.coef + bc.comp_off;
        const int nblk = bc.bw * bc.bh, ncta = (nblk + ENC_THREADS - 1) / ENC_THREADS;
        for (int x = ncta - 1; x >= 0; x--) {
            const int i0 = x * ENC_THREADS;
            for (int j = 0; j < bc.nscan; j++) {
                const EncVisit &v = bc.visit[j];
                typedef ge::KindTabs<const uint32_t> KT;
                uint32_t nb[ENC_THREADS] = {};
                int unit[ENC_THREADS];
                ge::Masks3 Ms[ENC_THREADS];
                ge::BlockRef refs[ENC_THREADS];
                for (int t = 0; t < ENC_THREADS; t++) {
                    const int i = i0 + t, row = i / bc.bw, col = i - row * bc.bw;
                    unit[t] = i < nblk ? enc_unit_of(bc, v.ns, row, col) : -1;
                    if (unit[t] < 0) continue;
                    ge::BlockRef &r = refs[t];
                    r.blk = cb + (long long)i * 64; r.prev = nullptr; r.slot = 0;
                    if (v.mode == ge::MODE_SEQ || v.mode == ge::MODE_DC_FIRST) { const int p = enc_dc_prev(bc, v.ns, row, col); if (p >= 0) r.prev = cb + (long long)p * 64; }
                    Ms[t] = ge::make_masks3(r.blk);
                }
                const ge::Scan &s = plan.scans[v.scan];
                auto orw = [&](long long w, uint32_t val) { w_dev[w] |= val; };
                auto ora = [&](long long w, uint32_t val) { arena[w] |= val; };
                auto sta = [&](long long w, uint32_t val) { arena[w] = val; };
                if (v.ns > 1) {
                    for (int t = 0; t < ENC_THREADS; t++) {
                        const int u = unit[t];
                        if (u < 0) continue;
                        ge::EmitSink<decltype(orw), decltype(orw), KT> sk(kind_tabs<const uint32_t>(tc, v), orw, orw, s.word_base, lbitoff[v.lu_base + u] - lbitoff[v.lu_base]);
                        ge::gen_block_m(v, v.tbl, refs[t], Ms[t], gcount[v.unit_base + u], sk);
                        sk.finish();
                    }
                    continue;
                }
                for (int t = 0; t < ENC_THREADS; t++) {
                    const int u = unit[t];
                    if (u < 0) continue;
                    auto sls = [&](long long w, uint32_t val) { if (w < slot_words) slot[(size_t)w * ENC_THREADS + t] = val; };
                    ge::EmitSink<decltype(sls), decltype(sls), KT> sk(kind_tabs<const uint32_t>(tc, v), sls, sls, 0, 0);
                    ge::gen_block_m(v, v.tbl, refs[t], Ms[t], gcount[v.unit_base + u], sk);
                    sk.finish();
                    nb[t] = (uint32_t)sk.bits_written(0);
                }
                uint32_t off[ENC_THREADS], L = 0;
                for (int t = 0; t < ENC_THREADS; t++) { off[t] = L; L += nb[t]; }
                const uint32_t a = arena_base[v.scan] + cursor[v.scan];
                cursor[v.scan] += (L + 31) / 32;
                if (cursor[v.scan] > (total[v.scan] + 31) / 32 + (uint32_t)s.nruns) return 5;
                runlen[v.run_base + x] = L; runpos[v.run_base + x] = a;
                for (int t = 0; t < ENC_THREADS; t++) {
                    const unsigned long long at = (unsigned long long)a * 32 + off[t];
                    if (nb[t] <= (uint32_t)slot_words * 32) {
                        ge::place_bits([&](long long k) { return slot[(size_t)k * ENC_THREADS + t]; }, nb[t], at, ora, sta);
                    } else {
                        nover++;
                        ge::EmitSink<decltype(ora), decltype(sta), KT> sk(kind_tabs<const uint32_t>(tc, v), ora, sta, 0, at);
                        ge::gen_block_m(v, v.tbl, refs[t], Ms[t], gcount[v.unit_base + unit[t]], sk);
                        sk.finish();
                    }
                }
            }
        }
    }
    // ---- run offsets and placement (k_ge_place), one lane stride at a time as a warp does it
    std::vector<uint32_t> runoff(runlen.size());
    { uint32_t run = 0; for (size_t r = 0; r < runlen.size(); r++) { runoff[r] = run; run += runlen[r]; } }
    for (const ge::Scan &s : plan.scans) for (int x = 0; x < s.nruns; x++) {
        const int r = s.run_base + x;
        const uint32_t *src = arena.data() + runpos[r];
        uint32_t *dst = w_dev.data() + s.word_base;
        for (int lane = 0; lane < 32; lane++)
            ge::place_bits([&](long long k) { return src[k]; }, runlen[r], runoff[r] - runoff[s.run_base],
                           [&](long long w, uint32_t val) { dst[w] |= val; }, [&](long long w, uint32_t val) { dst[w] = val; }, lane, 32);
    }
    if (overflowed) *overflowed = nover;
    return w_dev == w_ref ? 0 : 4;
}
