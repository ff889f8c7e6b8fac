// tests/emul/gpuenc_dcrun_emul.cpp -- TEST INFRASTRUCTURE.  Runs the device encoder's MCU-run coder of the DC-first interleaved
// scan (caesium-clt_b200/csrc/jpeg_gpuenc.cu: the compact DC array k_geb_classify writes, k_geb_dc_first's per-thread slots and CTA
// runs, k_ge_place) on the CPU, CTA by CTA and last CTA first, and compares the scan's bit buffer with the scan-major formulation
// (ge::locate + gen_block, unit after unit), bit for bit.  The CTA size and the slot capacity are parameters: small ones give many
// runs and send MCUs down the overflow path (coded a second time, straight to their place).
// Not linked into the product library.
#include <cstring>
#include <string>
#include <vector>
#include "../../caesium-clt_b200/csrc/jpeg_gpuenc_plan.h"

using namespace b200;

// dc_mode 0: the decoded DC values; 1: -1024 and 1023 alternating along each component's compact array (every difference of
// category 11, and a category-11 value against the predictor 0 at each component's start); 2: seeded values in [-1024, 1023].
// 0: equal; 1 / 2: the input does not parse / decode; 3: no DC-first interleaved scan; 4: bit buffers differ; 5: a run outgrew the
// scan's part of the arena.  *overflowed = MCUs that did not fit their slot.
extern "C" int emul_dcrun_check(const uint8_t *jpeg, size_t len, int dc_mode, int cta, int slot_words, long long *overflowed)
{
    std::string err;
    JpegReader rd(jpeg, len);
    if (!rd.read_header(err)) return 1;
    const JpegGeom &g = rd.geom();
    std::vector<int16_t> coefs((size_t)g.total_coefs);
    if (!rd.decode(coefs.data(), err)) return 2;
    GpuEncPlan plan;
    const int16_t *base = coefs.data();
    gpuenc_plan(g, true, &base, 1, plan);
    if (plan.dc_first_scan < 0) return 3;
    unsigned long long rng = 0x9E3779B97F4A7C15ull;
    for (const BlockComp &bc : plan.comps) for (int row = 0; row < bc.bh; row++) for (int col = 0; col < bc.bw; col++) {
        int16_t &dc = coefs[(size_t)bc.comp_off + ((size_t)row * bc.bw + col) * 64];
        const int k = enc_dc_index(bc, row, col);
        if (dc_mode == 1) dc = (k & 1) ? 1023 : -1024;
        else if (dc_mode == 2) { rng = rng * 6364136223846793005ull + 1442695040888963407ull; dc = (int16_t)((int)(rng >> 40) % 2048 - 1024); }
    }
    jpeg_fill_dummy_blocks(g, coefs.data());
    const ge::Scan &s = plan.scans[plan.dc_first_scan];

    // optimal DC tables of the scan from its symbol histogram
    std::vector<uint32_t> hist(4 * 256, 0);
    for (int u = 0; u < s.nblocks; u++) {
        auto add = [&](int idx) { hist[idx]++; };
        ge::HistSink<decltype(add)> sk(add);
        ge::gen_block(s, ge::locate(s, u), 0, sk);
    }
    std::vector<ge::Table> tabs(4);
    std::vector<int> cs(257), oth(257); std::vector<long long> fr(257);
    for (int t = 0; t < 4; t++) ge::build_table(hist.data() + t * 256, tabs[t], cs.data(), oth.data(), fr.data());

    // scan-major reference
    const long long nw = (long long)s.nblocks + 2;      // a DC unit takes at most 16 + 11 bits
    std::vector<uint32_t> w_ref((size_t)nw, 0), w_dev((size_t)nw, 0);
    unsigned long long total = 0;
    {
        auto orw = [&](long long i, uint32_t v) { w_ref[i] |= v; };
        for (int u = 0; u < s.nblocks; u++) {
            ge::EmitSink<decltype(orw)> sk(tabs.data(), orw, 0, total);
            ge::gen_block(s, ge::locate(s, u), 0, sk);
            sk.finish();
            total = sk.bits_written(0);
        }
    }

    // the compact DC array, as k_geb_classify writes it (component at mask_base, entries in MCU order)
    std::vector<int16_t> dcarr((size_t)plan.total_comp_blocks);
    for (const BlockComp &bc : plan.comps) for (int row = 0; row < bc.bh; row++) for (int col = 0; col < bc.bw; col++)
        dcarr[(size_t)bc.mask_base + enc_dc_index(bc, row, col)] = bc.coef[bc.comp_off + ((long long)row * bc.bw + col) * 64];

    // k_geb_dc_first with CTAs of `cta` MCUs, last CTA first
    const int nmcu = s.mcux * s.mcuy, nruns = (nmcu + cta - 1) / cta;
    const uint32_t arena_words = (uint32_t)((total + 31) / 32) + (uint32_t)nruns;
    std::vector<uint32_t> arena((size_t)arena_words + 1, 0), runlen(nruns), runpos(nruns), slot((size_t)std::max(slot_words, 1) * cta);
    uint32_t cursor = 0;
    long long nover = 0;
    ge::ScanTabs tc(tabs.data());
    auto ora = [&](long long w, uint32_t v) { arena[w] |= v; };
    auto sta = [&](long long w, uint32_t v) { arena[w] = v; };
    for (int x = nruns - 1; x >= 0; x--) {
        std::vector<uint32_t> nb(cta, 0), off(cta);
        for (int t = 0; t < cta; t++) {
            const int m = x * cta + t;
            if (m >= nmcu) continue;
            auto sls = [&](long long w, uint32_t v) { if (w < slot_words) slot[(size_t)w * cta + t] = v; };
            ge::EmitSink<decltype(sls), decltype(sls)> sk(tc, sls, sls, 0, 0);
            ge::gen_dc_mcu(s, dcarr.data(), m, sk);
            sk.finish();
            nb[t] = (uint32_t)sk.bits_written(0);
        }
        uint32_t L = 0;
        for (int t = 0; t < cta; t++) { off[t] = L; L += nb[t]; }
        const uint32_t a = cursor;
        cursor += (L + 31) / 32;
        if (cursor > arena_words) return 5;
        runlen[x] = L; runpos[x] = a;
        for (int t = 0; t < cta; t++) {
            const unsigned long long at = (unsigned long long)a * 32 + off[t];
            if (nb[t] <= (uint32_t)slot_words * 32) ge::place_bits([&](long long k) { return slot[(size_t)k * cta + t]; }, nb[t], at, ora, sta);
            else {
                nover++;
                ge::EmitSink<decltype(ora), decltype(sta)> sk(tc, ora, sta, 0, at);
                ge::gen_dc_mcu(s, dcarr.data(), x * cta + t, sk);
                sk.finish();
            }
        }
    }
    // k_ge_place: run offsets, one lane stride at a time as a warp does it
    uint32_t run = 0;
    for (int r = 0; r < nruns; r++) {
        const uint32_t *src = arena.data() + runpos[r];
        for (int lane = 0; lane < 32; lane++)
            ge::place_bits([&](long long k) { return src[k]; }, runlen[r], run,
                           [&](long long w, uint32_t v) { w_dev[w] |= v; }, [&](long long w, uint32_t v) { w_dev[w] = v; }, lane, 32);
        run += runlen[r];
    }
    if (overflowed) *overflowed = nover;
    return run == total && w_dev == w_ref ? 0 : 4;
}
