// tests/emul/gpudec_write_emul.cpp -- TEST INFRASTRUCTURE.  Serial CPU run of the device entropy DECODER's passes with the
// write pass as jpeg_gpudec.cu runs it: gd::decode_owned_blocks (a block belongs to the subsequence in which it starts) into a
// sink that stores whole sectors, on a buffer nobody cleared.  gpudec_emul.cpp next to it writes through decode_subsequence
// and single stores into a zeroed buffer: the two must agree on coefficients and anomalies.  Not part of the product.
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>
#include "../../caesium-clt_b200/csrc/jpeg_gpudec_core.h"
#include "../../caesium-clt_b200/csrc/jpeg_gpuenc_plan.h"

using namespace b200;

namespace {
constexpr int16_t POISON = 0x5A5A;     // what the coefficient buffer holds before the write pass: nothing clears it
// The device sink's shape: the current 16-coefficient sector of the current block is held and leaves whole, zero sectors fill
// the rest of the block, the sector with the DC coefficient delivers the DC difference; the end of a block only marks it ended,
// its last sectors leave when the next block's DC arrives or in finish().  A gd::Cursor is stepped per block and cross-checked
// against ge::locate / gd::dc_slot_index; every sector store is counted per block of the layout.
struct WriteSink {
    const ge::Scan *scan; const gd::Walk *walk; int16_t *base; int32_t *dc; uint8_t *stored /*[layout block]: mask of sectors*/; int *faults;
    uint32_t cur, total; gd::Cursor c{}; int16_t *ptr = nullptr; int32_t *dcp = nullptr; int16_t held[16] = {0}; int sec = 0; bool ended = true; uint32_t anom = 0;
    void seek() { c.seek(*walk, cur); }
    void locate()
    {
        ptr = cur < total ? base + c.offset(*walk) : nullptr; dcp = dc + c.dc_slot(*walk);
        uint32_t cs;
        if (ptr && (ptr != ge::locate(*scan, (int)cur).blk || c.dc_slot(*walk) != gd::dc_slot_index(*scan, cur, &cs))) (*faults)++;
    }
    void flush_to(int target)
    {
        for (; sec < target; sec++) {
            if (sec == 0) *dcp = held[0];
            uint8_t &m = stored[(ptr - base) / 64];
            if (m & (1 << sec)) (*faults)++;            // a sector stored twice: two writers, or one writer going backwards
            m |= (uint8_t)(1 << sec);
            memcpy(ptr + sec * 16, held, 32); memset(held, 0, 32);
        }
    }
    void coef(int k, int v)
    {
        const int s = k >> 4;
        if (ended || s != sec) {
            if (ptr) flush_to(ended ? 4 : s);
            if (ended) { ended = false; locate(); }
            sec = s;
        }
        if (ptr) held[k & 15] = (int16_t)v;
    }
    void anomaly(uint32_t m) { if (cur < total) anom |= m; }
    void block_done() { cur++; c.next(*walk); ended = true; }
    void finish() { if (ptr) flush_to(4); }
};
}

// returns 0 ok, 10 not eligible for the device decoder, 11 no convergence within max_rounds, 14 stream anomaly inside a real
// block (the host decodes the image; *anomalies = the gd::ANOM_* rules that fired), 13 / 15 the write pass addressed a block wrongly /
// did not store every block of the scan whole exactly once, other = parse error
extern "C" int emul_gpu_write_checked(const uint8_t *jpeg, size_t len, int subseq_bits, int max_rounds, int16_t *out, long long out_cap,
                                       int *rounds_used, int *anomalies)
{
    if (anomalies) *anomalies = 0;
    std::string err;
    JpegReader rd(jpeg, len);
    if (!rd.read_header(err)) return 1;
    JpegReader::DeviceScan ds;
    if (!rd.device_decodable(ds)) return 10;
    const JpegGeom &g = rd.geom();
    if (out_cap < g.total_coefs) return 2;
    // pass: unstuff
    std::vector<uint8_t> stream;
    for (size_t i = ds.ecs_begin; i < ds.ecs_end; i++) { stream.push_back(jpeg[i]); if (jpeg[i] == 0xFF && i + 1 < ds.ecs_end && jpeg[i + 1] == 0) i++; }
    const size_t stream_bytes = stream.size();
    stream.resize((stream_bytes + 3) / 4 * 4 + 16, 0xFF);          // word alignment + 0xFF padding, as the device buffer has
    gd::Geometry G{};
    int q = 0;
    for (int c = 0; c < g.ncomp; c++) for (int k = 0; k < (g.ncomp == 1 ? 1 : g.hs[c] * g.vs[c]); k++) { G.dc_tbl[q] = ds.td[c]; G.ac_tbl[q] = ds.ta[c]; q++; }
    G.blocks_per_mcu = q;
    G.total_blocks = g.ncomp == 1 ? (uint32_t)(g.rbw[0] * g.rbh[0]) : (uint32_t)(g.mcux * g.mcuy * q);
    G.nbits = (uint32_t)stream_bytes * 8; G.subseq_bits = (uint32_t)subseq_bits; G.nsub = (G.nbits + G.subseq_bits - 1) / G.subseq_bits;
    const uint8_t *db[8], *dv[8];
    for (int id = 0; id < 4; id++) for (int kind = 0; kind < 2; kind++) { const bool pr = rd.dht_present(kind, id); db[kind * 4 + id] = pr ? rd.dht_bits(kind, id) : nullptr; dv[kind * 4 + id] = pr ? rd.dht_vals(kind, id) : nullptr; }
    std::vector<gd::DecTables> tabv(1);
    if (!gd::build_dec_tables(db, dv, G, tabv[0])) return 12;
    const gd::DecTables &tabs = tabv[0];
    // as GpuDecoder does: cleared only where the layout has blocks the scan does not code, otherwise left as it was found
    const bool padded = (long long)G.total_blocks * 64 != g.total_coefs;
    for (long long j = 0; j < g.total_coefs; j++) out[j] = padded ? 0 : POISON;
    GpuEncPlan plan; const int16_t *base = out;
    gpuenc_plan(g, false, &base, 1, plan);
    const ge::Scan &scan = plan.scans[0];
    // pass: round 0
    std::vector<gd::DecState> A(G.nsub), B(G.nsub);
    std::vector<uint32_t> nblk(G.nsub);
    for (uint32_t i = 0; i < G.nsub; i++) { gd::NullSink sk; gd::DecState st{i * G.subseq_bits, 0, 0}; A[i] = gd::decode_subsequence(stream.data(), G, tabs, i, st, sk); nblk[i] = sk.nblk; }
    int rounds = 0; bool changed = true;
    while (changed && rounds < max_rounds) {
        changed = false; rounds++;
        for (uint32_t i = 0; i < G.nsub; i++) {
            gd::NullSink sk; gd::DecState st = i ? A[i - 1] : gd::DecState{0, 0, 0};
            B[i] = gd::decode_subsequence(stream.data(), G, tabs, i, st, sk); nblk[i] = sk.nblk;
            if (!gd::same_state(B[i], A[i])) changed = true;
        }
        A.swap(B);
    }
    if (rounds_used) *rounds_used = rounds;
    if (changed) return 11;
    // pass: prefix sum + write
    const gd::Walk walk = gd::make_walk(scan);
    int faults = 0; uint32_t anom = 0;
    std::vector<uint32_t> first(G.nsub); { uint32_t run = 0; for (uint32_t i = 0; i < G.nsub; i++) { first[i] = run; run += nblk[i]; } }
    std::vector<int32_t> dc(G.total_blocks, 0x7FFFFFFF);
    std::vector<uint8_t> stored((size_t)(g.total_coefs / 64), 0);
    for (uint32_t i = 0; i < G.nsub; i++) {
        gd::DecState st = i ? A[i - 1] : gd::DecState{0, 0, 0};
        WriteSink sk{&scan, &walk, out, dc.data(), stored.data(), &faults, gd::first_owned_block(first[i], st), G.total_blocks};
        sk.seek();
        gd::decode_owned_blocks(stream.data(), G, tabs, i, st, sk);
        sk.finish();
        anom |= sk.anom;
    }
    if (faults) return 13;
    if (anomalies) *anomalies = (int)anom;
    if (anom) return 14;
    // every block of the scan fully written exactly once, and no other block of the layout touched
    for (uint32_t u = 0; u < G.total_blocks; u++) { uint8_t &m = stored[(ge::locate(scan, (int)u).blk - out) / 64]; if (m != 0xF) return 15; m = 0; }
    for (uint8_t m : stored) if (m) return 15;
    // pass: DC prefix sums per component over the differences the write pass delivered
    int pred[4] = {0, 0, 0, 0};
    gd::Cursor c; c.seek(walk, 0);
    for (uint32_t u = 0; u < G.total_blocks; u++, c.next(walk)) { ge::BlockRef r = ge::locate(scan, (int)u); pred[r.slot] += dc[c.dc_slot(walk)]; const_cast<int16_t *>(r.blk)[0] = (int16_t)pred[r.slot]; }
    return 0;
}
