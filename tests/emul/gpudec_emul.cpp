// tests/emul/gpudec_emul.cpp -- TEST INFRASTRUCTURE.  Serial CPU run of the device entropy DECODER's passes
// (caesium-clt_b200/csrc/jpeg_gpudec_core.h), in the order jpeg_gpudec.cu launches them.  Not part of the product.
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>
#include "../../caesium-clt_b200/csrc/jpeg_gpudec_core.h"
#include "../../caesium-clt_b200/csrc/jpeg_gpuenc_plan.h"

using namespace b200;

namespace {
struct WriteSink {             // the device sink's logic: a gd::Cursor stepped per block, cross-checked against ge::locate
    const ge::Scan *scan; const gd::Walk *walk; int16_t *base; uint32_t cur, total; gd::Cursor c; int16_t *ptr; int *mismatch;
    void seek() { c.seek(*walk, cur); set(); }
    void set()
    {
        ptr = cur < total ? base + c.offset(*walk) : nullptr;
        if (ptr && ptr != ge::locate(*scan, (int)cur).blk) (*mismatch)++;
    }
    void coef(int k, int v) { if (ptr) ptr[k] = (int16_t)v; }
    void anomaly(uint32_t m) { if (ptr) anom |= m; }
    void block_done() { cur++; c.next(*walk); set(); }
    uint32_t anom = 0;
};
}

// returns 0 ok, 10 not eligible for the device decoder, 11 no convergence within max_rounds, 14 stream anomaly inside a real
// block (the host decodes the image; *anomalies = the gd::ANOM_* rules that fired), other = parse error
extern "C" int emul_gpu_decode_checked(const uint8_t *jpeg, size_t len, int subseq_bits, int max_rounds, int16_t *out, long long out_cap,
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
    memset(out, 0, (size_t)g.total_coefs * 2);
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
    int mismatch = 0; uint32_t anom = 0;
    std::vector<uint32_t> first(G.nsub); { uint32_t run = 0; for (uint32_t i = 0; i < G.nsub; i++) { first[i] = run; run += nblk[i]; } }
    for (uint32_t i = 0; i < G.nsub; i++) {
        WriteSink sk{&scan, &walk, out, first[i], G.total_blocks, {}, nullptr, &mismatch};
        sk.seek();
        gd::DecState st = i ? A[i - 1] : gd::DecState{0, 0, 0};
        gd::decode_subsequence(stream.data(), G, tabs, i, st, sk);
        anom |= sk.anom;
    }
    if (mismatch) return 13;
    if (anomalies) *anomalies = (int)anom;
    if (anom) return 14;
    // pass: DC prefix sums per component in scan order
    int pred[4] = {0, 0, 0, 0};
    for (uint32_t u = 0; u < G.total_blocks; u++) { ge::BlockRef r = ge::locate(scan, (int)u); int16_t *b = const_cast<int16_t *>(r.blk); pred[r.slot] += b[0]; b[0] = (int16_t)pred[r.slot]; }
    return 0;
}

// the same without the anomaly report
extern "C" int emul_gpu_decode(const uint8_t *jpeg, size_t len, int subseq_bits, int max_rounds, int16_t *out, long long out_cap, int *rounds_used)
{
    return emul_gpu_decode_checked(jpeg, len, subseq_bits, max_rounds, out, out_cap, rounds_used, nullptr);
}

// Kernel-form tables against the jdhuff.c reference form: every 16-bit pattern (followed by `tail` bits) through every table the
// scan uses must give the same (length, symbol).  Returns the number of disagreements, -1 if the file is not eligible, -2 if the
// tables do not fit the pool; *pool_used = second-level entries in use.
extern "C" long long emul_gpu_dec_table_check(const uint8_t *jpeg, size_t len, int *pool_used)
{
    std::string err;
    JpegReader rd(jpeg, len);
    if (!rd.read_header(err)) return -1;
    JpegReader::DeviceScan ds;
    if (!rd.device_decodable(ds)) return -1;
    const JpegGeom &g = rd.geom();
    gd::Geometry G{};
    int q = 0;
    for (int c = 0; c < g.ncomp; c++) for (int k = 0; k < (g.ncomp == 1 ? 1 : g.hs[c] * g.vs[c]); k++) { G.dc_tbl[q] = ds.td[c]; G.ac_tbl[q] = ds.ta[c]; q++; }
    G.blocks_per_mcu = q;
    const uint8_t *db[8], *dv[8];
    for (int id = 0; id < 4; id++) for (int kind = 0; kind < 2; kind++) { const bool pr = rd.dht_present(kind, id); db[kind * 4 + id] = pr ? rd.dht_bits(kind, id) : nullptr; dv[kind * 4 + id] = pr ? rd.dht_vals(kind, id) : nullptr; }
    std::vector<gd::DecTables> T(1);
    if (!gd::build_dec_tables(db, dv, G, T[0])) return -2;
    if (pool_used) *pool_used = T[0].next;
    long long bad = 0;
    for (int b = 0; b < q; b++) for (int ac = 0; ac < 2; ac++) {
        gd::DecTable ref;
        const int t = ac * 4 + (ac ? G.ac_tbl[b] : G.dc_tbl[b]);
        gd::build_dec_table(db[t], dv[t], ref);
        for (uint32_t pat = 0; pat < 65536; pat++) for (uint32_t tail = 0; tail < 2; tail++) {
            const uint32_t bits = (pat << 16) | (tail ? 0xFFFFu : 0u);
            int l; const int sym = gd::decode_symbol(ref, bits, &l);
            const uint32_t e = gd::lookup_symbol(T[0], T[0].sel[2 * b + ac], bits);
            if ((int)(e >> 8) != l || (int)(e & 0xFF) != sym) bad++;
        }
    }
    return bad;
}

// build_dec_tables on caller-supplied DHT payloads: `ntab` AC tables (ids 0..ntab-1, all with the same BITS / HUFFVAL) used by an
// MCU of `ntab` blocks, one shared DC table.  Returns 1 ok / 0 refused; *pool_used = second-level entries in use.  When the tables
// are accepted every 16-bit pattern is checked against the jdhuff.c search (*bad = disagreements).
extern "C" int emul_build_tables_raw(const uint8_t *ac_bits, const uint8_t *ac_vals, const uint8_t *dc_bits, const uint8_t *dc_vals, int ntab, int *pool_used, long long *bad)
{
    gd::Geometry G{};
    G.blocks_per_mcu = ntab;
    for (int q = 0; q < ntab; q++) { G.dc_tbl[q] = 0; G.ac_tbl[q] = q; }
    const uint8_t *db[8] = {dc_bits, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr}, *dv[8] = {dc_vals, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    for (int q = 0; q < ntab && q < 4; q++) { db[4 + q] = ac_bits; dv[4 + q] = ac_vals; }
    std::vector<gd::DecTables> T(1);
    const bool ok = gd::build_dec_tables(db, dv, G, T[0]);
    *pool_used = T[0].next; *bad = 0;
    // the kernels stage the first nlook slots only: a selector past them would read first-level entries nobody staged
    for (int i = 0; i < 20; i++) if (T[0].sel[i] >= T[0].nlook * gd::LOOK_N) (*bad)++;
    if (!ok) {
        for (int i = 0; i < gd::MAX_TABLES * gd::LOOK_N; i++) if (T[0].look[i] != (16 << 8)) (*bad)++;      // refused: all-invalid tables
        return 0;
    }
    gd::DecTable ref; gd::build_dec_table(ac_bits, ac_vals, ref);
    for (int q = 0; q < ntab; q++) for (uint32_t pat = 0; pat < 65536; pat++) {
        const uint32_t bits = (pat << 16) | 0x5A5Au;
        int l; const int sym = gd::decode_symbol(ref, bits, &l);
        const uint32_t e = gd::lookup_symbol(T[0], T[0].sel[2 * q + 1], bits);
        if ((int)(e >> 8) != l || (int)(e & 0xFF) != sym) (*bad)++;
    }
    return 1;
}
