// jpeg_gpuenc_plan.h -- host-side planning for the block-parallel entropy encoder: turns a geometry + scan script into
// the ge::Scan descriptors the kernels (or the CPU emulation in tests/emul/) iterate.  Plain C++, no CUDA.
#pragma once
#include <algorithm>
#include <vector>
#include "jpeg_gpuenc_core.h"
#include "jpeg_host.h"

namespace b200 {

// Block-major view used by the encoder passes: one descriptor per (image, component); a thread owns one block, reads it
// once, and serves every scan that visits the block (e.g. luma: DC scan + two AC bands + the refinement scan).
//
// A CTA copies the component's visit records to shared memory and keeps the Huffman tables of its visits on chip: one slot per
// table kind a visit codes, the AC tables first (256 symbols each), then the DC table (DC symbols are bit counts 0..16).
// jpeg_scan_script's progressive luma has three AC visits and one DC visit, a sequential scan one of each.
// A CTA of the block-major passes owns ENC_THREADS consecutive blocks of one component.  In a scan with one component these are
// consecutive units: the CTA's part of such a scan is one run of the scan's bits, coded in one pass (see k_geb_emit).
constexpr int ENC_THREADS = 128;
// The DC-first scan of a progressive colour script is coded one MCU per thread (k_geb_dc_first): a CTA's ENC_DC_MCUS consecutive
// MCUs are consecutive units of the scan, so it too is one run of the scan's bits.
constexpr int ENC_DC_MCUS = 128;
constexpr int ENC_MAX_VISITS = 6, ENC_AC_SLOTS = 3, ENC_DC_SLOTS = 1, ENC_DC_SYMBOLS = 17;
constexpr int ENC_TAB_ENTRIES = ENC_AC_SLOTS * 256 + ENC_DC_SLOTS * ENC_DC_SYMBOLS;   // entry of (AC slot a, symbol) = a * 256 + symbol
constexpr int ENC_DC_ENTRY = ENC_AC_SLOTS * 256;                                      // entry of (DC slot, symbol) = ENC_DC_ENTRY + symbol

struct EncVisit {                       // one scan visiting the component: what the symbol loops and the unit index need
    int scan;                           // index into GpuEncPlan::scans
    int mode, Ss, Se, Al, ns;
    int tbl;                            // the component's Huffman table id
    int unit_base;                      // Scan::unit_base (a batch has fewer than 2^31 units)
    int lu_base;                        // ns > 1: Scan::lu_base
    int run_base;                       // Scan::run_base
    int ac_entry;                       // first on-chip entry of the visit's AC table (unused by a DC-only scan)
};

struct BlockComp {
    const int16_t *coef;                // image base
    long long comp_off;
    int bw, bh, rbw, rbh, hs, vs;
    int q_base, blocks_per_mcu, mcux;   // position of the component's first block inside an MCU (interleaved scans)
    int nscan;
    EncVisit visit[ENC_MAX_VISITS];
    int tab[ENC_AC_SLOTS + ENC_DC_SLOTS];   // batch-wide table index (Scan::tab_base + kind * 2 + tbl) of each slot, -1: unused
    long long mask_base;                // first block of this component in the batch-wide per-block mask array
};

// the unit of component block (row, col) in a scan with ns components (-1: a padding block the scan does not code)
GE_HD int enc_unit_of(const BlockComp &bc, int ns, int row, int col)
{
    if (ns == 1) return (row < bc.rbh && col < bc.rbw) ? row * bc.rbw + col : -1;
    const int m = (row / bc.vs) * bc.mcux + col / bc.hs, q = bc.q_base + (row % bc.vs) * bc.hs + (col % bc.hs);
    return m * bc.blocks_per_mcu + q;
}
// the component block (index row * bw + col) whose DC value predicts that of block (row, col) in a scan with ns components, -1
// for the component's first block in the scan: ge::locate()'s predecessor, walked back on the component's own grid
GE_HD int enc_dc_prev(const BlockComp &bc, int ns, int row, int col)
{
    if (ns == 1) return col > 0 ? row * bc.bw + col - 1 : row > 0 ? (row - 1) * bc.bw + bc.rbw - 1 : -1;
    if (col % bc.hs) return row * bc.bw + col - 1;                      // earlier block of the same MCU row
    if (row % bc.vs) return (row - 1) * bc.bw + col + bc.hs - 1;        // last block of the MCU's previous row
    if (col) return (row + bc.vs - 1) * bc.bw + col - 1;               // last block of the previous MCU
    if (row) return (row - 1) * bc.bw + bc.mcux * bc.hs - 1;           // ... which ends the previous MCU row
    return -1;
}

// entry of component block (row, col) in the component's compact DC array: its blocks in MCU order, hs * vs per MCU (the grid of
// a component of an interleaved image is whole MCUs)
GE_HD int enc_dc_index(const BlockComp &bc, int row, int col)
{
    return ((row / bc.vs) * bc.mcux + col / bc.hs) * (bc.hs * bc.vs) + (row % bc.vs) * bc.hs + col % bc.hs;
}

// the table of on-chip entry k and the entry's symbol; -1 for a slot the component does not use
GE_HD int enc_entry_table(const BlockComp &bc, int k, int &symbol)
{
    if (k < ENC_DC_ENTRY) { symbol = k & 255; return bc.tab[k >> 8]; }
    symbol = k - ENC_DC_ENTRY; return bc.tab[ENC_AC_SLOTS];
}

struct GpuEncPlan {
    std::vector<BlockComp> comps;       // image-major
    bool on_chip = true;                // every component's visits fit ENC_MAX_VISITS and its tables the on-chip slots
    int max_comp_blocks = 0;
    std::vector<ge::Scan> scans;        // image-major: scans of image 0, then image 1, ...
    std::vector<ScanDef> defs;          // one script (shared by all images of the batch)
    int scans_per_image = 0;
    long long units_per_image = 0, words_per_image = 0;
    long long total_units = 0, total_words = 0, total_comp_blocks = 0;
    long long total_lunits = 0;         // units of the scans with ns > 1
    bool unit_coded = false;            // some scan with ns > 1 is coded unit by unit (k_geb_len, offsets): a sequential colour script
    int dc_first_scan = -1;             // index in the script of the DC-first scan with ns > 1, coded in MCU runs (k_geb_dc_first)
    int total_runs = 0, max_runs = 0;   // CTA runs of the scans coded in runs: in all, and in the largest scan
};

// coef_base[i] = device (or host) pointer to image i's coefficient buffer (geometry g, zigzag)
inline void gpuenc_plan(const JpegGeom &g, bool progressive, const int16_t *const *coef_base, int nimages, GpuEncPlan &p)
{
    ScanDef sc[16];
    const int ns = jpeg_scan_script(g, progressive, sc);
    p.defs.assign(sc, sc + ns);
    p.scans_per_image = ns;
    p.scans.clear();
    long long unit = 0, word = 0, lunit = 0;
    int run = 0;
    p.max_runs = 0; p.unit_coded = false; p.dc_first_scan = -1;
    long long image_blocks = 0;         // the compact DC arrays of an image's components, back to back (= BlockComp::mask_base)
    for (int c = 0; c < g.ncomp; c++) image_blocks += (long long)g.bw[c] * g.bh[c];
    for (int im = 0; im < nimages; im++) {
        for (int si = 0; si < ns; si++) {
            const ScanDef &d = sc[si];
            ge::Scan s{};
            s.coef = coef_base[im];
            s.ns = d.ns; s.Ss = d.Ss; s.Se = d.Se; s.Al = d.Al;
            if (!progressive) s.mode = ge::MODE_SEQ;
            else if (d.Ss == 0) s.mode = ge::MODE_DC_FIRST;          // the script has no DC refinement scans
            else s.mode = d.Ah == 0 ? ge::MODE_AC_FIRST : ge::MODE_AC_REFINE;
            s.blocks_per_mcu = 0;
            for (int i = 0; i < d.ns; i++) {
                const int c = d.ci[i];
                s.comp[i] = c; s.hs[i] = g.hs[c]; s.vs[i] = g.vs[c]; s.bw[i] = g.bw[c]; s.comp_off[i] = g.comp_offset[c]; s.tbl[i] = c ? 1 : 0;
                s.blocks_per_mcu += g.hs[c] * g.vs[c];
            }
            s.mcux = g.mcux; s.mcuy = g.mcuy;
            s.rbw = g.rbw[d.ci[0]]; s.rbh = g.rbh[d.ci[0]];
            s.nblocks = d.ns > 1 ? g.mcux * g.mcuy * s.blocks_per_mcu : s.rbw * s.rbh;
            s.unit_base = unit; unit += s.nblocks;
            s.lu_base = -1; s.run_base = -1; s.nruns = 0;
            if (d.ns > 1) { s.lu_base = lunit; lunit += s.nblocks; }
            if (d.ns > 1 && s.mode == ge::MODE_DC_FIRST) {
                if (im == 0) p.dc_first_scan = si;
                s.run_base = run; s.nruns = (g.mcux * g.mcuy + ENC_DC_MCUS - 1) / ENC_DC_MCUS; run += s.nruns; p.max_runs = std::max(p.max_runs, s.nruns);
                for (int i = 0; i < d.ns; i++) {
                    long long b = im * image_blocks;
                    for (int c = 0; c < d.ci[i]; c++) b += (long long)g.bw[c] * g.bh[c];
                    s.dc_base[i] = b;
                }
            } else if (d.ns > 1) p.unit_coded = true;
            else { s.run_base = run; s.nruns = (g.bw[d.ci[0]] * g.bh[d.ci[0]] + ENC_THREADS - 1) / ENC_THREADS; run += s.nruns; p.max_runs = std::max(p.max_runs, s.nruns); }
            s.tab_base = (int)p.scans.size() * 4;
            s.word_base = word; s.word_cap = (long long)s.nblocks * 32 + 64; word += s.word_cap;   // 128 B per block: the size of its coefficients
            p.scans.push_back(s);
        }
        if (im == 0) { p.units_per_image = unit; p.words_per_image = word; }
    }
    p.total_units = unit; p.total_words = word; p.total_lunits = lunit; p.total_runs = run;
    p.comps.clear(); p.max_comp_blocks = 0; p.total_comp_blocks = 0; p.on_chip = true;
    for (int im = 0; im < nimages; im++) {
        int qb = 0;
        for (int c = 0; c < g.ncomp; c++) {
            BlockComp bc{};
            bc.coef = coef_base[im]; bc.comp_off = g.comp_offset[c];
            bc.bw = g.bw[c]; bc.bh = g.bh[c]; bc.rbw = g.rbw[c]; bc.rbh = g.rbh[c]; bc.hs = g.hs[c]; bc.vs = g.vs[c];
            bc.q_base = qb; bc.mcux = g.mcux;
            bc.blocks_per_mcu = 0; for (int cc = 0; cc < g.ncomp; cc++) bc.blocks_per_mcu += g.hs[cc] * g.vs[cc];
            qb += g.hs[c] * g.vs[c];
            bc.nscan = 0;
            int nac = 0, ndc = 0;
            for (int k = 0; k < ENC_AC_SLOTS + ENC_DC_SLOTS; k++) bc.tab[k] = -1;
            for (int si = 0; si < ns; si++) for (int i = 0; i < sc[si].ns; i++) {
                if (sc[si].ci[i] != c) continue;
                const ge::Scan &s = p.scans[(size_t)im * ns + si];
                const bool dc = s.mode == ge::MODE_SEQ || s.mode == ge::MODE_DC_FIRST, ac = s.mode != ge::MODE_DC_FIRST;
                if (bc.nscan == ENC_MAX_VISITS || nac + ac > ENC_AC_SLOTS || ndc + dc > ENC_DC_SLOTS) { p.on_chip = false; continue; }
                EncVisit &v = bc.visit[bc.nscan++];
                v.scan = im * ns + si; v.mode = s.mode; v.Ss = s.Ss; v.Se = s.Se; v.Al = s.Al; v.ns = s.ns; v.tbl = s.tbl[i];
                v.unit_base = (int)s.unit_base; v.lu_base = (int)s.lu_base; v.run_base = s.run_base;
                v.ac_entry = ac ? nac * 256 : 0;
                if (ac) bc.tab[nac++] = s.tab_base + 2 + v.tbl;
                if (dc) bc.tab[ENC_AC_SLOTS + ndc++] = s.tab_base + v.tbl;
            }
            bc.mask_base = p.total_comp_blocks; p.total_comp_blocks += (long long)bc.bw * bc.bh;
            p.comps.push_back(bc);
            p.max_comp_blocks = std::max(p.max_comp_blocks, bc.bw * bc.bh);
        }
    }
}

} // namespace b200
