// main.cpp -- b200clt: a C++ stand-in for caesiumclt's main.rs (flags of caesium-clt's src/options.rs:47-190,
// flow of main.rs:43-113, JSON of main.rs:15-34,164-187) so the drop-in path can be exercised end to end on boxes
// without a Rust toolchain.  Presentation (progress bars, colours) is deliberately not reproduced.
#include <cerrno>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>
#include "compressor.h"

using namespace b200clt;

static void json_str(std::string &o, const std::string &s)
{
    o += '"';
    for (unsigned char c : s) {
        if (c == '"' || c == '\\') { o += '\\'; o += (char)c; }
        else if (c == '\n') o += "\\n";
        else if (c < 0x20) { char b[8]; snprintf(b, sizeof b, "\\u%04x", c); o += b; }
        else o += (char)c;
    }
    o += '"';
}

// clap rejects "8x" / "abc" for a numeric flag; atoi would read them as 8 / 0
static bool parse_uint(const char *v, long long lo, long long hi, long long &out)
{
    char *end = nullptr; errno = 0;
    const long long x = strtoll(v, &end, 10);
    if (errno || end == v || *end || x < lo || x > hi) return false;
    out = x; return true;
}

static int usage(const char *msg)
{
    fprintf(stderr, "error: %s\n\nUsage: b200clt [OPTIONS] <--quality <QUALITY>|--lossless|--max-size <MAX_SIZE>> <--output <OUTPUT>|--same-folder-as-input> [FILES]...\n", msg);
    return 2;
}

int main(int argc, char **argv)
{
    CompressionOptions o;
    std::vector<std::string> inputs;
    bool recursive = false, dry_run = false, quiet = false, json = false, timing = false;
    int threads = 0, n_gpus = 0, mode_count = 0, dest_count = 0;
    auto num = [&](int &i, long long lo, long long hi) -> long long { const std::string flag = argv[i]; long long v; const char *t = nullptr; if (i + 1 < argc) t = argv[++i]; if (!t || !parse_uint(t, lo, hi, v)) { usage(("invalid value for '" + flag + "'").c_str()); exit(2); } return v; };
    auto need = [&](int &i) -> const char * { if (i + 1 >= argc) { usage((std::string("a value is required for '") + argv[i] + "'").c_str()); exit(2); } return argv[++i]; };
    for (int i = 1; i < argc; i++) {
        std::string a = argv[i];
        if (a == "-q" || a == "--quality") { o.quality = (uint32_t)num(i, 0, 100); mode_count++; }
        else if (a == "--lossless") { o.lossless = true; mode_count++; }
        else if (a == "--max-size") { uint64_t b; if (!parse_byte_size(need(i), b)) return usage("Invalid size format"); o.max_size = (size_t)b; mode_count++; }
        else if (a == "--width") o.width = (uint32_t)num(i, 0, 0xFFFFFFFFll);
        else if (a == "--height") o.height = (uint32_t)num(i, 0, 0xFFFFFFFFll);
        else if (a == "--long-edge") o.long_edge = (uint32_t)num(i, 0, 0xFFFFFFFFll);
        else if (a == "--short-edge") o.short_edge = (uint32_t)num(i, 0, 0xFFFFFFFFll);
        else if (a == "-o" || a == "--output") { o.output_folder = need(i); dest_count++; }
        else if (a == "--same-folder-as-input") { o.same_folder_as_input = true; dest_count++; }
        else if (a == "-R" || a == "--recursive") recursive = true;
        else if (a == "-S" || a == "--keep-structure") o.keep_structure = true;
        else if (a == "-O" || a == "--overwrite") { std::string v = need(i); if (v == "all") o.overwrite_policy = OverwritePolicy::All; else if (v == "never") o.overwrite_policy = OverwritePolicy::Never; else if (v == "bigger") o.overwrite_policy = OverwritePolicy::Bigger; else return usage("invalid value for --overwrite"); }
        else if (a == "--format") { std::string v = need(i); if (v == "jpeg") o.format = OutputFormat::Jpeg; else if (v == "png") o.format = OutputFormat::Png; else if (v == "webp") o.format = OutputFormat::Webp; else if (v == "tiff") o.format = OutputFormat::Tiff; else if (v == "gif") o.format = OutputFormat::Gif; else if (v == "original") o.format = OutputFormat::Original; else return usage("invalid value for --format"); }
        else if (a == "--suffix") o.suffix = need(i);
        else if (a == "-e" || a == "--exif") o.exif = true;
        else if (a == "--keep-dates") o.keep_dates = true;
        else if (a == "--png-opt-level") o.png_opt_level = (uint8_t)num(i, 0, 6);
        else if (a == "--zopfli") o.zopfli = true;
        else if (a == "--jpeg-chroma-subsampling") { std::string v = need(i); if (v == "4:4:4") o.jpeg_chroma_subsampling = B200_CS_444; else if (v == "4:2:2") o.jpeg_chroma_subsampling = B200_CS_422; else if (v == "4:2:0") o.jpeg_chroma_subsampling = B200_CS_420; else if (v == "4:1:1") o.jpeg_chroma_subsampling = B200_CS_411; else if (v == "auto") o.jpeg_chroma_subsampling = B200_CS_AUTO; else return usage("invalid value for --jpeg-chroma-subsampling"); }
        else if (a == "--jpeg-baseline") o.jpeg_baseline = true;
        else if (a == "--no-upscale") o.no_upscale = true;
        else if (a == "--strip-icc") o.strip_icc = true;
        else if (a == "--min-savings") { MinSavingsThreshold t; std::string e; if (!parse_min_savings(need(i), t, e)) return usage(e.c_str()); o.min_savings = t; }
        else if (a == "--threads") threads = (int)num(i, 0, 4096);
        else if (a == "--gpus") n_gpus = (int)num(i, 0, 64);          // extension: number of GPUs to shard over (0 = all)
        else if (a == "--timing") timing = true;                 // extension: print MP/s to stderr
        else if (a == "--dry-run" || a == "-d") dry_run = true;
        else if (a == "-Q" || a == "--quiet") quiet = true;
        else if (a == "--json") json = true;
        else if (a == "--verbose") need(i);
        else if (!a.empty() && a[0] == '-') return usage(("unexpected argument '" + a + "'").c_str());
        else inputs.push_back(a);
    }
    if (mode_count != 1) return usage("exactly one of --quality, --lossless, --max-size is required");        // options.rs:141
    if (dest_count != 1) return usage("exactly one of --output, --same-folder-as-input is required");          // options.rs:181
    if ((o.width || o.height) && (o.long_edge || o.short_edge)) return usage("--width/--height cannot be used with --long-edge/--short-edge");
    std::string base;
    std::vector<std::string> files = scan_files(inputs, recursive, base);
    if (files.empty() || base.empty()) { if (json) printf("{\"version\":\"1.0.0\",\"dry_run\":%s,\"error\":\"No valid base path found\",\"files\":[],\"summary\":{\"total_files\":0,\"success\":0,\"skipped\":0,\"errors\":0,\"original_size\":0,\"compressed_size\":0,\"savings_bytes\":0,\"savings_percent\":0.0}}\n", dry_run ? "true" : "false"); else if (!quiet) fprintf(stderr, "No valid base path found\n"); return files.empty() ? 0 : 255; }
    o.base_path = base;
    if (!dry_run) b200_init(n_gpus);                    // before any lazy initialisation, so --gpus always takes effect
    auto t0 = std::chrono::steady_clock::now();
    std::vector<CompressionResult> res = start_compression(files, o, dry_run, threads);
    double secs = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    uint64_t orig = 0, comp = 0; size_t ok = 0, sk = 0, er = 0;
    for (auto &r : res) { orig += r.original_size; comp += r.compressed_size; if (r.status == CompressionStatus::Success) ok++; else if (r.status == CompressionStatus::Skipped) sk++; else er++; }
    long long savings = (long long)orig - (long long)comp;
    double pct = orig ? (double)savings / (double)orig * 100.0 : 0.0;
    if (json) {
        std::string s = "{\"version\":\"1.0.0\",\"dry_run\":"; s += dry_run ? "true" : "false"; s += ",\"error\":null,\"files\":[";
        for (size_t i = 0; i < res.size(); i++) {
            const auto &r = res[i];
            if (i) s += ',';
            s += "{\"original_path\":"; json_str(s, r.original_path); s += ",\"output_path\":"; json_str(s, r.output_path);
            s += ",\"original_size\":" + std::to_string(r.original_size) + ",\"compressed_size\":" + std::to_string(r.compressed_size);
            s += ",\"status\":\""; s += r.status == CompressionStatus::Success ? "success" : r.status == CompressionStatus::Skipped ? "skipped" : "error"; s += "\",\"message\":"; json_str(s, r.message); s += '}';
        }
        char tail[256]; snprintf(tail, sizeof tail, "],\"summary\":{\"total_files\":%zu,\"success\":%zu,\"skipped\":%zu,\"errors\":%zu,\"original_size\":%llu,\"compressed_size\":%llu,\"savings_bytes\":%lld,\"savings_percent\":%.6g}}",
                                  res.size(), ok, sk, er, (unsigned long long)orig, (unsigned long long)comp, savings, pct);
        s += tail; puts(s.c_str());
    } else if (!quiet) {
        for (auto &r : res) if (r.status != CompressionStatus::Success) printf("[%s] %s: %s\n", r.status == CompressionStatus::Skipped ? "SKIPPED" : "ERROR", r.original_path.c_str(), r.message.c_str());
        printf("Compressed %zu files (%zu success, %zu skipped, %zu errors)\n%llu -> %llu bytes [Saved %lld bytes (%.2f%%)]\n", res.size(), ok, sk, er, (unsigned long long)orig, (unsigned long long)comp, savings, pct);
    }
    if (timing) fprintf(stderr, "b200clt: %zu files in %.3f s (%.1f files/s)\n", res.size(), secs, res.size() / (secs > 0 ? secs : 1));
    b200_shutdown();
    return 0;
}
