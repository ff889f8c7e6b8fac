// compressor_c.cpp -- plain-C hooks over the C++ host mirror (compressor.h) so the Python tests can drive the same
// cases the reference's inline unit tests cover (caesium-clt's src/compressor.rs:607-1109).  Built into libb200clt.so.
#include <cstring>
#include <string>
#include "compressor.h"

using namespace b200clt;

extern "C" {

struct b200clt_options {   // flat CompressionOptions (compressor.rs:46-70); -1 / NULL = None
    int quality; long long max_size; int lossless, exif, png_opt_level, zopfli;
    int width, height, long_edge, short_edge;
    const char *output_folder; int same_folder_as_input; const char *base_path; const char *suffix;
    int overwrite_policy /*0 all,1 never,2 bigger*/, format /*0 jpeg,1 png,2 gif,3 webp,4 tiff,5 original*/;
    int keep_dates, keep_structure; unsigned jpeg_chroma_subsampling; int jpeg_baseline, no_upscale, strip_icc;
    const char *min_savings;   // "10%" / "100KB" / NULL
};

static CompressionOptions conv(const b200clt_options *c)
{
    CompressionOptions o;
    if (c->quality >= 0) o.quality = (uint32_t)c->quality;
    if (c->max_size >= 0) o.max_size = (size_t)c->max_size;
    o.lossless = c->lossless; o.exif = c->exif; o.png_opt_level = (uint8_t)c->png_opt_level; o.zopfli = c->zopfli;
    if (c->width >= 0) o.width = (uint32_t)c->width;
    if (c->height >= 0) o.height = (uint32_t)c->height;
    if (c->long_edge >= 0) o.long_edge = (uint32_t)c->long_edge;
    if (c->short_edge >= 0) o.short_edge = (uint32_t)c->short_edge;
    if (c->output_folder) o.output_folder = std::string(c->output_folder);
    o.same_folder_as_input = c->same_folder_as_input;
    o.base_path = c->base_path ? c->base_path : "";
    if (c->suffix) o.suffix = std::string(c->suffix);
    o.overwrite_policy = (OverwritePolicy)c->overwrite_policy;
    static const OutputFormat fm[] = {OutputFormat::Jpeg, OutputFormat::Png, OutputFormat::Gif, OutputFormat::Webp, OutputFormat::Tiff, OutputFormat::Original};
    o.format = fm[c->format < 0 || c->format > 5 ? 5 : c->format];
    o.keep_dates = c->keep_dates; o.keep_structure = c->keep_structure; o.jpeg_chroma_subsampling = c->jpeg_chroma_subsampling;
    o.jpeg_baseline = c->jpeg_baseline; o.no_upscale = c->no_upscale; o.strip_icc = c->strip_icc;
    if (c->min_savings) { MinSavingsThreshold t; std::string e; if (parse_min_savings(c->min_savings, t, e)) o.min_savings = t; }
    return o;
}

static void put(char *dst, size_t cap, const std::string &s) { if (!dst || !cap) return; size_t n = s.size() < cap - 1 ? s.size() : cap - 1; memcpy(dst, s.data(), n); dst[n] = 0; }

int b200clt_build_compression_parameters(const b200clt_options *c, const uint8_t *buf, size_t len, b200_params *out, char *err, size_t err_cap)
{
    std::vector<uint8_t> b(buf, buf + len); std::string e;
    bool ok = build_compression_parameters(conv(c), b, *out, e);
    put(err, err_cap, e);
    return ok ? 0 : 1;
}

int b200clt_compute_output_full_path(const char *output_directory, const char *input_file, const char *base_directory, int keep_structure,
                                     const char *suffix, int format, int same_folder, char *out_dir, char *out_name, size_t cap)
{
    static const OutputFormat fm[] = {OutputFormat::Jpeg, OutputFormat::Png, OutputFormat::Gif, OutputFormat::Webp, OutputFormat::Tiff, OutputFormat::Original};
    std::string d, n;
    bool ok = compute_output_full_path(output_directory, input_file, base_directory, keep_structure, suffix, fm[format], same_folder, d, n);
    put(out_dir, cap, d); put(out_name, cap, n);
    return ok ? 0 : 1;
}

// start_compression over n files; status[i] 0 success / 1 skipped / 2 error; messages/output paths '\n'-joined into text
int b200clt_start_compression(const char *const *files, int n, const b200clt_options *c, int dry_run, int threads,
                              int *status, unsigned long long *original_size, unsigned long long *compressed_size, char *text, size_t text_cap)
{
    std::vector<std::string> f(files, files + n);
    auto res = start_compression(f, conv(c), dry_run, threads);
    std::string t;
    for (int i = 0; i < n; i++) {
        status[i] = (int)res[i].status; original_size[i] = res[i].original_size; compressed_size[i] = res[i].compressed_size;
        t += res[i].output_path + "\t" + res[i].message + "\n";
    }
    put(text, text_cap, t);
    return 0;
}

int b200clt_parse_min_savings(const char *v, int *is_pct, double *pct, unsigned long long *bytes)
{
    MinSavingsThreshold t; std::string e;
    if (!parse_min_savings(v, t, e)) return 1;
    *is_pct = t.is_percentage; *pct = t.percent; *bytes = t.bytes; return 0;
}

int b200clt_scan_files(const char *const *args, int n, int recursive, char *text, size_t cap)
{
    std::vector<std::string> a(args, args + n); std::string base;
    auto files = scan_files(a, recursive, base);
    std::string t = base + "\n";
    for (auto &f : files) t += f + "\n";
    put(text, cap, t);
    return (int)files.size();
}

} // extern "C"
