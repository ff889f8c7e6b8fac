// compressor.h -- C++ mirror of caesiumclt's host side around the codec boundary (caesium-clt's src/compressor.rs).
// The reference host is Rust; no cargo/rustc exists in this image, so the same interface is kept here in C++ (same
// names, argument meaning, messages and policies) on top of the C-ABI, for the b200clt CLI and the tests.  A Rust
// maintainer keeps the original file and swaps only the three caesium::* calls (INTEGRATION.md).
#pragma once
#include <cstdint>
#include <optional>
#include <string>
#include <vector>
#include "../../include/b200_caesium.h"

namespace b200clt {

enum class OverwritePolicy { All, Never, Bigger };                         // options.rs:14-22
enum class OutputFormat { Jpeg, Png, Gif, Webp, Tiff, Original };          // options.rs:24-32
enum class CompressionStatus { Success, Skipped, Error };                  // compressor.rs:19-25

struct MinSavingsThreshold { bool is_percentage; double percent; uint64_t bytes; };   // options.rs:6-11

struct CompressionResult {                                                 // compressor.rs:37-44
    std::string original_path, output_path;
    uint64_t original_size = 0, compressed_size = 0;
    CompressionStatus status = CompressionStatus::Error;
    std::string message;
};

struct CompressionOptions {                                                // compressor.rs:46-70
    std::optional<uint32_t> quality;
    std::optional<size_t> max_size;
    bool lossless = false, exif = false;
    uint8_t png_opt_level = 3;
    bool zopfli = false;
    std::optional<uint32_t> width, height, long_edge, short_edge;
    std::optional<std::string> output_folder;
    bool same_folder_as_input = false;
    std::string base_path;
    std::optional<std::string> suffix;
    OverwritePolicy overwrite_policy = OverwritePolicy::All;
    OutputFormat format = OutputFormat::Original;
    bool keep_dates = false, keep_structure = false;
    uint32_t jpeg_chroma_subsampling = B200_CS_AUTO;
    bool jpeg_baseline = false, no_upscale = false, strip_icc = false;
    std::optional<MinSavingsThreshold> min_savings;
};

constexpr uint64_t MAX_FILE_SIZE = 500ull * 1024 * 1024;                   // compressor.rs:72

// compressor.rs:74-101 -- data-parallel map over files, input order preserved; threads = 0 -> all usable cores
std::vector<CompressionResult> start_compression(const std::vector<std::string> &input_files, const CompressionOptions &options,
                                                 bool dry_run, int threads);
CompressionResult perform_compression(const std::string &input_file, const CompressionOptions &options, bool dry_run);   // :103-184
// :266-315 -- returns false with result.message set on failure
bool perform_image_compression(const std::string &input_file, const CompressionOptions &options, CompressionResult &result, std::vector<uint8_t> &out);
// :411-446 (+ :503-561) -- false + err when the resize parameters cannot be derived
bool build_compression_parameters(const CompressionOptions &options, const std::vector<uint8_t> &buffer, b200_params &params, std::string &err);
// :448-501
bool compute_output_full_path(const std::string &output_directory, const std::string &input_file_path, const std::string &base_directory,
                              bool keep_structure, const std::string &suffix, OutputFormat format, bool same_folder_as_input,
                              std::string &out_dir, std::string &out_name);
// imagesize::blob_size + EXIF orientation swap (:538-561)
bool get_real_resolution(const std::vector<uint8_t> &buffer, bool keep_metadata, size_t &width, size_t &height, std::string &err);
// scan_files.rs:50-92 (extension list + magic sniff: jpeg/png/webp/gif), returns files and the common base path
std::vector<std::string> scan_files(const std::vector<std::string> &args, bool recursive, std::string &base_path);
bool parse_min_savings(const std::string &val, MinSavingsThreshold &out, std::string &err);   // options.rs:232-257
bool parse_byte_size(const std::string &val, uint64_t &out);                                  // bytesize::ByteSize FromStr

} // namespace b200clt
