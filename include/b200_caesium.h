/*
 * b200_caesium.h -- C-ABI of libb200caesium.so, the H100-native replacement for the
 * `libcaesium` crate calls made by caesiumclt's per-image hot path.
 *
 * The reference has no FFI of its own; the seam is the Rust crate boundary in
 * caesium-clt's src/compressor.rs:287-306:
 *     caesium::compress_in_memory(Vec<u8>, &CSParameters)                        (compressor.rs:305)
 *     caesium::convert_in_memory(Vec<u8>, &CSParameters, SupportedFileTypes)     (compressor.rs:289,300)
 *     caesium::compress_to_size_in_memory(Vec<u8>, &mut CSParameters, usize, bool)(compressor.rs:295,298)
 * Each entry point below names the call it replaces.  All functions are thread-safe and
 * re-entrant (the caller is a rayon par_iter, compressor.rs:81-83), never abort, and never
 * fall back to a CPU codec: if no CUDA device / kernel image is available they return
 * B200_ERR_NO_DEVICE.  Inputs are borrowed for the duration of the call; outputs are
 * allocated by the library and released with b200_free().
 */
#ifndef B200_CAESIUM_H
#define B200_CAESIUM_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- status codes (CaesiumError.code analogue; message mirrors "{message} [{code}]") ---- */
enum {
    B200_OK = 0,
    B200_ERR_INVALID_ARGUMENT = 1,
    B200_ERR_UNKNOWN_FORMAT = 2,     /* input sniffed as none of jpeg/png/webp/gif/tiff */
    B200_ERR_UNSUPPORTED = 3,        /* recognised, but this path is not implemented on the GPU build:
                                        the Rust host may route the file to caesium::* instead */
    B200_ERR_CORRUPT_INPUT = 4,
    B200_ERR_NO_DEVICE = 5,          /* no CUDA device / sm_90a image -- there is NO CPU fallback */
    B200_ERR_CUDA = 6,
    B200_ERR_OUT_OF_MEMORY = 7,
    B200_ERR_SAME_FORMAT = 8,        /* convert_in_memory asked for the input's own format */
    B200_ERR_TOO_LARGE = 9           /* compress_to_size could not reach max_output_size */
};

typedef struct {
    int32_t code;        /* B200_OK or B200_ERR_* */
    char *message;       /* NULL when code == 0; malloc'd, release with b200_free() */
} b200_status;

/* caesium::SupportedFileTypes (compressor.rs:589-598 map_supported_formats) */
enum { B200_FMT_JPEG = 0, B200_FMT_PNG = 1, B200_FMT_GIF = 2, B200_FMT_WEBP = 3, B200_FMT_TIFF = 4, B200_FMT_UNKNOWN = 5 };

/* caesium::parameters::ChromaSubsampling as libcaesium's C interface spells it */
enum { B200_CS_AUTO = 0, B200_CS_444 = 444, B200_CS_422 = 422, B200_CS_420 = 420, B200_CS_411 = 411 };

/* caesium::parameters::CSParameters -- exactly the 15 fields compressor.rs:411-446 and :503-536 set */
typedef struct {
    uint8_t  keep_metadata;             /* compressor.rs:431  (options.exif) */
    uint32_t jpeg_quality;              /* :415 */
    uint32_t jpeg_chroma_subsampling;   /* :433  B200_CS_* */
    uint8_t  jpeg_progressive;          /* :434  (!jpeg_baseline) */
    uint8_t  jpeg_optimize;             /* :427  (lossless => coefficient-domain transcode) */
    uint8_t  jpeg_preserve_icc;         /* :425  (!strip_icc) */
    uint32_t png_quality;               /* :416 */
    uint32_t png_optimization_level;    /* :436  0..6 */
    uint8_t  png_force_zopfli;          /* :437 */
    uint8_t  png_optimize;              /* :428  (lossless) */
    uint32_t gif_quality;               /* :418-424 */
    uint32_t webp_quality;              /* :417 */
    uint8_t  webp_lossless;             /* :429 */
    uint32_t width;                     /* :512-528, 0 = keep aspect */
    uint32_t height;
} b200_params;

/* CSParameters::new() defaults */
void b200_params_default(b200_params *p);

/* ---- lifecycle -------------------------------------------------------------------------------- */
/* Optional (every entry point lazily initialises): n_gpus = 0 means all visible devices.  A maintainer
 * would call this after the rayon pool is built (main.rs:65).  Returns B200_OK or B200_ERR_NO_DEVICE. */
int  b200_init(int n_gpus);
/* One-process-per-GPU launchers (torchrun): bind the library to exactly this CUDA ordinal. */
int  b200_init_device(int device_ordinal);
/* Frees every slot (streams, pinned and device buffers).  Calls made afterwards initialise the library again. */
void b200_shutdown(void);
int  b200_device_count(void);         /* devices the library is driving (0 before init / without GPU) */
/* jobs (megabatches or single images) device `index` (0 .. b200_device_count()-1) has been handed so far, and the NUMA node its
 * worker threads are bound to (-1: unknown / binding off) -- how b200_compress_batch's sharding can be observed */
long long b200_device_jobs(int index);
int  b200_device_numa_node(int index);
const char *b200_version(void);
void b200_free(void *p);
/* Where JPEG entropy coding runs.  Bit 0: Huffman ENCODE on the device; bit 1: Huffman DECODE on the device (baseline
 * single-scan inputs; anything else is decoded on the calling thread).  Default 3 (env B200_ENTROPY=gpu); 0
 * (B200_ENTROPY=host) keeps both on the host as north_star words it; gpuenc = 1, gpudec = 2.  Output bytes are identical
 * in every mode. */
int  b200_set_entropy_mode(int mode);

/* ---- the three calls of compressor.rs:287-306 -------------------------------------------------- */
/* replaces caesium::compress_in_memory (compressor.rs:305) */
b200_status b200_compress_in_memory(const uint8_t *in, size_t in_len, const b200_params *params,
                                    uint8_t **out, size_t *out_len);
/* replaces caesium::convert_in_memory (compressor.rs:289, :300); fmt = B200_FMT_* */
b200_status b200_convert_in_memory(const uint8_t *in, size_t in_len, const b200_params *params, uint32_t fmt,
                                   uint8_t **out, size_t *out_len);
/* replaces caesium::compress_to_size_in_memory (compressor.rs:295, :298); may mutate params->*_quality */
b200_status b200_compress_to_size_in_memory(const uint8_t *in, size_t in_len, b200_params *params,
                                            size_t max_output_size, uint8_t return_smallest,
                                            uint8_t **out, size_t *out_len);

/* ---- batch form of start_compression's par_iter (compressor.rs:74-101) -------------------------
 * Blocking; runs the n images on an internal worker pool (n_threads = 0: one per usable host core)
 * and shards them round-robin over the initialised GPUs.  status[i]/out[i]/out_len[i] per image,
 * input order preserved like par_iter().collect().  Returns the number of failed images. */
int b200_compress_batch(const uint8_t *const *in, const size_t *in_len, int n, const b200_params *params,
                        int n_threads, uint8_t **out, size_t *out_len, b200_status *status);

/* ---- format sniff (infer::get in compressor.rs:259-264 / scan_files.rs:30-40) ------------------ */
uint32_t b200_sniff_format(const uint8_t *in, size_t in_len);

/* ---- JPEG stage entry points (the pieces compress_in_memory is assembled from) ----------------
 * Coefficient buffers are int16, one 64-entry block after another in ZIGZAG order, blocks in raster
 * order per component, components back to back, each component padded to whole MCUs. */
typedef struct {
    int32_t width, height, ncomp, progressive;
    int32_t hs[4], vs[4];             /* sampling factors */
    int32_t bw[4], bh[4];             /* allocated blocks across / down (padded to MCUs) */
    int32_t rbw[4], rbh[4];           /* real blocks: ceil(component samples / 8) */
    int64_t comp_offset[4];           /* offset of the component's first coefficient, in int16 units */
    int64_t total_coefs;              /* int16 count of the whole buffer */
    uint16_t qt[4][64];               /* quantisation table of each COMPONENT, zigzag order */
} b200_jpeg_layout;

/* host: markers + Huffman decode (baseline and progressive).  *coefs is library-allocated. */
b200_status b200_jpeg_decode_coefficients(const uint8_t *in, size_t in_len, b200_jpeg_layout *layout, int16_t **coefs);
/* layout the encoder side of compress_in_memory would produce for an input layout + params */
b200_status b200_jpeg_output_layout(const b200_jpeg_layout *in_layout, const b200_params *params, b200_jpeg_layout *out_layout);
/* device: dequant -> IDCT -> chroma upsample -> downsample -> FDCT -> quantise -> zigzag, host buffers in/out
 * (H2D, kernels, D2H on an internal stream).  out_coefs must hold out_layout->total_coefs int16. */
b200_status b200_jpeg_requantize(const b200_jpeg_layout *in_layout, const int16_t *in_coefs,
                                 const b200_jpeg_layout *out_layout, int16_t *out_coefs);
/* host: entropy-code coefficients (optimised Huffman tables; progressive = mozjpeg-style 8-scan script) */
b200_status b200_jpeg_encode_coefficients(const b200_jpeg_layout *layout, const int16_t *coefs, int progressive,
                                          uint8_t **out, size_t *out_len);
/* device: the same encoder as b200_jpeg_encode_coefficients run on the GPU (statistics, optimal tables, bit packing, byte
 * stuffing as block-parallel kernels); output bytes are identical */
b200_status b200_jpeg_encode_coefficients_device(const b200_jpeg_layout *layout, const int16_t *coefs, int progressive,
                                                 uint8_t **out, size_t *out_len);
/* device: dequant + IDCT + fancy upsample to planar full-resolution native-space planes [ncomp][H][W] */
b200_status b200_jpeg_decode_planes(const b200_jpeg_layout *in_layout, const int16_t *in_coefs, uint8_t *planes);
/* mozjpeg table idx 3 scaled by jpeg_set_quality(q, FALSE); natural order */
void b200_jpeg_quant_table(int quality, int which, uint16_t out[64]);

/* ---- device-resident FULL path (bench "value": scan bytes in HBM -> scan bytes in HBM) ------------------
 * n baseline single-scan JPEGs of one shape: parsed and uploaded once at create; every run enqueues Huffman decode ->
 * dequant/IDCT/resample/FDCT/quantise -> Huffman encode (optimal tables, stuffing) for all of them, `group` images per launch
 * sequence, each group on its own stream, joined back into `cuda_stream`; no host wait inside run.  params as for
 * b200_compress_in_memory (jpeg_optimize = 1: the lossless transcode, no transform). */
typedef struct b200_jpeg_pipe b200_jpeg_pipe;
b200_status b200_jpeg_pipe_create(const uint8_t *const *in, const size_t *in_len, int n, const b200_params *params, int group, b200_jpeg_pipe **pipe);
/* which: 0 whole path, 1 entropy decode, 2 transform, 3 entropy encode (stage timing; 2 / 3 reuse the last whole run's data) */
b200_status b200_jpeg_pipe_run(b200_jpeg_pipe *p, void *cuda_stream, int which, int *launches);
/* after the caller has synchronised: out_sizes[n] = entropy-coded bytes per image; *not_settled = images the device decoder
 * would hand to the host decoder; *enc_retries = encoder back halves repeated because an output estimate was too small */
b200_status b200_jpeg_pipe_finish(b200_jpeg_pipe *p, size_t *out_sizes, int *not_settled, int *enc_retries);
/* the complete output file of image `index` (for parity checks); after finish */
b200_status b200_jpeg_pipe_fetch(b200_jpeg_pipe *p, int index, uint8_t **out, size_t *out_len);
/* one group alone on its stream, an event after every launch: writes up to `cap` records "name ms_per_launch launches\n" into
 * `text` (NUL-terminated); the per-kernel table behind bench.py's roofline object */
b200_status b200_jpeg_pipe_kernel_times(b200_jpeg_pipe *p, int iters, char *text, size_t cap);
void b200_jpeg_pipe_destroy(b200_jpeg_pipe *p);

/* ---- PNG stage entry points (lossless path: libcaesium png::lossless -> oxipng, compressor.rs:428,436-437) ------- */
/* Row-filter strategies (oxipng RowFilter order): 0 None 1 Sub 2 Up 3 Average 4 Paeth 5 MinSum 6 Entropy 7 Bigrams 8 BigEnt 9 Brute */
/* host: parse + inflate + unfilter.  *raw (library-allocated) = height * row_bytes packed samples.  info: width, height,
 * bit depth, colour type, bytes-per-pixel filter distance, row bytes. */
typedef struct { uint32_t width, height; int32_t bit_depth, color_type, bpp; uint64_t row_bytes; } b200_png_info;
b200_status b200_png_decode(const uint8_t *in, size_t in_len, b200_png_info *info, uint8_t **raw);
/* host: b200_png_decode followed by the lossless path's palette reduction (oxipng reduction::palette: an 8-bit RGB / RGBA image
 * with at most 256 distinct pixels becomes indexed).  *npalette = 0: nothing was reduced, info / raw are as decoded;
 * otherwise raw holds the packed indices (info->bit_depth = 8, 4, 2 or 1 bits each, rows MSB first and padded to bytes) and
 * palette_rgba (caller-allocated, 1024 bytes) the entries as R, G, B, A. */
b200_status b200_png_decode_reduced(const uint8_t *in, size_t in_len, b200_png_info *info, uint8_t **raw, uint8_t *palette_rgba, int *npalette);
/* device K6: filter raw[h][row_bytes] with `strategy` -> filtered[h][row_bytes + 1] (caller-allocated) */
b200_status b200_png_filter(const uint8_t *raw, int h, int row_bytes, int bpp, int strategy, uint8_t *filtered);
/* device K7: LZ77 tokens of a filtered stream (literal = byte; match = 0x80000000 | (len-3) << 16 | (dist-1)).
 * *tokens library-allocated; hist[316] = litlen (286) + dist (30) symbol counts. */
b200_status b200_png_lz77(const uint8_t *filtered, size_t n, int bpp, int stride, uint32_t **tokens, size_t *ntokens, uint32_t *hist);
/* host: DEFLATE (dynamic Huffman) + zlib framing of a token stream; adler = Adler-32 of the bytes the tokens expand to */
b200_status b200_png_deflate_tokens(const uint32_t *tokens, size_t ntokens, uint32_t adler, uint8_t **out, size_t *out_len);
/* the device side of b200_compress_in_memory on ONE PNG, timed: the file is parsed and inflated once, then the device pipeline
 * (un-filter, checksum, probes, K6 / K7 per strategy, DEFLATE coding, H2D / D2H around it) runs `iters` times with a CUDA event
 * after every launch.  text receives "name ms_per_launch launches\n" records (NUL-terminated, cap bytes); host decision waits between
 * launches are listed as host_wait and are NOT device time.  bench.py's device-resident figure for BASELINE configs[3]. */
b200_status b200_png_device_times(const uint8_t *in, size_t in_len, int level, int iters, char *text, size_t cap);
/* strategies tried for an optimisation level (returns the count; out[] holds up to 10) */
int b200_png_level_strategies(int level, int *out);

/* ---- WebP stage entry points (lossy VP8 key frame: caesium::convert_in_memory(.., WebP), compressor.rs:288-292) ---- */
/* device K8 + host writer: planar RGB [3][h][w] (host) -> a complete .webp file at `quality` (0..100).  levels / modes may
 * be NULL; otherwise they receive the per-macroblock stage output: levels [mbh*mbw][25][16] int16 (Y2, 16 Y, 4 U, 4 V in
 * zigzag order), modes [mbh*mbw][4] = {ymode, uvmode, skip, 0} with modes 0 DC, 1 TM, 2 V, 3 H; mbw = ceil(w/16). */
b200_status b200_webp_encode_rgb(const uint8_t *rgb, int w, int h, int quality, uint8_t **out, size_t *out_len,
                                 int16_t *levels, uint8_t *modes);
/* host: the prediction filter the alpha plane is coded with (0 none, 1 horizontal, 2 vertical, 3 gradient: lowest order-0 cost of the
 * residuals) and the residual plane (`filtered`, caller-allocated, width * height; a copy of the plane for filter 0) */
int b200_webp_alpha_filter(const uint8_t *alpha, int width, int height, uint8_t *filtered);
/* host: the ALPH chunk payload (header byte + VP8L image stream: WebP lossless bitstream, alpha in green, no transforms) of a
 * width x height (filtered) alpha plane given its LZ77 tokens in b200_png_lz77's format (bpp 1, stride = width) -- the alpha plane
 * libwebp's WebPEncodeRGBA writes next to the lossy frame (compressor.rs:288-292 on an image with transparency). */
b200_status b200_webp_alpha_chunk(const uint32_t *tokens, size_t ntokens, int width, int height, int filter, uint8_t **out, size_t *out_len);
/* host: RIFF / VP8X container with alpha from a simple lossy file (RIFF + one 'VP8 ' chunk) and an ALPH payload */
b200_status b200_webp_wrap_alpha(const uint8_t *simple_file, size_t file_len, const uint8_t *alph, size_t alph_len, int width, int height, uint8_t **out, size_t *out_len);
/* host: decode a still WebP to planar RGB [3][h][w] exactly as libwebp's WebPDecodeRGB does -- the front end of compress_in_memory /
 * convert_in_memory / compress_to_size_in_memory on WebP inputs: lossy (VP8 key frame) and lossless (VP8L) files; animation: code 3.
 * An alpha plane is dropped here; b200_webp_decode_rgba returns it as well (*alpha = NULL when every pixel is opaque).
 * *rgb / *alpha are library-allocated. */
b200_status b200_webp_decode(const uint8_t *in, size_t in_len, int *width, int *height, uint8_t **rgb);
b200_status b200_webp_decode_rgba(const uint8_t *in, size_t in_len, int *width, int *height, uint8_t **rgb, uint8_t **alpha);
/* diagnostics: bytes the WebP leg has copied device -> host since the library was loaded (modes, tallies and decision records per frame) */
unsigned long long b200_webp_d2h_bytes(void);
/* host only: boolean-code levels + modes (layout above) into a .webp file -- the entropy-coding half on its own.  A ymode of 4 (B_PRED)
 * needs sub-block modes and is refused here with B200_ERR_INVALID_ARGUMENT (b200_webp_write_levels_bpred writes it). */
b200_status b200_webp_write_levels(int w, int h, int quality, const int16_t *levels, const uint8_t *modes, uint8_t **out, size_t *out_len);
/* libwebp's quality -> quantiser index curve and the six dequantisation factors (y1 dc/ac, y2 dc/ac, uv dc/ac) it selects */
int b200_webp_qindex(int quality, int factors[6]);

#ifdef __cplusplus
}
#endif
#endif /* B200_CAESIUM_H */
