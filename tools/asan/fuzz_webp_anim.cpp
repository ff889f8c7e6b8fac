// Animated WebP reader (webp_anim_host.cpp) and the host compositor under AddressSanitizer + UBSan: every mutated file is decoded
// to the end or refused, never read out of bounds.  Usage: fuzz_webp_anim a.webp b.webp ...
#include <cstdio>
#include <cstdlib>
#include <random>
#include <string>
#include <vector>
#include "webp_anim_host.h"
using namespace b200;
static std::vector<uint8_t> slurp(const char *p) { FILE *f = fopen(p, "rb"); std::vector<uint8_t> v; if (!f) return v; fseek(f, 0, SEEK_END); v.resize(ftell(f)); fseek(f, 0, SEEK_SET); if (fread(v.data(), 1, v.size(), f)) {} fclose(f); return v; }
int main(int argc, char **argv)
{
    std::mt19937 rng(12345);
    long ok = 0, bad = 0;
    for (int a = 1; a < argc; a++) {
        const std::vector<uint8_t> src = slurp(argv[a]);
        if (src.size() < 32) continue;
        for (int it = 0; it < 4000; it++) {
            std::vector<uint8_t> d = src;
            const int mode = rng() % 4;
            if (mode == 0) for (int k = 0; k < 1 + (int)(rng() % 6); k++) d[rng() % d.size()] = (uint8_t)rng();
            else if (mode == 1) d.resize(1 + rng() % d.size());
            else if (mode == 2) { const size_t i = rng() % d.size(); d.insert(d.begin() + i, (size_t)(1 + rng() % 40), (uint8_t)rng()); }
            else { for (int k = 0; k < 3; k++) { const size_t i = 12 + rng() % (d.size() - 12); d[i] ^= (uint8_t)(1u << (rng() % 8)); } }
            // keep the canvas sane so that a flipped VP8X bit does not ask for gigabytes of canvases
            if (d.size() >= 30 && (long long)(1 + (d[24] | d[25] << 8 | d[26] << 16)) * (1 + (d[27] | d[28] << 8 | d[29] << 16)) > 1000000) continue;
            WebpAnimReader rd; std::string err;
            std::vector<uint32_t> canvases, durations;
            if (webp_anim_decode_all(d.data(), d.size(), rd, canvases, durations, err)) ok++; else bad++;
        }
    }
    printf("decoded %ld, refused %ld\n", ok, bad);
    return 0;
}
