// GIF decoder (gif_host.cpp) under AddressSanitizer + UBSan: every mutated file is decoded to the end or refused, never read out of
// bounds.  Usage: fuzz_gif a.gif b.gif ...
#include <cstdio>
#include <cstdlib>
#include <random>
#include <string>
#include <vector>
#include "gif_host.h"
using namespace b200;
static std::vector<uint8_t> slurp(const char *p) { FILE *f = fopen(p, "rb"); std::vector<uint8_t> v; if (!f) return v; fseek(f, 0, SEEK_END); v.resize(ftell(f)); fseek(f, 0, SEEK_SET); if (fread(v.data(), 1, v.size(), f)) {} fclose(f); return v; }
int main(int argc, char **argv)
{
    std::mt19937 rng(12345);
    long ok = 0, bad = 0;
    for (int a = 1; a < argc; a++) {
        const std::vector<uint8_t> src = slurp(argv[a]);
        if (src.empty()) continue;
        for (int it = 0; it < 4000; it++) {
            std::vector<uint8_t> d = src;
            const int mode = rng() % 4;
            if (mode == 0) for (int k = 0; k < 1 + (int)(rng() % 6); k++) d[rng() % d.size()] = (uint8_t)rng();
            else if (mode == 1) d.resize(1 + rng() % d.size());
            else if (mode == 2) { const size_t i = rng() % d.size(); d.insert(d.begin() + i, (size_t)(1 + rng() % 40), (uint8_t)rng()); }
            else { for (int k = 0; k < 3; k++) { const size_t i = 13 + rng() % (d.size() > 14 ? d.size() - 13 : 1); if (i < d.size()) d[i] ^= (uint8_t)(1u << (rng() % 8)); } }
            // keep the logical screen sane so that a flipped header bit does not ask for gigabytes
            if (d.size() >= 10 && (long long)(d[6] | d[7] << 8) * (d[8] | d[9] << 8) > 4000000) continue;
            GifReader rd; std::string err;
            if (!rd.open(d.data(), d.size(), err)) { bad++; continue; }
            std::vector<uint32_t> canvas((size_t)rd.width * rd.height);
            int delay = 0, n = 0;
            while (rd.next(canvas.data(), delay, err)) n++;
            if (err.empty() && n == rd.frames) ok++; else bad++;
        }
    }
    printf("decoded %ld, refused %ld\n", ok, bad);
    return 0;
}
