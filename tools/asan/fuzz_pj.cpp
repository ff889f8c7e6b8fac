#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <string>
#include <vector>
#include "png_host.h"
#include "jpeg_host.h"
using namespace b200;
bool b200::png_interlaced() { return true; }          // the C ABI's switch (api.cpp): Adam7 files are fuzzed too
static std::vector<uint8_t> slurp(const char *p) { FILE *f = fopen(p, "rb"); std::vector<uint8_t> v; if (!f) return v; fseek(f, 0, SEEK_END); v.resize(ftell(f)); fseek(f, 0, SEEK_SET); if (fread(v.data(), 1, v.size(), f)) {} fclose(f); return v; }
int main(int argc, char **argv)
{
    std::mt19937 rng(777);
    long ok = 0, bad = 0;
    for (int a = 1; a < argc; a++) {
        const std::vector<uint8_t> src = slurp(argv[a]);
        if (src.size() < 16) continue;
        const bool is_png = !memcmp(src.data(), "\x89PNG", 4);
        for (int it = 0; it < 3000; it++) {
            std::vector<uint8_t> d = src;
            const int mode = rng() % 4;
            if (mode == 0) for (int k = 0; k < 1 + (int)(rng() % 6); k++) d[rng() % d.size()] = (uint8_t)rng();
            else if (mode == 1) d.resize(1 + rng() % d.size());
            else if (mode == 2) { const size_t i = rng() % d.size(); d.insert(d.begin() + i, (size_t)(1 + rng() % 40), (uint8_t)rng()); }
            else { for (int k = 0; k < 3; k++) { const size_t i = 40 + rng() % (d.size() > 41 ? d.size() - 40 : 1); if (i < d.size()) d[i] ^= (uint8_t)(1u << (rng() % 8)); } }
            std::string err;
            if (is_png) {
                PngInfo info; PngIdat idat;
                if (!png_parse_chunks(d.data(), d.size(), false, info, idat, err)) { bad++; continue; }
                const unsigned long long nin = png_inflated_size(info);
                if (nin > 50000000ull) { bad++; continue; }
                // the product's shape: inflate into a fixed buffer of nin + 4096 (+ 64) bytes
                std::vector<uint8_t> buf(nin + 4096 + 64); size_t got = 0; uint32_t ad = 0;
                if (!zlib_inflate_to(idat.p, idat.n, buf.data(), buf.size(), nin, &got, &ad, err)) { bad++; }
                std::vector<uint8_t> raw; PngInfo i2;
                if (png_decode(d.data(), d.size(), false, i2, raw, err)) { ok++; png_reduce_palette(i2, raw); } else bad++;
            } else {
                JpegReader rd(d.data(), d.size());
                if (!rd.read_header(err)) { bad++; continue; }
                if (rd.geom().total_coefs > 60000000) { bad++; continue; }
                std::vector<int16_t> c((size_t)rd.geom().total_coefs + 64);
                JpegReader::DeviceScan ds; rd.device_decodable(ds); rd.device_decodable(ds, true);
                if (rd.decode(c.data(), err)) ok++; else bad++;
            }
        }
    }
    printf("decoded %ld, refused %ld\n", ok, bad);
    return 0;
}
