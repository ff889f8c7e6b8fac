// The buffer growth rules of dev_buffer.h, compiled on the CPU: grow_bytes over an array of requests.
#include <cstddef>
#include <cstdint>
#include <cstring>
#define B200_GROW_RULES_ONLY
#include "../../caesium-clt_b200/csrc/dev_buffer.h"

using b200::Grow;

static_assert(b200::grow_bytes(1, Grow::Slot) == 65536, "grow_bytes is usable in constant expressions");

extern "C" int emul_grow_bytes(const char *rule, const uint64_t *need, uint64_t *out, size_t n)
{
    struct { const char *name; Grow rule; } rules[] = {{"exact", Grow::Exact}, {"slot", Grow::Slot}, {"pow2", Grow::Pow2},
                                                      {"pow2_quarter", Grow::Pow2Quarter}, {"pow2_half", Grow::Pow2Half}};
    for (const auto &r : rules) {
        if (strcmp(r.name, rule)) continue;
        for (size_t i = 0; i < n; i++) out[i] = b200::grow_bytes((size_t)need[i], r.rule);
        return 0;
    }
    return -1;
}
