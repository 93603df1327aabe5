// env.cpp — validated CRO_* knobs (see env.hpp; wording after
// internal/controller/composableresource_adapter.go:44).
#include "env.hpp"

#include <cstdlib>
#include <cstring>

namespace cro {
namespace env {

namespace {
// name, lo, hi, default, multiple_of, what
const Knob kKnobs[] = {
    {"CRO_FILL_WAVES", 1, 1024, 64, 0, "CTA waves of the fill kernel"},
    {"CRO_READ_WAVES", 1, 1024, 1, 0, "CTA waves of the LDG read kernels"},
    {"CRO_COPY_WAVES", 1, 1024, 128, 0, "CTA waves of the LDG copy kernel"},
    {"CRO_TMA_READ_TILE", 1024, 114688, 32768, 16, "bytes per TMA bulk load of the read ring"},
    {"CRO_TMA_READ_STAGES", 2, 16, 4, 0, "ring depth of the read kernel"},
    {"CRO_TMA_READ_THREADS", 64, 1024, 1024, 32, "1 producer warp + consumer warps"},
    {"CRO_TMA_READ_CHUNK", 1, 4096, 1, 0, "tiles claimed per atomic"},
    {"CRO_TMA_READ_HINT", 0, 1, 0, 0, "1 = L2 evict_first on the bulk loads"},
    {"CRO_TMA_READ_DYN", 0, 1, 1, 0, "1 = dynamic tile claims"},
    {"CRO_TMA_READ_WAVES", 1, 64, 1, 0, "CTAs per SM slot"},
    {"CRO_TMA_COPY_TILE", 1024, 114688, 32768, 16, "bytes per TMA bulk copy of the copy ring"},
    {"CRO_TMA_COPY_STAGES", 2, 16, 4, 0, "ring depth of the copy kernel"},
    {"CRO_TMA_COPY_CHUNK", 1, 4096, 1, 0, "tiles claimed per atomic"},
    {"CRO_TMA_COPY_HINT", 0, 7, 0, 0, "bit0 evict_first loads, bit1 evict_first stores, bit2 evict_last stores"},
    {"CRO_TMA_COPY_DYN", 0, 1, 1, 0, "1 = dynamic tile claims"},
    {"CRO_TMA_COPY_WAVES", 1, 64, 1, 0, "CTAs per SM slot"},
    {"CRO_FUSED_TILE", 1024, 114688, 32768, 16, "bytes per tile of the checksumming copy"},
    {"CRO_FUSED_STAGES", 2, 16, 4, 0, "ring depth of the checksumming copy"},
    {"CRO_FUSED_CHUNK", 1, 4096, 1, 0, "tiles claimed per atomic"},
    {"CRO_FUSED_THREADS", 64, 1024, 160, 32, "1 producer warp + consumer warps of the checksumming copy"},
    {"CRO_READ_VARIANT", 0, 3, 0, 0, "CRO_READ_* forced for every sweep (0 = by size)"},
    {"CRO_COPY_VARIANT", 0, 3, 0, 0, "CRO_COPY_* forced (0 = checksumming TMA copy)"},
    {"CRO_USE_GRAPH", 0, 1, 1, 0, "replay the probe as one CUDA graph"},
    {"CRO_EXPECT_OVERLAP", 0, 1, 1, 0, "closed-form generator on a side stream under the copy sweeps"},
    {"CRO_EXPECT_CTAS", 1, 8, 1, 0, "CTAs per SM of the closed-form generator (it must leave room for the copy's CTA)"},
    {"CRO_CARVEOUT_FILL", 0, 1, 1, 0, "the fill kernel asks for the largest shared memory too (it runs beside a generator in cro_probe_all)"},
    {"CRO_P2P_UNIDIR", 0, 1, 0, 0, "measurement only: one direction per NVLink pair"},
    {"CRO_P2P_READ_VARIANT", 1, 3, 2, 0, "kernel of the NVLink read leg"},
    {"CRO_P2P_WRITE_VARIANT", 1, 3, 3, 0, "kernel of the NVLink push leg"},
    {"CRO_NVTX", 0, 1, 1, 0, "NVTX ranges around the probe phases"},
    {"CRO_HELPER_TIMEOUT_MS", 100, 600000, 30000, 0, "deadline of the out-of-process probe helper"},
};
constexpr int kN = (int)(sizeof kKnobs / sizeof kKnobs[0]);

int index_of(const char* name) {
    for (int i = 0; i < kN; ++i)
        if (strcmp(kKnobs[i].name, name) == 0) return i;
    return -1;
}
}  // namespace

const Knob* table(int* n_out) {
    if (n_out) *n_out = kN;
    return kKnobs;
}

std::string refusal(const char* name, const std::string& text) {
    return std::string("the env variable ") + name + " has an invalid value: '" + text + "'";
}

bool parse(const Knob& k, const char* text, unsigned* out, std::string* err) {
    auto bad = [&]() {
        if (err) *err = refusal(k.name, text ? text : "");
        return false;
    };
    if (!text || !*text) {
        *out = k.dflt;
        return true;
    }
    unsigned long long v = 0;
    size_t n = 0;
    for (const char* p = text; *p; ++p, ++n) {
        if (*p < '0' || *p > '9' || n > 10) return bad();
        v = v * 10 + (unsigned)(*p - '0');
    }
    if (v < k.lo || v > k.hi) return bad();
    if (k.multiple_of && v % k.multiple_of != 0) return bad();
    *out = (unsigned)v;
    return true;
}

Values::Values() {
    static_assert(kN <= kMax, "Values::kMax is smaller than the knob table");
    for (int i = 0; i < kN; ++i) v_[i] = kKnobs[i].dflt;
}

unsigned Values::get(const char* name) const {
    const int i = index_of(name);
    return i < 0 ? 0u : v_[i];
}

bool read(Values* out, std::string* err) {
    Values fresh;
    for (int i = 0; i < kN; ++i)
        if (!parse(kKnobs[i], getenv(kKnobs[i].name), &fresh.v_[i], err)) return false;
    // the ring must fit the shared memory a CTA may own, next to the ring kernels' own
    const char* rings[3][2] = {{"CRO_TMA_READ_TILE", "CRO_TMA_READ_STAGES"}, {"CRO_TMA_COPY_TILE", "CRO_TMA_COPY_STAGES"},
                               {"CRO_FUSED_TILE", "CRO_FUSED_STAGES"}};
    for (auto& r : rings) {
        if ((unsigned long long)fresh.get(r[0]) * fresh.get(r[1]) > kRingMaxBytes) {
            const char* v = getenv(r[0]);
            if (err) *err = refusal(r[0], v ? v : "");
            return false;
        }
    }
    *out = fresh;
    return true;
}

}  // namespace env
}  // namespace cro
