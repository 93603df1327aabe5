// xlane_probe.cu — the cross-lane probe (cro_probe_xlane, cro_probe_xlane_uuid): every SM's shuffle, vote, match,
// warp-reduce and shared-atomic units checked op by op on every lane, one launch per leg.
#include "lane_report.hpp"
#include "xlane_kernels.cuh"

namespace cro {

namespace {
// What every CTA's fold of a leg must be: the last iteration's expected results over every warp, lane and op.
void closed_form(uint64_t seed, uint32_t iterations, uint32_t legs, cro_xlane_result* r) {
    std::vector<uint64_t> e((size_t)CRO_XLANE_MAX_OPS * 32);
    for (unsigned leg = 0; leg < CRO_XLANE_LEGS; ++leg) {
        if (!(legs >> leg & 1u)) continue;
        uint64_t x = 0, s = 0, w = 0;
        for (unsigned warp = 0; warp < CRO_XLANE_WARPS; ++warp) {
            xlane_expected(leg, seed, iterations - 1, warp, e.data());
            for (uint64_t op = 0; op < xlane::kOps[leg]; ++op)
                for (unsigned l = 0; l < 32; ++l) {
                    const uint64_t v = e[op * 32 + l];
                    x ^= v;
                    s += v;
                    w += v * (2 * op + 1);
                }
        }
        r->expect[leg][0] = x;
        r->expect[leg][1] = s;
        r->expect[leg][2] = w;
    }
}

// What the lane probes' host driver (lane_report.hpp) needs of the cross-lane probe.  The device computes every
// expected value from the seed, so there are no tables.
struct XlaneProbe {
    using Opts = cro_xlane_opts;
    using Result = cro_xlane_result;
    using Sm = cro_xlane_sm;
    using Fault = cro_xlane_fault;
    using Thread = cro_xlane_thread;
    using Cta = cro_xlane_cta;
    using Args = XlaneArgs;
    struct Tables {};
    static constexpr unsigned kLegs = CRO_XLANE_LEGS, kAllLegs = CRO_XLANE_ALL_LEGS, kThreads = CRO_XLANE_THREADS,
                              kThreadRecs = CRO_XLANE_THREAD_RECORDS, kRecords = CRO_XLANE_RECORDS, kMaxSms = CRO_XLANE_MAX_SMS,
                              kMaxIterations = CRO_XLANE_MAX_ITERATIONS, kMaxRounds = CRO_XLANE_MAX_ROUNDS,
                              kPersistent = CRO_XLANE_PERSISTENT, kIntermittent = CRO_XLANE_INTERMITTENT, kNone = CRO_XLANE_NONE,
                              kSm = CRO_XLANE_SM, kAll = CRO_XLANE_ALL;
    static constexpr const char* kName = "cross-lane";
    static constexpr const char* kId = "xlane";
    static constexpr const cro_wire& kWire = cro_wire_xlane;
    static constexpr uint64_t Device::*kCalls = &Device::xlane_calls;
    static constexpr SeedSpace kSeeds = kSeedXlane;
    // Iterations per CTA and leg, and launches per leg, when the caller gives none.  On an H100 80GB HBM3 at a 700 W
    // limit (profiles/h100_700w_xlane_rate.jsonl) one iteration of the five legs takes 1.57 ms and one launch per leg
    // covers all 132 SMs, so 3 iterations cost about the SRAM and register-file probes' 5 ms (DESIGN.md "The cross-lane
    // probe").
    static constexpr uint32_t kDefaultIterations = 3, kDefaultRounds = 4;
    static constexpr unsigned kBlobs = 0;

    static unsigned ops(unsigned leg) { return xlane::kOps[leg]; }
    static std::string opts_error(const cro_xlane_opts& o) { return xlane_opts_error(o); }
    static cudaError_t plan(int device, unsigned leg) { return xlane_plan(device, leg); }
    static int grids(cro_ctx*, const cro_xlane_opts&, uint32_t, int sm_count, int (&grid)[kLegs]) {
        std::fill(grid, grid + kLegs, sm_count);
        return CRO_OK;
    }
    static cudaError_t launch(const cro_xlane_opts&, unsigned leg, const XlaneArgs& a, int grid, cudaStream_t st) {
        return launch_xlane(leg, a, grid, st);
    }
    static void open(const cro_xlane_opts&, cro_xlane_result* r, Tables&, bool) { closed_form(r->seed, r->iterations, r->legs, r); }
    static std::array<LaneBlob, kBlobs> blobs(const Tables&, unsigned) { return {}; }
    static void args(const cro_xlane_opts&, const cro_xlane_result& r, unsigned, const std::array<const void*, kBlobs>&,
                     XlaneArgs* a) {
        a->seed = r.seed;
    }
    static bool no_new_sm_ends(unsigned) { return false; }
    static int close(cro_xlane_result* r, LaneTally<XlaneProbe>& t, std::vector<cro_xlane_sm>* sms,
                     std::vector<cro_xlane_fault>* faults) {
        return close_lane_call<XlaneProbe>(r, t, sms, faults);
    }
    static void keep(cro_xlane_result*, const cro_xlane_result&) {}
};
}  // namespace

void xlane_expected(unsigned leg, uint64_t seed, uint32_t iteration, unsigned warp, uint64_t* out) {
    xlane::expected(leg, seed + (uint64_t)iteration * kNonceStride, warp, reinterpret_cast<xlane::u64*>(out));
}

std::string xlane_opts_error(const cro_xlane_opts& o) {
    const unsigned kind = o.test_inject_op / xlane::kAtomsShapes;
    const bool atoms_order =
        o.test_inject_mask && o.test_inject_leg == CRO_XLANE_LEG_ATOMS && (kind == xlane::kAtInc || kind == xlane::kAtDec);
    if (!lane_opts_ok<XlaneProbe>(o) || atoms_order)
        return "cross-lane probe: iterations at most " + std::to_string(CRO_XLANE_MAX_ITERATIONS) + ", legs at most 0x1F, max_rounds at most " +
               std::to_string(CRO_XLANE_MAX_ROUNDS) + ", deadline_ms not negative, and an injection must name a leg the call runs, an SM "
               "id below " + std::to_string(CRO_XLANE_MAX_SMS) + ", a warp below 8 and a lane below 32 (each or -1), an op of the "
               "leg (not ATOMS inc or dec) and an iteration the call runs";
    return "";
}

int ctx_probe_xlane(cro_ctx* c, int idx, const cro_xlane_opts& o, cro_xlane_result* r, std::vector<cro_xlane_sm>* sms,
                    std::vector<cro_xlane_fault>* faults) {
    return probe_lane_legs<XlaneProbe>(c, idx, o, r, sms, faults);
}

int classify_xlane(uint32_t legs, uint32_t iterations, uint64_t seed, uint32_t sm_count, uint64_t k, uint32_t rounds,
                   const cro_xlane_cta* ctas, const cro_xlane_thread* threads, const cro_xlane_fault* records,
                   cro_xlane_result* r, std::vector<cro_xlane_sm>* sms, std::vector<cro_xlane_fault>* faults) {
    cro_xlane_opts o{};
    o.legs = legs;
    o.iterations = iterations;
    return classify_lane_legs<XlaneProbe>(o, seed, sm_count, k, rounds, ctas, threads, records, r, sms, faults);
}

int ctx_probe_xlane_uuid(cro_ctx* c, const char* uuid, const cro_xlane_opts& o, cro_xlane_result* r,
                         std::vector<cro_xlane_sm>* sms, std::vector<cro_xlane_fault>* faults, int cap) {
    return probe_lane_legs_uuid<XlaneProbe>(c, uuid, o, r, sms, faults, cap);
}

}  // namespace cro
