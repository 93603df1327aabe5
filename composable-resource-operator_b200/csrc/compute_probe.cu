// compute_probe.cu — the SM compute probe (cro_probe_compute): every SM's tensor cores and ALUs against an exact answer.
#include "compute.hpp"
#include "sm_legs.hpp"

namespace cro {

namespace {
// What the per-SM driver (sm_legs.hpp) needs of the compute probe.  Legs: s8, bf16, e4m3 tensor legs; ffma, imad ALU
// legs.
struct ComputeProbe {
    using Opts = cro_compute_opts;
    using Result = cro_compute_result;
    using Sm = cro_compute_sm;
    using Fault = cro_compute_fault;
    using Args = ComputeArgs;
    using Tile = int32_t;
    static constexpr const char* kName = "compute";
    static constexpr uint32_t kLegs = CRO_COMPUTE_LEGS, kAllLegs = CRO_COMPUTE_ALL_LEGS, kMaxSms = CRO_COMPUTE_MAX_SMS;
    static constexpr uint32_t kRecords = CRO_COMPUTE_RECORDS;
    static constexpr int kAnswers = 2;      // CRO_COMPUTE_ANSWER_S8, _SMALL
    static constexpr uint64_t Device::*kCalls = &Device::compute_calls;
    static constexpr SeedSpace kSeeds = kSeedCompute;
    // Tensor legs: iterations per CTA when the caller gives none (DESIGN.md "The compute probe" for the measurement).
    static constexpr uint32_t kDefaultIterations = 256, kDefaultAluIterations = 4, kDefaultRounds = 4;
    static constexpr bool kAluLeg[CRO_COMPUTE_LEGS] = {false, false, false, true, true};

    static int elements(int) { return compute::kTile; }
    static void expected(int answer, uint64_t seed, int32_t* out) { compute::Expected(answer, seed, out); }
    static uint64_t fold(int, const int32_t* tile) { return compute::CtaFold(tile); }
    static int answer(uint32_t leg) {
        return leg == CRO_COMPUTE_LEG_S8 || leg == CRO_COMPUTE_LEG_IMAD ? CRO_COMPUTE_ANSWER_S8 : CRO_COMPUTE_ANSWER_SMALL;
    }
    static uint64_t ops(uint32_t) { return 2ull * CRO_COMPUTE_M * CRO_COMPUTE_N * CRO_COMPUTE_K; }
    static cudaError_t launch(uint32_t leg, const ComputeArgs& a, int grid, cudaStream_t st) { return launch_compute(leg, a, grid, st); }

    static std::string opts_error(const cro_compute_opts& o) {
        const uint32_t legs = o.legs ? o.legs : CRO_COMPUTE_ALL_LEGS;
        uint32_t iters[CRO_COMPUTE_LEGS];
        leg_iterations<ComputeProbe>(o, iters);
        const uint32_t max_rounds = o.max_rounds ? o.max_rounds : kDefaultRounds;
        if ((legs & ~CRO_COMPUTE_ALL_LEGS) || iters[0] > CRO_COMPUTE_MAX_ITERATIONS || iters[3] > CRO_COMPUTE_MAX_ALU_ITERATIONS ||
            max_rounds > CRO_COMPUTE_MAX_ROUNDS ||
            (o.test_inject_mask &&
             (o.test_inject_leg < 0 || o.test_inject_leg >= CRO_COMPUTE_LEGS || o.test_inject_sm < -1 ||
              o.test_inject_sm >= CRO_COMPUTE_MAX_SMS || o.test_inject_row < -1 || o.test_inject_row >= CRO_COMPUTE_M ||
              o.test_inject_col < -1 || o.test_inject_col >= CRO_COMPUTE_N || o.test_inject_iteration >= iters[o.test_inject_leg])))
            return "compute probe: legs must be CRO_COMPUTE_ALL_LEGS bits, iterations at most " +
                   std::to_string(CRO_COMPUTE_MAX_ITERATIONS) + ", alu_iterations at most " +
                   std::to_string(CRO_COMPUTE_MAX_ALU_ITERATIONS) + ", max_rounds at most " +
                   std::to_string(CRO_COMPUTE_MAX_ROUNDS) + ", and an injection must name a leg, an SM id below " +
                   std::to_string(CRO_COMPUTE_MAX_SMS) + " (or -1), a row, a column (or -1) and an iteration the leg runs";
        return "";
    }
};
}  // namespace

int ctx_probe_compute(cro_ctx* c, int idx, const cro_compute_opts& o, cro_compute_result* r, std::vector<cro_compute_sm>* sms,
                      std::vector<cro_compute_fault>* faults) {
    return probe_sm_legs<ComputeProbe>(c, idx, o, r, sms, faults);
}

int ctx_probe_compute_uuid(cro_ctx* c, const char* uuid, const cro_compute_opts& o, int deadline_ms, cro_compute_result* r,
                           std::vector<cro_compute_sm>* sms, std::vector<cro_compute_fault>* faults, int cap, uint64_t* helper_ns) {
    return probe_sm_legs_uuid<ComputeProbe>(c, uuid, o, deadline_ms, r, sms, faults, cap, helper_ns);
}

int classify_compute(uint32_t legs, const uint32_t* iterations, uint32_t grid, uint64_t k, const uint32_t* rounds,
                     const cro_sm_cta* ctas, const uint64_t* sm_bits, const uint64_t* claims, const cro_compute_fault* records,
                     cro_compute_result* r, std::vector<cro_compute_sm>* sms, std::vector<cro_compute_fault>* faults) {
    return classify_sm_legs<ComputeProbe>(legs, iterations, grid, k, rounds, ctas, sm_bits, claims, records, r, sms, faults);
}

}  // namespace cro
