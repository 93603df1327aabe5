// warpmma_probe.cu — the SM warp-MMA probe (cro_probe_warpmma): every SM's mma.sync tensor-core path and its ldmatrix,
// stmatrix and movmatrix fragment moves against an exact answer; its expected answers, computed on the host; and its
// helper form.
#include "compute.hpp"
#include "sm_legs.hpp"
#include "warpmma_kernels.cuh"

namespace cro {

namespace warpmma {

namespace {
constexpr uint32_t M = CRO_WARPMMA_M, N = CRO_WARPMMA_N;

// The MOVE answer: the source tile S (S[r][c] halfword e % 4 of pattern_word(seed, e / 4), e = r * N + c) transposed
// in each 8 x 8 block, E[8a + i][8b + j] = S[8a + j][8b + i].
void move_tile(uint64_t seed, int32_t* out) {
    std::vector<uint16_t> s((size_t)M * N);
    for (uint32_t w = 0; w < M * N / 4; ++w) {
        const uint64_t v = pattern_word(seed, w);
        for (uint32_t h = 0; h < 4; ++h) s[4 * w + h] = (uint16_t)(v >> (16 * h));
    }
    for (uint32_t r = 0; r < M; ++r)
        for (uint32_t c = 0; c < N; ++c) out[r * N + c] = s[((r & ~7u) | (c & 7u)) * N + ((c & ~7u) | (r & 7u))];
}

// The precision probe's answer `answer` narrowed to int32 (every value is at most 4096 in magnitude).
void precision_tile(int answer, uint64_t seed, int32_t* out) {
    std::vector<int64_t> wide((size_t)M * N);
    precision::Expected(answer, seed, wide.data());
    for (size_t e = 0; e < wide.size(); ++e) out[e] = (int32_t)wide[e];
}
}  // namespace

const int kLegAnswer[CRO_WARPMMA_LEGS] = {CRO_WARPMMA_ANSWER_S8,       CRO_WARPMMA_ANSWER_SMALL,  CRO_WARPMMA_ANSWER_SMALL,
                                          CRO_WARPMMA_ANSWER_SMALL128, CRO_WARPMMA_ANSWER_NARROW, CRO_WARPMMA_ANSWER_MOVE};

int Expected(int answer, uint64_t seed, int32_t* out) {
    if (answer < 0 || answer >= CRO_WARPMMA_ANSWERS || !out) return CRO_ERR_INVALID_ARG;
    switch (answer) {
        case CRO_WARPMMA_ANSWER_S8: return compute::Expected(CRO_COMPUTE_ANSWER_S8, seed, out);
        case CRO_WARPMMA_ANSWER_SMALL: return compute::Expected(CRO_COMPUTE_ANSWER_SMALL, seed, out);
        case CRO_WARPMMA_ANSWER_SMALL128: precision_tile(CRO_PRECISION_ANSWER_SMALL128, seed, out); break;
        case CRO_WARPMMA_ANSWER_NARROW: precision_tile(CRO_PRECISION_ANSWER_NARROW, seed, out); break;
        default: move_tile(seed, out);
    }
    return CRO_OK;
}

// The sum over every element e of an answer's tile of canon(expected value in its legs' type) * (2e + 1) (mod 2^64):
// int32 bits for S8 and the raw 16 bits for MOVE; the f32 and f16 answers are encoded as the precision probe's.
uint64_t TileFold(int answer, const int32_t* tile) {
    if (answer == CRO_WARPMMA_ANSWER_S8 || answer == CRO_WARPMMA_ANSWER_MOVE) {
        uint64_t f = 0;
        for (uint64_t e = 0; e < (uint64_t)M * N; ++e) f += (uint64_t)(uint32_t)tile[e] * (2 * e + 1);
        return f;
    }
    const std::vector<int64_t> wide(tile, tile + (size_t)M * N);
    return precision::TileFold(answer == CRO_WARPMMA_ANSWER_NARROW ? CRO_PRECISION_ANSWER_NARROW : CRO_PRECISION_ANSWER_SMALL,
                               wide.data());
}

}  // namespace warpmma

namespace {
constexpr unsigned kElementBits[CRO_WARPMMA_LEGS] = {32, 32, 32, 32, 16, 16};

// 16-byte K segments of an A row: the k-steps a fragment-address substitution may name.
uint32_t k_steps(uint32_t leg) {
    return leg == CRO_WARPMMA_LEG_S8 ? CRO_WARPMMA_K / 16 : leg == CRO_WARPMMA_LEG_TF32 ? CRO_WARPMMA_TF32_K * 4 / 16 : CRO_WARPMMA_K * 2 / 16;
}

// What the per-SM driver (sm_legs.hpp) needs of the warp-MMA probe.
struct WarpMmaProbe {
    using Opts = cro_warpmma_opts;
    using Result = cro_warpmma_result;
    using Sm = cro_warpmma_sm;
    using Fault = cro_warpmma_fault;
    using Args = WarpMmaArgs;
    using Tile = int32_t;
    static constexpr const char* kName = "warpmma";
    static constexpr const cro_wire& kWire = cro_wire_warpmma;
    static constexpr uint32_t kLegs = CRO_WARPMMA_LEGS, kAllLegs = CRO_WARPMMA_ALL_LEGS, kMaxSms = CRO_WARPMMA_MAX_SMS;
    static constexpr uint32_t kRecords = CRO_WARPMMA_RECORDS;
    static constexpr int kAnswers = CRO_WARPMMA_ANSWERS;
    static constexpr uint64_t Device::*kCalls = &Device::warpmma_calls;
    static constexpr SeedSpace kSeeds = kSeedWarpMma;
    // Iterations per CTA when the caller gives none: the six legs' device time near the sparse probe's default (DESIGN.md
    // "The warp-MMA probe" for the measurement).
    static constexpr uint32_t kDefaultIterations = 128, kDefaultRounds = 4;
    static constexpr bool kAluLeg[CRO_WARPMMA_LEGS] = {false, false, false, false, false, false};

    static int elements(int) { return CRO_WARPMMA_M * CRO_WARPMMA_N; }
    static void expected(int answer, uint64_t seed, int32_t* out) { warpmma::Expected(answer, seed, out); }
    static uint64_t fold(int answer, const int32_t* tile) { return warpmma::TileFold(answer, tile); }
    static int answer(uint32_t leg) { return warpmma::kLegAnswer[leg]; }
    // 2 M N K; MOVE: the M N elements it moves
    static uint64_t ops(uint32_t leg) {
        if (leg == CRO_WARPMMA_LEG_MOVE) return (uint64_t)CRO_WARPMMA_M * CRO_WARPMMA_N;
        return 2ull * CRO_WARPMMA_M * CRO_WARPMMA_N * (leg == CRO_WARPMMA_LEG_TF32 ? CRO_WARPMMA_TF32_K : CRO_WARPMMA_K);
    }
    static cudaError_t launch(uint32_t leg, const WarpMmaArgs& a, int grid, cudaStream_t st) { return launch_warpmma(leg, a, grid, st); }
    static void test_args(const cro_warpmma_opts& o, uint32_t leg, WarpMmaArgs* a) {
        a->addr = (o.test_addr && (uint32_t)o.test_addr_leg == leg) ? 1u : 0u;
        a->addr_sm = o.test_addr_sm;
        a->addr_iter = o.test_addr_iteration;
        a->addr_row = o.test_addr_row;
        a->addr_kstep = o.test_addr_kstep;
    }

    static std::string opts_error(const cro_warpmma_opts& o) {
        const uint32_t legs = o.legs ? o.legs : CRO_WARPMMA_ALL_LEGS;
        const uint32_t iters = o.iterations ? o.iterations : kDefaultIterations;
        const uint32_t max_rounds = o.max_rounds ? o.max_rounds : kDefaultRounds;
        const int l = o.test_inject_leg, al = o.test_addr_leg;
        if ((legs & ~CRO_WARPMMA_ALL_LEGS) || iters > CRO_WARPMMA_MAX_ITERATIONS || max_rounds > CRO_WARPMMA_MAX_ROUNDS ||
            (o.test_inject_mask &&
             (l < 0 || l >= CRO_WARPMMA_LEGS || o.test_inject_sm < -1 || o.test_inject_sm >= CRO_WARPMMA_MAX_SMS ||
              o.test_inject_row < -1 || o.test_inject_row >= CRO_WARPMMA_M || o.test_inject_col < -1 ||
              o.test_inject_col >= CRO_WARPMMA_N || o.test_inject_iteration >= iters ||
              (o.test_inject_mask >> kElementBits[l]))) ||
            o.test_addr > 1 ||
            (o.test_addr &&
             (al < 0 || al >= CRO_WARPMMA_LEG_MOVE || o.test_addr_sm < -1 || o.test_addr_sm >= CRO_WARPMMA_MAX_SMS ||
              o.test_addr_iteration >= iters || o.test_addr_row >= CRO_WARPMMA_M || o.test_addr_kstep >= k_steps((uint32_t)al))))
            return "warpmma probe: legs must be CRO_WARPMMA_ALL_LEGS bits, iterations at most " +
                   std::to_string(CRO_WARPMMA_MAX_ITERATIONS) + ", max_rounds at most " + std::to_string(CRO_WARPMMA_MAX_ROUNDS) +
                   ", an injection must name a leg, an SM id below " + std::to_string(CRO_WARPMMA_MAX_SMS) +
                   " (or -1), a row, a column (or -1), an iteration the leg runs and a mask no wider than the leg's value, " +
                   "and a fragment-address substitution (test_addr 0 or 1) an arithmetic leg, an SM id (or -1), an " +
                   "iteration the leg runs, a row and a k-step of the leg";
        return "";
    }
};
}  // namespace

int ctx_probe_warpmma(cro_ctx* c, int idx, const cro_warpmma_opts& o, cro_warpmma_result* r, std::vector<cro_warpmma_sm>* sms,
                      std::vector<cro_warpmma_fault>* faults) {
    return probe_sm_legs<WarpMmaProbe>(c, idx, o, r, sms, faults);
}

int ctx_probe_warpmma_uuid(cro_ctx* c, const char* uuid, const cro_warpmma_opts& o, int deadline_ms, cro_warpmma_result* r,
                           std::vector<cro_warpmma_sm>* sms, std::vector<cro_warpmma_fault>* faults, int cap, uint64_t* helper_ns) {
    return probe_sm_legs_uuid<WarpMmaProbe>(c, uuid, o, deadline_ms, r, sms, faults, cap, helper_ns);
}

int classify_warpmma(uint32_t legs, const uint32_t* iterations, uint32_t grid, uint64_t k, const uint32_t* rounds,
                     const cro_sm_cta* ctas, const uint64_t* sm_bits, const uint64_t* claims, const cro_warpmma_fault* records,
                     cro_warpmma_result* r, std::vector<cro_warpmma_sm>* sms, std::vector<cro_warpmma_fault>* faults) {
    return classify_sm_legs<WarpMmaProbe>(legs, iterations, grid, k, rounds, ctas, sm_bits, claims, records, r, sms, faults);
}

}  // namespace cro
