// sparse_probe.cu — the SM sparse probe (cro_probe_sparse): every SM's 2:4 structured-sparsity tensor cores against an
// exact answer; its expected answers, computed on the host; and its helper form.
#include "sm_legs.hpp"
#include "sparse_kernels.cuh"

namespace cro {

namespace sparse {

namespace {
struct Shape {
    uint32_t k, g, p;       // logical K, K positions per group, legal pairs
    bool s8;                // s8 reading (otherwise small-int)
};
constexpr Shape kShape[CRO_SPARSE_ANSWERS] = {{CRO_SPARSE_K, 4, 6, true},
                                              {CRO_SPARSE_K, 4, 6, false},
                                              {CRO_SPARSE_K16, 4, 6, false},
                                              {CRO_SPARSE_TF32_K, 2, 2, false}};
// The kept K positions of each pair, in pair order (include/croprobe.h).
constexpr uint32_t kPair6[6][2] = {{0, 1}, {0, 2}, {0, 3}, {1, 2}, {1, 3}, {2, 3}};
}  // namespace

const int kLegAnswer[CRO_SPARSE_LEGS] = {CRO_SPARSE_ANSWER_S8,       CRO_SPARSE_ANSWER_SMALL,    CRO_SPARSE_ANSWER_SMALL,
                                         CRO_SPARSE_ANSWER_SMALL256, CRO_SPARSE_ANSWER_SMALL256, CRO_SPARSE_ANSWER_SMALL128};

uint32_t Groups(int answer) { return kShape[answer].k / kShape[answer].g; }

namespace {
// D = A * B over the kept values, each product in int16 (at most 2^14 in magnitude) and summed in T: int16 holds every
// small-int partial sum (at most 4096), int32 every s8 one (at most 2^22).  Both vectorise.
template <class T>
void multiply(const Shape& s, uint64_t seed, int32_t* out) {
    constexpr uint32_t M = CRO_SPARSE_M, N = CRO_SPARSE_N;
    const uint32_t KC = s.k / 2, groups = s.k / s.g, blocks = (groups + s.p - 1) / s.p, kept = s.g == 4 ? 2 : 1;
    // every byte of the operands, one pattern word per eight (byte e: byte e mod 8 of pattern_word(seed, e / 8))
    std::vector<uint8_t> bytes(((size_t)M * KC + (size_t)s.k * N + (size_t)M * blocks + 7) & ~(size_t)7);
    for (size_t w = 0; w < bytes.size() / 8; ++w) {
        const uint64_t v = pattern_word(seed, w);
        for (int b = 0; b < 8; ++b) bytes[8 * w + b] = (uint8_t)(v >> (8 * b));
    }
    auto value = [&](size_t e) { return s.s8 ? (int32_t)(int8_t)bytes[e] : (int32_t)(bytes[e] & 7u) - 4; };
    std::vector<int16_t> b((size_t)s.k * N);        // B[k][n]
    for (size_t e = 0; e < b.size(); ++e) b[e] = (int16_t)value((size_t)M * KC + e);
    const uint8_t* rot = bytes.data() + (size_t)M * KC + (size_t)s.k * N;
    std::vector<T> row(N);
    for (uint32_t m = 0; m < M; ++m) {
        std::fill(row.begin(), row.end(), (T)0);
        for (uint32_t g = 0; g < groups; ++g) {
            const uint32_t p = (g + rot[m * blocks + g / s.p]) % s.p;
            for (uint32_t j = 0; j < kept; ++j) {
                int32_t x = value((size_t)m * KC + kept * g + j);
                x = s.s8 ? (x ? x : 1) : x + (x >= 0);          // a kept value is never 0
                const int16_t t = (int16_t)x;
                const int16_t* bk = b.data() + (size_t)(s.g * g + (s.g == 4 ? kPair6[p][j] : p)) * N;
                for (uint32_t n = 0; n < N; ++n) row[n] = (T)(row[n] + (int16_t)(t * bk[n]));
            }
        }
        for (uint32_t n = 0; n < N; ++n) out[(size_t)m * N + n] = row[n];
    }
}
}  // namespace

int Expected(int answer, uint64_t seed, int32_t* out) {
    if (answer < 0 || answer >= CRO_SPARSE_ANSWERS || !out) return CRO_ERR_INVALID_ARG;
    if (kShape[answer].s8) multiply<int32_t>(kShape[answer], seed, out);
    else multiply<int16_t>(kShape[answer], seed, out);
    return CRO_OK;
}

// The sum over every element e of an answer's tile of canon(expected value's 32 bits) * (2e + 1) (mod 2^64): int32
// bits for the s8 answer, f32 bits otherwise (an integer's f32 is never -0).
uint64_t TileFold(int answer, const int32_t* tile) {
    uint64_t f = 0;
    for (uint64_t e = 0; e < (uint64_t)CRO_SPARSE_M * CRO_SPARSE_N; ++e) {
        uint32_t bits;
        if (answer == CRO_SPARSE_ANSWER_S8) {
            bits = (uint32_t)tile[e];
        } else {
            const float x = (float)tile[e];
            memcpy(&bits, &x, sizeof bits);
        }
        f += (uint64_t)bits * (2 * e + 1);
    }
    return f;
}

}  // namespace sparse

namespace {
// What the per-SM driver (sm_legs.hpp) needs of the sparse probe.
struct SparseProbe {
    using Opts = cro_sparse_opts;
    using Result = cro_sparse_result;
    using Sm = cro_sparse_sm;
    using Fault = cro_sparse_fault;
    using Args = SparseArgs;
    using Tile = int32_t;
    static constexpr const char* kName = "sparse";
    static constexpr const cro_wire& kWire = cro_wire_sparse;
    static constexpr uint32_t kLegs = CRO_SPARSE_LEGS, kAllLegs = CRO_SPARSE_ALL_LEGS, kMaxSms = CRO_SPARSE_MAX_SMS;
    static constexpr uint32_t kRecords = CRO_SPARSE_RECORDS;
    static constexpr int kAnswers = CRO_SPARSE_ANSWERS;
    static constexpr uint64_t Device::*kCalls = &Device::sparse_calls;
    static constexpr SeedSpace kSeeds = kSeedSparse;
    // Iterations per CTA when the caller gives none (DESIGN.md "The sparse probe" for the measurement).
    static constexpr uint32_t kDefaultIterations = 256, kDefaultRounds = 4;
    static constexpr bool kAluLeg[CRO_SPARSE_LEGS] = {false, false, false, false, false, false};

    static int elements(int) { return CRO_SPARSE_M * CRO_SPARSE_N; }
    static void expected(int answer, uint64_t seed, int32_t* out) { sparse::Expected(answer, seed, out); }
    static uint64_t fold(int answer, const int32_t* tile) { return sparse::TileFold(answer, tile); }
    static int answer(uint32_t leg) { return sparse::kLegAnswer[leg]; }
    // dense-equivalent: 2 M N K over the logical K
    static uint64_t ops(uint32_t leg) {
        const int a = sparse::kLegAnswer[leg];
        return 2ull * CRO_SPARSE_M * CRO_SPARSE_N *
               (a == CRO_SPARSE_ANSWER_SMALL128 ? CRO_SPARSE_TF32_K : a == CRO_SPARSE_ANSWER_SMALL256 ? CRO_SPARSE_K16 : CRO_SPARSE_K);
    }
    static cudaError_t launch(uint32_t leg, const SparseArgs& a, int grid, cudaStream_t st) { return launch_sparse(leg, a, grid, st); }
    static void test_args(const cro_sparse_opts& o, uint32_t leg, SparseArgs* a) {
        a->meta = (o.test_meta && (uint32_t)o.test_meta_leg == leg) ? 1u : 0u;
        a->meta_sm = o.test_meta_sm;
        a->meta_iter = o.test_meta_iteration;
        a->meta_row = o.test_meta_row;
        a->meta_group = o.test_meta_group;
    }

    static std::string opts_error(const cro_sparse_opts& o) {
        const uint32_t legs = o.legs ? o.legs : CRO_SPARSE_ALL_LEGS;
        const uint32_t iters = o.iterations ? o.iterations : kDefaultIterations;
        const uint32_t max_rounds = o.max_rounds ? o.max_rounds : kDefaultRounds;
        const int l = o.test_inject_leg, ml = o.test_meta_leg;
        if ((legs & ~CRO_SPARSE_ALL_LEGS) || iters > CRO_SPARSE_MAX_ITERATIONS || max_rounds > CRO_SPARSE_MAX_ROUNDS ||
            (o.test_inject_mask &&
             (l < 0 || l >= CRO_SPARSE_LEGS || o.test_inject_sm < -1 || o.test_inject_sm >= CRO_SPARSE_MAX_SMS ||
              o.test_inject_row < -1 || o.test_inject_row >= CRO_SPARSE_M || o.test_inject_col < -1 ||
              o.test_inject_col >= CRO_SPARSE_N || o.test_inject_iteration >= iters || (o.test_inject_mask >> 32))) ||
            o.test_meta > 1 ||
            (o.test_meta &&
             (ml < 0 || ml >= CRO_SPARSE_LEGS || o.test_meta_sm < -1 || o.test_meta_sm >= CRO_SPARSE_MAX_SMS ||
              o.test_meta_iteration >= iters || o.test_meta_row >= CRO_SPARSE_M ||
              o.test_meta_group >= sparse::Groups(sparse::kLegAnswer[ml]))))
            return "sparse probe: legs must be CRO_SPARSE_ALL_LEGS bits, iterations at most " +
                   std::to_string(CRO_SPARSE_MAX_ITERATIONS) + ", max_rounds at most " + std::to_string(CRO_SPARSE_MAX_ROUNDS) +
                   ", an injection must name a leg, an SM id below " + std::to_string(CRO_SPARSE_MAX_SMS) +
                   " (or -1), a row, a column (or -1), an iteration the leg runs and a mask of at most 32 bits, and a " +
                   "metadata substitution (test_meta 0 or 1) a leg, an SM id (or -1), an iteration the leg runs, a row " +
                   "and a group of the leg";
        return "";
    }
};
}  // namespace

int ctx_probe_sparse(cro_ctx* c, int idx, const cro_sparse_opts& o, cro_sparse_result* r, std::vector<cro_sparse_sm>* sms,
                     std::vector<cro_sparse_fault>* faults) {
    return probe_sm_legs<SparseProbe>(c, idx, o, r, sms, faults);
}

int ctx_probe_sparse_uuid(cro_ctx* c, const char* uuid, const cro_sparse_opts& o, int deadline_ms, cro_sparse_result* r,
                          std::vector<cro_sparse_sm>* sms, std::vector<cro_sparse_fault>* faults, int cap, uint64_t* helper_ns) {
    return probe_sm_legs_uuid<SparseProbe>(c, uuid, o, deadline_ms, r, sms, faults, cap, helper_ns);
}

int classify_sparse(uint32_t legs, const uint32_t* iterations, uint32_t grid, uint64_t k, const uint32_t* rounds,
                    const cro_sm_cta* ctas, const uint64_t* sm_bits, const uint64_t* claims, const cro_sparse_fault* records,
                    cro_sparse_result* r, std::vector<cro_sparse_sm>* sms, std::vector<cro_sparse_fault>* faults) {
    return classify_sm_legs<SparseProbe>(legs, iterations, grid, k, rounds, ctas, sm_bits, claims, records, r, sms, faults);
}

}  // namespace cro
