// precision_probe.cu — the SM precision probe (cro_probe_precision): every SM's FP64, TF32, FP16 and E5M2 arithmetic
// against an exact answer, compared bit for bit; its expected answers, computed on the host; and its helper form.
#include "precision_kernels.cuh"
#include "sm_legs.hpp"

namespace cro {

namespace precision {

namespace {
struct Shape {
    int m, n, k;
};
constexpr Shape kShape[CRO_PRECISION_ANSWERS] = {{CRO_PRECISION_M, CRO_PRECISION_F64_N, CRO_PRECISION_F64_K},
                                                 {CRO_PRECISION_M, CRO_PRECISION_N, CRO_PRECISION_TF32_K},
                                                 {CRO_PRECISION_M, CRO_PRECISION_N, CRO_PRECISION_K},
                                                 {CRO_PRECISION_M, CRO_PRECISION_N, CRO_PRECISION_K}};

// Element e of the operands of `seed` under answer's reading (include/croprobe.h, "SM precision").
inline int64_t operand(int answer, uint64_t seed, uint32_t e) {
    if (answer == CRO_PRECISION_ANSWER_WIDE) return (int64_t)(pattern_word(seed, e) << 44) >> 44;
    const unsigned byte = (unsigned)(pattern_word(seed, e / 8) >> (8 * (e % 8))) & 0xFFu;
    return answer == CRO_PRECISION_ANSWER_NARROW ? (int64_t)(byte & 3u) - 2 : (int64_t)(byte & 7u) - 4;
}

// IEEE binary16 bits of an integer of magnitude at most 2048 (exact: 11 significant bits).
uint64_t f16_bits(int64_t v) {
    if (v == 0) return 0;
    const uint64_t sign = v < 0 ? 0x8000u : 0u, a = (uint64_t)(v < 0 ? -v : v);
    const int e = 63 - __builtin_clzll(a);
    const uint64_t frac = (e <= 10 ? a << (10 - e) : a >> (e - 10)) & 0x3FFu;
    return sign | (uint64_t)(e + 15) << 10 | frac;
}
}  // namespace

const int kLegAnswer[CRO_PRECISION_LEGS] = {CRO_PRECISION_ANSWER_WIDE,  CRO_PRECISION_ANSWER_WIDE,   CRO_PRECISION_ANSWER_SMALL128,
                                            CRO_PRECISION_ANSWER_SMALL, CRO_PRECISION_ANSWER_NARROW, CRO_PRECISION_ANSWER_SMALL,
                                            CRO_PRECISION_ANSWER_NARROW};

int Elements(int answer) { return kShape[answer].m * kShape[answer].n; }

namespace {
// D = A * B with T arithmetic, exact for the answer's bounds: int16 holds every small-int and narrow partial sum (at
// most 4096 in magnitude) and vectorises eight to a register; double holds every wide one (at most 2^45 < 2^53).
template <class T>
void multiply(int answer, uint64_t seed, int64_t* out) {
    const Shape s = kShape[answer];
    std::vector<T> a((size_t)s.m * s.k), b((size_t)s.k * s.n);      // A[m][k], B[k][n]
    for (uint32_t e = 0; e < (uint32_t)(s.m * s.k + s.k * s.n); ++e) {
        const T x = (T)operand(answer, seed, e);
        if (e < (uint32_t)(s.m * s.k)) a[e] = x;
        else b[e - s.m * s.k] = x;
    }
    std::vector<T> row((size_t)s.n);
    for (int m = 0; m < s.m; ++m) {
        std::fill(row.begin(), row.end(), (T)0);
        for (int k = 0; k < s.k; ++k) {
            const T x = a[(size_t)m * s.k + k];
            const T* bk = b.data() + (size_t)k * s.n;
            for (int n = 0; n < s.n; ++n) row[n] = (T)(row[n] + x * bk[n]);
        }
        for (int n = 0; n < s.n; ++n) out[(size_t)m * s.n + n] = (int64_t)row[n];
    }
}
}  // namespace

int Expected(int answer, uint64_t seed, int64_t* out) {
    if (answer < 0 || answer >= CRO_PRECISION_ANSWERS || !out) return CRO_ERR_INVALID_ARG;
    if (answer == CRO_PRECISION_ANSWER_WIDE) multiply<double>(answer, seed, out);
    else multiply<int16_t>(answer, seed, out);
    return CRO_OK;
}

// The sum over every element e of an answer's tile of canon(expected value in its legs' type) * (2e + 1) (mod 2^64):
// what one iteration adds to a CTA's running fold when every value is right.
uint64_t TileFold(int answer, const int64_t* tile) {
    uint64_t f = 0;
    for (uint64_t e = 0; e < (uint64_t)Elements(answer); ++e) {
        const int64_t v = tile[e];
        uint64_t bits;
        if (answer == CRO_PRECISION_ANSWER_WIDE) {
            const double x = (double)v;
            memcpy(&bits, &x, sizeof bits);
        } else if (answer == CRO_PRECISION_ANSWER_NARROW) {
            bits = f16_bits(v);
        } else {
            const float x = (float)v;
            uint32_t u;
            memcpy(&u, &x, sizeof u);
            bits = u;
        }
        f += bits * (2 * e + 1);        // an integer's encoding is never -0: canon is the identity here
    }
    return f;
}

}  // namespace precision

namespace {
constexpr unsigned kElementBits[CRO_PRECISION_LEGS] = {64, 64, 32, 32, 16, 32, 16};

uint32_t leg_n(uint32_t leg) { return precision::Elements(precision::kLegAnswer[leg]) / CRO_PRECISION_M; }

// What the per-SM driver (sm_legs.hpp) needs of the precision probe.
struct PrecisionProbe {
    using Opts = cro_precision_opts;
    using Result = cro_precision_result;
    using Sm = cro_precision_sm;
    using Fault = cro_precision_fault;
    using Args = PrecisionArgs;
    using Tile = int64_t;
    static constexpr const char* kName = "precision";
    static constexpr const cro_wire& kWire = cro_wire_precision;
    static constexpr uint32_t kLegs = CRO_PRECISION_LEGS, kAllLegs = CRO_PRECISION_ALL_LEGS, kMaxSms = CRO_PRECISION_MAX_SMS;
    static constexpr uint32_t kRecords = CRO_PRECISION_RECORDS;
    static constexpr int kAnswers = CRO_PRECISION_ANSWERS;
    static constexpr uint64_t Device::*kCalls = &Device::precision_calls;
    static constexpr SeedSpace kSeeds = kSeedPrecision;
    // Iterations per CTA when the caller gives none (DESIGN.md "The precision probe" for the measurement).
    static constexpr uint32_t kDefaultIterations = 256, kDefaultAluIterations = 16, kDefaultRounds = 4;
    static constexpr bool kAluLeg[CRO_PRECISION_LEGS] = {false, true, false, false, false, false, true};     // DFMA, HFMA2

    static int elements(int answer) { return precision::Elements(answer); }
    static void expected(int answer, uint64_t seed, int64_t* out) { precision::Expected(answer, seed, out); }
    static uint64_t fold(int answer, const int64_t* tile) { return precision::TileFold(answer, tile); }
    static int answer(uint32_t leg) { return precision::kLegAnswer[leg]; }
    static uint64_t ops(uint32_t leg) {
        const int a = precision::kLegAnswer[leg];
        return 2ull * CRO_PRECISION_M * leg_n(leg) *
               (a == CRO_PRECISION_ANSWER_SMALL || a == CRO_PRECISION_ANSWER_NARROW ? CRO_PRECISION_K : 128);
    }
    static cudaError_t launch(uint32_t leg, const PrecisionArgs& a, int grid, cudaStream_t st) { return launch_precision(leg, a, grid, st); }

    static void test_args(const cro_precision_opts&, uint32_t, PrecisionArgs*) {}

    static std::string opts_error(const cro_precision_opts& o) {
        const uint32_t legs = o.legs ? o.legs : CRO_PRECISION_ALL_LEGS;
        uint32_t iters[CRO_PRECISION_LEGS];
        leg_iterations<PrecisionProbe>(o, iters);
        const uint32_t max_rounds = o.max_rounds ? o.max_rounds : kDefaultRounds;
        const int l = o.test_inject_leg;
        if ((legs & ~CRO_PRECISION_ALL_LEGS) || iters[CRO_PRECISION_LEG_F64] > CRO_PRECISION_MAX_ITERATIONS ||
            iters[CRO_PRECISION_LEG_DFMA] > CRO_PRECISION_MAX_ALU_ITERATIONS || max_rounds > CRO_PRECISION_MAX_ROUNDS ||
            (o.test_inject_mask &&
             (l < 0 || l >= CRO_PRECISION_LEGS || o.test_inject_sm < -1 || o.test_inject_sm >= CRO_PRECISION_MAX_SMS ||
              o.test_inject_row < -1 || o.test_inject_row >= CRO_PRECISION_M || o.test_inject_col < -1 ||
              o.test_inject_col >= (int32_t)leg_n((uint32_t)l) || o.test_inject_iteration >= iters[l] ||
              (kElementBits[l] < 64 && (o.test_inject_mask >> kElementBits[l])))))
            return "precision probe: legs must be CRO_PRECISION_ALL_LEGS bits, iterations at most " +
                   std::to_string(CRO_PRECISION_MAX_ITERATIONS) + ", alu_iterations at most " +
                   std::to_string(CRO_PRECISION_MAX_ALU_ITERATIONS) + ", max_rounds at most " +
                   std::to_string(CRO_PRECISION_MAX_ROUNDS) + ", and an injection must name a leg, an SM id below " +
                   std::to_string(CRO_PRECISION_MAX_SMS) + " (or -1), a row, a column of the leg (or -1), an iteration the leg " +
                   "runs and a mask no wider than the leg's element";
        return "";
    }
};
}  // namespace

int ctx_probe_precision(cro_ctx* c, int idx, const cro_precision_opts& o, cro_precision_result* r,
                        std::vector<cro_precision_sm>* sms, std::vector<cro_precision_fault>* faults) {
    return probe_sm_legs<PrecisionProbe>(c, idx, o, r, sms, faults);
}

std::string precision_opts_error(const cro_precision_opts& o) { return PrecisionProbe::opts_error(o); }

int ctx_probe_precision_uuid(cro_ctx* c, const char* uuid, const cro_precision_opts& o, int deadline_ms, cro_precision_result* r,
                             std::vector<cro_precision_sm>* sms, std::vector<cro_precision_fault>* faults, int cap,
                             uint64_t* helper_ns) {
    return probe_sm_legs_uuid<PrecisionProbe>(c, uuid, o, deadline_ms, r, sms, faults, cap, helper_ns);
}

int classify_precision(uint32_t legs, const uint32_t* iterations, uint32_t grid, uint64_t k, const uint32_t* rounds,
                       const cro_sm_cta* ctas, const uint64_t* sm_bits, const uint64_t* claims, const cro_precision_fault* records,
                       cro_precision_result* r, std::vector<cro_precision_sm>* sms, std::vector<cro_precision_fault>* faults) {
    return classify_sm_legs<PrecisionProbe>(legs, iterations, grid, k, rounds, ctas, sm_bits, claims, records, r, sms, faults);
}

}  // namespace cro
