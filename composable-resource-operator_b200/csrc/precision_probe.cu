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

// The sum over every element e of a leg's tile of canon(expected value in the leg's type) * (2e + 1) (mod 2^64): what
// one iteration adds to a CTA's running fold when every value is right.
uint64_t TileFold(unsigned leg, const int64_t* tile) {
    const int answer = kLegAnswer[leg];
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
// Operands of call k: seed_dev + 2^58 + k * kNonceStride.  No other seed of the device reaches it while every count
// stays below 2^57.  The stride is odd, hence invertible mod 2^64, so seed_dev + O + n * stride (another probe's
// offset O, a multiple of 2^58 as every offset below is) equals it only when (k - n) * stride = O - 2^58, i.e. k - n is
// a nonzero multiple of 2^58 mod 2^64, which needs k or n at least 2^57:
//   probe nonce n:       O = 0;          locator retest:  O = 2^63 (k' = 0);
//   link pattern 3k'+j:  O = 2^62;       compute call k': O = 2^61;
//   SRAM seeds:          O = 2^60;       L2 seeds:        O = 2^59 (their counts counted as n).
// Distinct calls get distinct seeds, so no call passes on the operands an earlier call used.
constexpr uint64_t kPrecisionSeedOffset = 1ull << 58;
// Iterations per CTA when the caller gives none (DESIGN.md "The precision probe" for the measurement).
constexpr uint32_t kPrecisionDefaultIterations = 256;
constexpr uint32_t kPrecisionDefaultAluIterations = 16;
constexpr uint32_t kPrecisionDefaultRounds = 4;
constexpr int kSmWords = CRO_PRECISION_MAX_SMS / 64;
constexpr bool kAluLeg[CRO_PRECISION_LEGS] = {false, true, false, false, false, false, true};     // DFMA, HFMA2
constexpr unsigned kElementBits[CRO_PRECISION_LEGS] = {64, 64, 32, 32, 16, 32, 16};

void blank_result(cro_precision_result* r, const cro_precision_result from, std::vector<cro_precision_sm>* sms,
                  std::vector<cro_precision_fault>* faults) {
    memset(r, 0, sizeof *r);
    r->seed = from.seed;
    r->call = from.call;
    r->sm_count = from.sm_count;
    r->legs = from.legs;
    sms->clear();
    faults->clear();
}

void leg_iterations(const cro_precision_opts& o, uint32_t (&iters)[CRO_PRECISION_LEGS]) {
    const uint32_t ti = o.iterations ? o.iterations : kPrecisionDefaultIterations;
    const uint32_t ai = o.alu_iterations ? o.alu_iterations : kPrecisionDefaultAluIterations;
    for (int l = 0; l < CRO_PRECISION_LEGS; ++l) iters[l] = kAluLeg[l] ? ai : ti;
}

uint32_t leg_n(uint32_t leg) { return precision::Elements(precision::kLegAnswer[leg]) / CRO_PRECISION_M; }

// Why the options are refused ("" when they pass): both forms' argument checks.
std::string precision_opts_error(const cro_precision_opts& o) {
    const uint32_t legs = o.legs ? o.legs : CRO_PRECISION_ALL_LEGS;
    uint32_t iters[CRO_PRECISION_LEGS];
    leg_iterations(o, iters);
    const uint32_t max_rounds = o.max_rounds ? o.max_rounds : kPrecisionDefaultRounds;
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
}  // namespace

int ctx_probe_precision(cro_ctx* c, int idx, const cro_precision_opts& o, cro_precision_result* r,
                        std::vector<cro_precision_sm>* sms, std::vector<cro_precision_fault>* faults) {
    blank_result(r, cro_precision_result{}, sms, faults);
    Device* d = dev_at(c, idx);
    if (!d) return r->status = unknown_device(c, idx, "a GPU probed through the helper process cannot be given kernels from here");
    const uint32_t legs = o.legs ? o.legs : CRO_PRECISION_ALL_LEGS;
    uint32_t iters[CRO_PRECISION_LEGS];
    leg_iterations(o, iters);
    const bool inj = o.test_inject_mask != 0;
    const std::string why = precision_opts_error(o);
    if (!why.empty()) {
        c->set_error(why);
        return r->status = CRO_ERR_INVALID_ARG;
    }
    const uint32_t max_rounds = o.max_rounds ? o.max_rounds : kPrecisionDefaultRounds;
    DeviceGuard g = enter_device(c, idx);
    if (g.rc) return r->status = g.rc;
    std::map<uint32_t, cro_precision_sm> per_sm;
    cudaEvent_t ev[2] = {nullptr, nullptr};     // the call's own, destroyed on every way out
    int rc = [&]() -> int {
        const int grid = d->plan.sm_count;
        const uint64_t k = d->precision_calls++;
        const uint64_t seed = d->seed_dev + kPrecisionSeedOffset + k * kNonceStride;
        r->seed = seed;
        r->call = k;
        r->sm_count = (uint32_t)grid;
        r->legs = legs;
        size_t tile_at[CRO_PRECISION_ANSWERS + 1] = {0};
        for (int a = 0; a < CRO_PRECISION_ANSWERS; ++a) tile_at[a + 1] = tile_at[a] + (size_t)precision::Elements(a);
        std::vector<int64_t> tiles(tile_at[CRO_PRECISION_ANSWERS]);
        const uint64_t h0 = now_ns();
        for (int a = 0; a < CRO_PRECISION_ANSWERS; ++a) precision::Expected(a, seed, tiles.data() + tile_at[a]);
        r->host_ref_ns = now_ns() - h0;

        // [tiles][per leg: sm bitmap, claims][per leg: records][CTA records], allocated per call
        const size_t tile_bytes = tiles.size() * sizeof(int64_t);
        const size_t ctr_off = tile_bytes, ctr_bytes = (size_t)CRO_PRECISION_LEGS * (kSmWords + 1) * 8;
        const size_t rec_off = ctr_off + ctr_bytes, rec_bytes = (size_t)CRO_PRECISION_LEGS * CRO_PRECISION_RECORDS * sizeof(cro_precision_fault);
        const size_t cta_off = (rec_off + rec_bytes + 63) & ~(size_t)63, cta_bytes = (size_t)grid * sizeof(ComputeCta);
        DeviceMem<unsigned char> b;
        CU_TRY(c, cudaMalloc(&b.p, cta_off + cta_bytes));
        for (cudaEvent_t& x : ev) CU_TRY(c, cudaEventCreate(&x));
        cudaStream_t st = d->stream;
        CU_TRY(c, cudaMemcpyAsync(b.p, tiles.data(), tile_bytes, cudaMemcpyHostToDevice, st));
        CU_TRY(c, cudaMemsetAsync(b.p + ctr_off, 0, ctr_bytes, st));
        unsigned long long* ctr = reinterpret_cast<unsigned long long*>(b.p + ctr_off);
        ComputeCta* cta = reinterpret_cast<ComputeCta*>(b.p + cta_off);
        std::vector<ComputeCta> hc((size_t)grid);
        unsigned long long hbits[kSmWords + 1];

        for (uint32_t leg = 0; leg < CRO_PRECISION_LEGS; ++leg) {
            if (!(legs >> leg & 1u)) continue;
            cro_compute_leg& R = r->leg[leg];
            const int answer = precision::kLegAnswer[leg];
            const uint64_t ops = 2ull * CRO_PRECISION_M * leg_n(leg) *
                                 (answer == CRO_PRECISION_ANSWER_SMALL || answer == CRO_PRECISION_ANSWER_NARROW ? CRO_PRECISION_K : 128);
            PrecisionArgs a{};
            a.expect = reinterpret_cast<const long long*>(b.p) + tile_at[answer];
            a.cta = cta;
            a.sm_bits = ctr + (size_t)leg * (kSmWords + 1);
            a.claims = a.sm_bits + kSmWords;
            a.rec = reinterpret_cast<cro_precision_fault*>(b.p + rec_off) + (size_t)leg * CRO_PRECISION_RECORDS;
            a.seed = seed;
            a.stamp = k;
            a.iterations = iters[leg];
            a.inj_sm = o.test_inject_sm;
            a.inj_row = o.test_inject_row;
            a.inj_col = o.test_inject_col;
            a.inj_iter = o.test_inject_iteration;
            a.inj_mask = (inj && (uint32_t)o.test_inject_leg == leg) ? o.test_inject_mask : 0ull;
            R.iterations = iters[leg];
            R.expect_fold = (uint64_t)iters[leg] * precision::TileFold(leg, tiles.data() + tile_at[answer]);
            uint32_t fold_sm = ~0u;
            auto launch = [&] { return launch_precision(leg, a, grid, st); };
            auto fetch = [&] {
                cudaError_t e = cudaMemcpyAsync(hc.data(), cta, cta_bytes, cudaMemcpyDeviceToHost, st);
                return e ? e : cudaMemcpyAsync(hbits, a.sm_bits, sizeof hbits, cudaMemcpyDeviceToHost, st);
            };
            auto take = [&](uint32_t* covered) -> int {
                return take_leg_round(c, "precision probe", hc, k, leg, ops * iters[leg] * (uint64_t)grid, hbits, kSmWords,
                                      CRO_PRECISION_MAX_SMS, R, &r->nsmid, &fold_sm, per_sm, covered);
            };
            const int e = coverage_rounds(c, d, ev, cta, cta_bytes, (uint32_t)grid, max_rounds, &R.rounds, &R.ns, launch, fetch, take);
            if (e) return e;
            R.complete = R.sms_covered >= (uint32_t)grid ? 1u : 0u;
            R.recorded = std::min<uint64_t>(hbits[kSmWords], CRO_PRECISION_RECORDS);
            if (R.recorded) {
                std::vector<cro_precision_fault> f((size_t)R.recorded);
                CU_TRY(c, cudaMemcpy(f.data(), a.rec, f.size() * sizeof(cro_precision_fault), cudaMemcpyDeviceToHost));
                faults->insert(faults->end(), f.begin(), f.end());
            }
            finish_leg(R, per_sm, leg, iters[leg]);
        }
        return CRO_OK;
    }();
    for (cudaEvent_t x : ev)
        if (x) cudaEventDestroy(x);
    if (rc) {
        blank_result(r, *r, sms, faults);
        return r->status = rc;
    }
    return close_call(r, CRO_PRECISION_LEGS, per_sm, sms, faults);
}

int ctx_probe_precision_uuid(cro_ctx* c, const char* uuid, const cro_precision_opts& o, int deadline_ms, cro_precision_result* r,
                             std::vector<cro_precision_sm>* sms, std::vector<cro_precision_fault>* faults, int cap,
                             uint64_t* helper_ns) {
    blank_result(r, cro_precision_result{}, sms, faults);
    *helper_ns = 0;
    if (!uuid) return r->status = CRO_ERR_INVALID_ARG;
    const std::string why = precision_opts_error(o);
    if (!why.empty()) {
        set_call_error(c, why);
        return r->status = CRO_ERR_INVALID_ARG;
    }
    const std::string want = uuid;
    auto num = [](int64_t v) { return std::to_string(v); };
    const std::vector<std::string> args = {"precision-raw", want, std::to_string(helper_seed_base(c)), num(o.iterations),
                                           num(o.alu_iterations), num(o.legs), num(o.max_rounds), num(o.test_inject_leg),
                                           num(o.test_inject_sm), num(o.test_inject_iteration), num(o.test_inject_row),
                                           num(o.test_inject_col), std::to_string(o.test_inject_mask), num(cap)};
    using Frame = SmFrame<cro_precision_result, cro_precision_sm, cro_precision_fault, CRO_PRECISION_MAX_SMS>;
    std::string got;
    const int rc = run_probe_helper(c, want, "precision helper", "cro.probe_precision.helper", args, deadline_ms, Frame::kHead,
                                    sizeof(cro_precision_fault), (size_t)cap, Frame::tail, &got, helper_ns);
    if (rc != CRO_OK) return r->status = rc;
    Frame::read(got, r, sms, faults);
    return r->status;
}

}  // namespace cro
