// compute_probe.cu — the SM compute probe (cro_probe_compute): every SM's tensor cores and ALUs against an exact answer.
#include "compute.hpp"
#include "sm_legs.hpp"

namespace cro {

namespace {
// Operands of call k: seed_dev + 2^61 + k * kNonceStride.  No other seed of the device reaches it while every count
// stays below 2^61.  The stride is odd, hence invertible mod 2^64, and 2^61 times an odd number is c * 2^61 with c odd
// (mod 2^64), which as a signed difference is +-2^61 or +-3 * 2^61.
//   probe nonce n:       seed_dev + n * stride equals it only when (n - k) * stride = 2^61, i.e. n - k = c * 2^61: n or
//                        k must be at least 2^61;
//   locator retest:      seed_dev + 2^63 needs k * stride = 2^63 - 2^61 = 3 * 2^61, so k = c * 2^61 >= 2^61;
//   link pattern 3k'+j:  seed_dev + 2^62 + (3k' + j) * stride needs (k - 3k' - j) * stride = 2^61, so k or 3k' + j is
//                        at least 2^61.
// Distinct calls get distinct seeds, so no call passes on the operands an earlier call used.
constexpr uint64_t kComputeSeedOffset = 1ull << 61;
// Tensor legs: iterations per CTA when the caller gives none (DESIGN.md "The compute probe" for the measurement).
constexpr uint32_t kComputeDefaultIterations = 256;
constexpr uint32_t kComputeDefaultAluIterations = 4;
constexpr uint32_t kComputeDefaultRounds = 4;
constexpr uint64_t kComputeOps = 2ull * CRO_COMPUTE_M * CRO_COMPUTE_N * CRO_COMPUTE_K;   // one tile, one iteration
constexpr int kSmWords = CRO_COMPUTE_MAX_SMS / 64;

// The result of a call that computed nothing: zeroes but for what the call had settled before it stopped (`from`'s
// seed, call number, SM count and legs).
void blank_result(cro_compute_result* r, const cro_compute_result from, std::vector<cro_compute_sm>* sms,
                  std::vector<cro_compute_fault>* faults) {
    memset(r, 0, sizeof *r);
    r->seed = from.seed;
    r->call = from.call;
    r->sm_count = from.sm_count;
    r->legs = from.legs;
    sms->clear();
    faults->clear();
}

// Why the options are refused ("" when they pass): both forms' argument checks.
std::string compute_opts_error(const cro_compute_opts& o) {
    const uint32_t legs = o.legs ? o.legs : CRO_COMPUTE_ALL_LEGS;
    const uint32_t ti = o.iterations ? o.iterations : kComputeDefaultIterations;
    const uint32_t ai = o.alu_iterations ? o.alu_iterations : kComputeDefaultAluIterations;
    const uint32_t iters[CRO_COMPUTE_LEGS] = {ti, ti, ti, ai, ai};
    const uint32_t max_rounds = o.max_rounds ? o.max_rounds : kComputeDefaultRounds;
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
}  // namespace

int ctx_probe_compute(cro_ctx* c, int idx, const cro_compute_opts& o, cro_compute_result* r, std::vector<cro_compute_sm>* sms,
                      std::vector<cro_compute_fault>* faults) {
    blank_result(r, cro_compute_result{}, sms, faults);
    Device* d = dev_at(c, idx);
    if (!d) return r->status = unknown_device(c, idx, "a GPU probed through the helper process cannot be given kernels from here");
    const uint32_t legs = o.legs ? o.legs : CRO_COMPUTE_ALL_LEGS;
    const uint32_t ti = o.iterations ? o.iterations : kComputeDefaultIterations;
    const uint32_t ai = o.alu_iterations ? o.alu_iterations : kComputeDefaultAluIterations;
    const uint32_t iters[CRO_COMPUTE_LEGS] = {ti, ti, ti, ai, ai};   // s8, bf16, e4m3 tensor legs; ffma, imad ALU legs
    const bool inj = o.test_inject_mask != 0;
    const std::string why = compute_opts_error(o);
    if (!why.empty()) {
        c->set_error(why);
        return r->status = CRO_ERR_INVALID_ARG;
    }
    const uint32_t max_rounds = o.max_rounds ? o.max_rounds : kComputeDefaultRounds;
    DeviceGuard g = enter_device(c, idx);
    if (g.rc) return r->status = g.rc;
    std::map<uint32_t, cro_compute_sm> per_sm;
    cudaEvent_t ev[2] = {nullptr, nullptr};     // the call's own, destroyed on every way out
    int rc = [&]() -> int {
        const int grid = d->plan.sm_count;
        const uint64_t k = d->compute_calls++;
        const uint64_t seed = d->seed_dev + kComputeSeedOffset + k * kNonceStride;
        r->seed = seed;
        r->call = k;
        r->sm_count = (uint32_t)grid;
        r->legs = legs;
        std::vector<int32_t> tiles(2 * (size_t)compute::kTile);
        const uint64_t h0 = now_ns();
        compute::Expected(CRO_COMPUTE_ANSWER_S8, seed, tiles.data());
        compute::Expected(CRO_COMPUTE_ANSWER_SMALL, seed, tiles.data() + compute::kTile);
        r->host_ref_ns = now_ns() - h0;
        const uint64_t cta_fold[2] = {compute::CtaFold(tiles.data()), compute::CtaFold(tiles.data() + compute::kTile)};

        // [tiles][per leg: sm bitmap, claims][per leg: records][CTA records], allocated per call
        const size_t tile_bytes = tiles.size() * sizeof(int32_t);
        const size_t ctr_off = tile_bytes, ctr_bytes = (size_t)CRO_COMPUTE_LEGS * (kSmWords + 1) * 8;
        const size_t rec_off = ctr_off + ctr_bytes, rec_bytes = (size_t)CRO_COMPUTE_LEGS * CRO_COMPUTE_RECORDS * sizeof(cro_compute_fault);
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

        for (uint32_t leg = 0; leg < CRO_COMPUTE_LEGS; ++leg) {
            if (!(legs >> leg & 1u)) continue;
            cro_compute_leg& R = r->leg[leg];
            const int answer = (leg == CRO_COMPUTE_LEG_S8 || leg == CRO_COMPUTE_LEG_IMAD) ? 0 : 1;
            ComputeArgs a{};
            a.expect = reinterpret_cast<const int*>(b.p) + (size_t)answer * compute::kTile;
            a.cta = cta;
            a.sm_bits = ctr + (size_t)leg * (kSmWords + 1);
            a.claims = a.sm_bits + kSmWords;
            a.rec = reinterpret_cast<cro_compute_fault*>(b.p + rec_off) + (size_t)leg * CRO_COMPUTE_RECORDS;
            a.seed = seed;
            a.stamp = k;
            a.iterations = iters[leg];
            a.inj_sm = o.test_inject_sm;
            a.inj_row = o.test_inject_row;
            a.inj_col = o.test_inject_col;
            a.inj_iter = o.test_inject_iteration;
            a.inj_mask = (inj && (uint32_t)o.test_inject_leg == leg) ? o.test_inject_mask : 0u;
            R.iterations = iters[leg];
            R.expect_fold = (uint64_t)iters[leg] * cta_fold[answer];
            uint32_t fold_sm = ~0u;
            auto launch = [&] { return launch_compute(leg, a, grid, st); };
            auto fetch = [&] {
                cudaError_t e = cudaMemcpyAsync(hc.data(), cta, cta_bytes, cudaMemcpyDeviceToHost, st);
                return e ? e : cudaMemcpyAsync(hbits, a.sm_bits, sizeof hbits, cudaMemcpyDeviceToHost, st);
            };
            auto take = [&](uint32_t* covered) -> int {
                return take_leg_round(c, "compute probe", hc, k, leg, kComputeOps * iters[leg] * (uint64_t)grid, hbits, kSmWords,
                                      CRO_COMPUTE_MAX_SMS, R, &r->nsmid, &fold_sm, per_sm, covered);
            };
            const int e = coverage_rounds(c, d, ev, cta, cta_bytes, (uint32_t)grid, max_rounds, &R.rounds, &R.ns, launch, fetch, take);
            if (e) return e;
            R.complete = R.sms_covered >= (uint32_t)grid ? 1u : 0u;
            R.recorded = std::min<uint64_t>(hbits[kSmWords], CRO_COMPUTE_RECORDS);
            if (R.recorded) {
                std::vector<cro_compute_fault> f((size_t)R.recorded);
                CU_TRY(c, cudaMemcpy(f.data(), a.rec, f.size() * sizeof(cro_compute_fault), cudaMemcpyDeviceToHost));
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
    return close_call(r, CRO_COMPUTE_LEGS, per_sm, sms, faults);
}

int ctx_probe_compute_uuid(cro_ctx* c, const char* uuid, const cro_compute_opts& o, int deadline_ms, cro_compute_result* r,
                           std::vector<cro_compute_sm>* sms, std::vector<cro_compute_fault>* faults, int cap, uint64_t* helper_ns) {
    blank_result(r, cro_compute_result{}, sms, faults);
    *helper_ns = 0;
    if (!uuid) return r->status = CRO_ERR_INVALID_ARG;
    const std::string why = compute_opts_error(o);
    if (!why.empty()) {
        set_call_error(c, why);
        return r->status = CRO_ERR_INVALID_ARG;
    }
    const std::string want = uuid;
    auto num = [](int64_t v) { return std::to_string(v); };
    const std::vector<std::string> args = {"compute-raw", want, std::to_string(helper_seed_base(c)), num(o.iterations),
                                           num(o.alu_iterations), num(o.legs), num(o.max_rounds), num(o.test_inject_leg),
                                           num(o.test_inject_sm), num(o.test_inject_iteration), num(o.test_inject_row),
                                           num(o.test_inject_col), num(o.test_inject_mask), num(cap)};
    using Frame = SmFrame<cro_compute_result, cro_compute_sm, cro_compute_fault, CRO_COMPUTE_MAX_SMS>;
    std::string got;
    const int rc = run_probe_helper(c, want, "compute helper", "cro.probe_compute.helper", args, deadline_ms, Frame::kHead,
                                    sizeof(cro_compute_fault), (size_t)cap, Frame::tail, &got, helper_ns);
    if (rc != CRO_OK) return r->status = rc;
    Frame::read(got, r, sms, faults);
    return r->status;
}

}  // namespace cro
