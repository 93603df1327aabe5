// xlane_probe.cu — the cross-lane probe (cro_probe_xlane, cro_probe_xlane_uuid): every SM's shuffle, vote, match,
// warp-reduce and shared-atomic units checked op by op on every lane, one launch per leg.
#include "lane_report.hpp"
#include "xlane_kernels.cuh"

namespace cro {

namespace {
// Iterations per CTA and leg, and launches per leg, when the caller gives none.  On an H100 80GB HBM3 at a 700 W limit
// (profiles/h100_700w_xlane_rate.jsonl) one iteration of the five legs takes 1.57 ms and one launch per leg covers all
// 132 SMs, so 3 iterations cost about the SRAM and register-file probes' 5 ms (DESIGN.md "The cross-lane probe").
constexpr uint32_t kXlaneDefaultIterations = 3;
constexpr uint32_t kXlaneDefaultRounds = 4;
constexpr size_t kThreadRecs = CRO_XLANE_THREAD_RECORDS;

uint32_t legs_of(const cro_xlane_opts& o) { return o.legs ? o.legs : CRO_XLANE_ALL_LEGS; }

// The result of a call that checked nothing: zeroes but for what the call had settled before it stopped.
void blank_result(cro_xlane_result* r, const cro_xlane_result& from, std::vector<cro_xlane_sm>* sms,
                  std::vector<cro_xlane_fault>* faults) {
    const cro_xlane_result keep = from;
    memset(r, 0, sizeof *r);
    r->seed = keep.seed;
    r->call = keep.call;
    r->sm_count = keep.sm_count;
    r->legs = keep.legs;
    r->iterations = keep.iterations;
    r->cuda_error = keep.cuda_error;
    sms->clear();
    faults->clear();
}

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

// The cross-lane probe's types and constants for the shared report path (lane_report.hpp).
struct XlaneReport {
    using Result = cro_xlane_result;
    using Sm = cro_xlane_sm;
    using Fault = cro_xlane_fault;
    using Thread = cro_xlane_thread;
    using Cta = cro_xlane_cta;
    static constexpr unsigned kLegs = CRO_XLANE_LEGS, kThreads = CRO_XLANE_THREADS, kThreadRecs = CRO_XLANE_THREAD_RECORDS,
                              kRecords = CRO_XLANE_RECORDS, kMaxSms = CRO_XLANE_MAX_SMS, kPersistent = CRO_XLANE_PERSISTENT,
                              kIntermittent = CRO_XLANE_INTERMITTENT, kNone = CRO_XLANE_NONE, kSm = CRO_XLANE_SM, kAll = CRO_XLANE_ALL;
    static constexpr const char* kName = "cross-lane probe";
    static unsigned ops(unsigned leg) { return xlane::kOps[leg]; }
};
using XlaneTally = LaneTally<XlaneReport>;

// The call's settings before anything runs.
void open_xlane_call(cro_xlane_result* r, uint64_t seed, uint64_t k, uint32_t sm_count, uint32_t legs, uint32_t iters) {
    r->seed = seed;
    r->call = k;
    r->sm_count = sm_count;
    r->legs = legs;
    r->iterations = iters;
    closed_form(seed, iters, legs, r);
}
}  // namespace

void xlane_expected(unsigned leg, uint64_t seed, uint32_t iteration, unsigned warp, uint64_t* out) {
    xlane::expected(leg, seed + (uint64_t)iteration * kNonceStride, warp, reinterpret_cast<xlane::u64*>(out));
}

std::string xlane_opts_error(const cro_xlane_opts& o) {
    const uint32_t iters = o.iterations ? o.iterations : kXlaneDefaultIterations;
    const int leg = o.test_inject_leg;
    const bool inj_ok = !o.test_inject_mask ||
                        (leg >= 0 && leg < CRO_XLANE_LEGS && (legs_of(o) >> leg & 1u) && o.test_inject_sm >= -1 &&
                         o.test_inject_sm < CRO_XLANE_MAX_SMS && o.test_inject_warp >= -1 && o.test_inject_warp < CRO_XLANE_WARPS &&
                         o.test_inject_lane >= -1 && o.test_inject_lane < 32 && o.test_inject_op < xlane::kOps[leg] &&
                         o.test_inject_iteration < iters &&
                         !(leg == CRO_XLANE_LEG_ATOMS && (o.test_inject_op / xlane::kAtomsShapes == xlane::kAtInc ||
                                                          o.test_inject_op / xlane::kAtomsShapes == xlane::kAtDec)));
    if (iters > CRO_XLANE_MAX_ITERATIONS || o.legs > CRO_XLANE_ALL_LEGS || o.max_rounds > CRO_XLANE_MAX_ROUNDS || o.deadline_ms < 0 ||
        !inj_ok)
        return "cross-lane probe: iterations at most " + std::to_string(CRO_XLANE_MAX_ITERATIONS) + ", legs at most 0x1F, max_rounds at most " +
               std::to_string(CRO_XLANE_MAX_ROUNDS) + ", deadline_ms not negative, and an injection must name a leg the call runs, an SM "
               "id below " + std::to_string(CRO_XLANE_MAX_SMS) + ", a warp below 8 and a lane below 32 (each or -1), an op of the "
               "leg (not ATOMS inc or dec) and an iteration the call runs";
    return "";
}

int ctx_probe_xlane(cro_ctx* c, int idx, const cro_xlane_opts& o, cro_xlane_result* r, std::vector<cro_xlane_sm>* sms,
                    std::vector<cro_xlane_fault>* faults) {
    const uint64_t t_call = now_ns();
    blank_result(r, cro_xlane_result{}, sms, faults);
    Device* d = dev_at(c, idx);
    if (!d) return r->status = unknown_device(c, idx, "a GPU attached after init is probed through the helper process, cro_probe_xlane_uuid");
    const uint32_t iters = o.iterations ? o.iterations : kXlaneDefaultIterations;
    const uint32_t max_rounds = o.max_rounds ? o.max_rounds : kXlaneDefaultRounds;
    const uint32_t legs = legs_of(o);
    const std::string why = xlane_opts_error(o);
    if (!why.empty()) {
        c->set_error(why);
        return r->status = CRO_ERR_INVALID_ARG;
    }
    DeviceGuard g = enter_device(c, idx);
    if (g.rc) return r->status = g.rc;
    Range nv(c, "cro.probe_xlane");
    XlaneTally t;
    cudaEvent_t ev[2] = {nullptr, nullptr};                  // the call's own, destroyed on every way out
    int rc = [&]() -> int {
        const int sm_count = d->plan.sm_count;
        for (unsigned leg = 0; leg < CRO_XLANE_LEGS; ++leg)
            if (legs >> leg & 1u) CU_TRY(c, xlane_plan(d->ordinal, leg));
        const uint64_t k = d->xlane_calls++;
        open_xlane_call(r, space_seed(d, kSeedXlane, k), k, (uint32_t)sm_count, legs, iters);

        // [CTA entries][thread entries] (armed together every round), then [records], allocated per call
        const size_t n_thr = (size_t)sm_count * CRO_XLANE_THREADS;
        const size_t cta_bytes = (size_t)sm_count * sizeof(cro_xlane_cta), thr_bytes = n_thr * sizeof(cro_xlane_thread);
        const size_t rec_off = (cta_bytes + thr_bytes + 255) & ~(size_t)255, rec_bytes = n_thr * kThreadRecs * sizeof(cro_xlane_fault);
        DeviceMem<unsigned char> b;
        CU_TRY(c, cudaMalloc(&b.p, rec_off + rec_bytes));
        for (cudaEvent_t& x : ev) CU_TRY(c, cudaEventCreate(&x));
        cudaStream_t st = d->stream;
        XlaneArgs a{};
        a.cta = reinterpret_cast<cro_xlane_cta*>(b.p);
        a.thr = reinterpret_cast<cro_xlane_thread*>(b.p + cta_bytes);
        a.rec = reinterpret_cast<cro_xlane_fault*>(b.p + rec_off);
        a.seed = r->seed;
        a.stamp = k;
        a.iterations = iters;
        a.inj_sm = o.test_inject_sm;
        a.inj_warp = o.test_inject_warp;
        a.inj_lane = o.test_inject_lane;
        a.inj_op = o.test_inject_op;
        a.inj_iter = o.test_inject_iteration;
        std::vector<unsigned char> head(cta_bytes + thr_bytes);
        std::vector<cro_xlane_fault> hr(n_thr * kThreadRecs);
        const auto* hc = reinterpret_cast<const cro_xlane_cta*>(head.data());
        const auto* ht = reinterpret_cast<const cro_xlane_thread*>(head.data() + cta_bytes);
        for (unsigned leg = 0; leg < CRO_XLANE_LEGS; ++leg) {
            if (!(legs >> leg & 1u)) continue;
            a.inj_mask = o.test_inject_mask && o.test_inject_leg == (int)leg ? o.test_inject_mask : 0ull;
            auto launch = [&] { return launch_xlane(leg, a, sm_count, st); };
            auto fetch = [&] { return cudaMemcpyAsync(head.data(), b.p, head.size(), cudaMemcpyDeviceToHost, st); };
            auto take = [&](uint32_t* covered) -> int {
                if (lane_any_failed<XlaneReport>(ht, sm_count, k)) CU_TRY(c, cudaMemcpy(hr.data(), a.rec, rec_bytes, cudaMemcpyDeviceToHost));
                return take_lane_round<XlaneReport>(c, leg, hc, ht, hr.data(), sm_count, k, r, t, covered);
            };
            uint32_t rounds = 0;
            const int e = coverage_rounds(c, d, ev, b.p, head.size(), (uint32_t)sm_count, max_rounds, &rounds, &r->leg_ns[leg], launch,
                                          fetch, take);
            r->rounds += rounds;
            r->ns += r->leg_ns[leg];
            if (e) return e;
        }
        return CRO_OK;
    }();
    for (cudaEvent_t x : ev)
        if (x) cudaEventDestroy(x);
    if (rc == CRO_ERR_CUDA) r->cuda_error = (int32_t)cudaGetLastError();
    if (rc) {
        blank_result(r, *r, sms, faults);
        r->wall_ns = now_ns() - t_call;
        return r->status = rc;
    }
    const int status = close_lane_call<XlaneReport>(r, t, sms, faults);
    r->wall_ns = now_ns() - t_call;
    return status;
}

int classify_xlane(uint32_t legs, uint32_t iterations, uint64_t seed, uint32_t sm_count, uint64_t k, uint32_t rounds,
                   const cro_xlane_cta* ctas, const cro_xlane_thread* threads, const cro_xlane_fault* records,
                   cro_xlane_result* r, std::vector<cro_xlane_sm>* sms, std::vector<cro_xlane_fault>* faults) {
    blank_result(r, cro_xlane_result{}, sms, faults);
    open_xlane_call(r, seed, k, sm_count, legs, iterations);
    XlaneTally t;
    const size_t n_thr = (size_t)sm_count * CRO_XLANE_THREADS;
    for (unsigned leg = 0; leg < CRO_XLANE_LEGS; ++leg) {
        if (!(legs >> leg & 1u)) continue;
        for (uint32_t j = 0; j < rounds; ++j, ctas += sm_count, threads += n_thr, records += n_thr * kThreadRecs) {
            ++r->rounds;
            uint32_t covered = 0;
            const int e = take_lane_round<XlaneReport>(nullptr, leg, ctas, threads, records, (int)sm_count, k, r, t, &covered);
            if (e) {
                blank_result(r, *r, sms, faults);
                return r->status = e;
            }
        }
    }
    return close_lane_call<XlaneReport>(r, t, sms, faults);
}

int ctx_probe_xlane_uuid(cro_ctx* c, const char* uuid, const cro_xlane_opts& o, cro_xlane_result* r,
                         std::vector<cro_xlane_sm>* sms, std::vector<cro_xlane_fault>* faults, int cap) {
    blank_result(r, cro_xlane_result{}, sms, faults);
    if (!uuid) return r->status = CRO_ERR_INVALID_ARG;
    const std::string why = xlane_opts_error(o);
    if (!why.empty()) {
        set_call_error(c, why);
        return r->status = CRO_ERR_INVALID_ARG;
    }
    uint64_t helper_ns = 0;
    if (run_check_helper(c, cro_wire_xlane, uuid, "cross-lane helper", "cro.probe_xlane.helper", &o, cap, o.deadline_ms, &helper_ns,
                         r, faults, sms) == CRO_OK)
        r->helper_ns = helper_ns;
    return r->status;
}

}  // namespace cro
