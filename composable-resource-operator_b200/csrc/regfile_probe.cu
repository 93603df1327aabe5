// regfile_probe.cu — the register-file probe (cro_probe_regfile, cro_probe_regfile_uuid): every SM's registers held
// as 0 and as 1 across two barriers and checked word by word, and the SRAM ECC record NVML keeps.
#include <tuple>

#include "cell_report.hpp"

namespace cro {

namespace {
// Iterations per CTA and launches when the caller gives none.  On an H100 80GB HBM3 at a 700 W limit
// (profiles/h100_700w_regfile_rate.jsonl) one iteration takes 51 us and one launch covers all 132 SMs, so 96 iterations
// cost about the SRAM probe's 5 ms (DESIGN.md "The register-file probe").
constexpr uint32_t kRegfileDefaultIterations = 96;
constexpr uint32_t kRegfileDefaultRounds = 4;

// What every CTA's fold must be: the last iteration's E1 words ~P(t, s) over every thread and slot.
void closed_form(uint64_t seed, uint32_t iterations, cro_regfile_result* r) {
    const uint64_t si = seed + (uint64_t)(iterations - 1) * kNonceStride;
    uint64_t x = 0, s = 0, w = 0;
    for (uint64_t t = 0; t < CRO_REGFILE_THREADS; ++t)
        for (uint64_t k = 0; k < CRO_REGFILE_SLOTS; ++k) {
            const uint64_t v = (uint32_t)~pattern_word(si, t * CRO_REGFILE_SLOTS + k);
            x ^= v;
            s += v;
            w += v * (2 * k + 1);
        }
    r->expect_xor = x;
    r->expect_sum = s;
    r->expect_wsum = w;
}

// What the memory-cell probes' host driver (cell_report.hpp) needs of the register-file probe: one leg, whose totals
// and per-SM parts are the result and the SM entry themselves.
struct RegfileProbe {
    using Opts = cro_regfile_opts;
    using Result = cro_regfile_result;
    using Sm = cro_regfile_sm;
    using Fault = cro_regfile_fault;
    using Cta = cro_regfile_cta;
    using Record = cro_regfile_fault;
    using Args = RegfileArgs;
    struct Call {
        uint32_t legs = 1, iterations = 0;
    };
    static constexpr unsigned kLegs = 1, kElements = CRO_REGFILE_ELEMENTS, kRecords = CRO_REGFILE_RECORDS,
                              kMaxSms = CRO_REGFILE_MAX_SMS, kPersistent = CRO_REGFILE_PERSISTENT,
                              kIntermittent = CRO_REGFILE_INTERMITTENT, kDefaultRounds = kRegfileDefaultRounds;
    static constexpr const char* kName = "register-file";
    static constexpr const char* kId = "regfile";
    static constexpr const cro_wire& kWire = cro_wire_regfile;
    static constexpr auto kCalls = &Device::regfile_calls;
    static constexpr SeedSpace kSeeds = kSeedRegfile;

    static cro_regfile_result& leg(cro_regfile_result& r, unsigned) { return r; }
    static cro_regfile_sm& leg(cro_regfile_sm& s, unsigned) { return s; }
    static std::string opts_error(const cro_regfile_opts& o) { return regfile_opts_error(o); }
    static std::string helper_opts_error(const cro_regfile_opts& o) { return regfile_opts_error(o); }

    // The kernel's shared memory and carve-out, and the registers it and the SM have.
    static int plan(cro_ctx* c, Device* d, const cro_regfile_opts& o, cro_regfile_result* r, Call* call) {
        call->iterations = o.iterations ? o.iterations : kRegfileDefaultIterations;
        cudaFuncAttributes fa{};
        CU_TRY(c, regfile_plan(d->ordinal, &fa));
        int regs = 0;
        CU_TRY(c, cudaDeviceGetAttribute(&regs, cudaDevAttrMaxRegistersPerMultiprocessor, d->ordinal));
        r->num_regs = (uint32_t)fa.numRegs;
        r->regs_per_sm = (uint32_t)regs;
        return CRO_OK;
    }
    static void open(const Call& call, cro_regfile_result* r) {      // slots and threads: keep() set them when r was blanked
        r->iterations = call.iterations;
        closed_form(r->seed, call.iterations, r);
    }
    static int grid(const Call&, unsigned, int sm_count) { return sm_count; }
    static void args(const cro_regfile_opts& o, const Call&, unsigned, RegfileArgs* a) {
        a->inj_sm = o.test_inject_sm;
        a->inj_warp = o.test_inject_warp;
        a->inj_lane = o.test_inject_lane;
        a->inj_slot = o.test_inject_slot;
        a->inj_element = o.test_inject_element;
        a->inj_iter = o.test_inject_iteration;
        a->inj_mask = o.test_inject_mask;
    }
    static cudaError_t launch(const Call&, unsigned, RegfileArgs& a, uint32_t, int grid, cudaStream_t st) {
        return launch_regfile(a, grid, st);
    }
    static void round(Call&, cro_regfile_result&, unsigned, const cro_regfile_cta*, int, uint64_t) {}
    static bool folds(unsigned) { return true; }

    static int close(cro_regfile_result* r, const CellTally<RegfileProbe>& t, const Call&, std::vector<cro_regfile_sm>* sms,
                     std::vector<cro_regfile_fault>* faults);
    static void keep(cro_regfile_result* r, const cro_regfile_result& from) {
        r->iterations = from.iterations;
        r->slots = CRO_REGFILE_SLOTS;
        r->threads = CRO_REGFILE_THREADS;
        r->num_regs = from.num_regs;
        r->regs_per_sm = from.regs_per_sm;
    }
};

// The call's end: the bits checked by the CTAs that published, the SM list, the bad SMs, the records sorted and the
// verdict.
int RegfileProbe::close(cro_regfile_result* r, const CellTally<RegfileProbe>& t, const Call&, std::vector<cro_regfile_sm>* sms,
                        std::vector<cro_regfile_fault>* faults) {
    r->bits_checked = 32ull * CRO_REGFILE_SLOTS * CRO_REGFILE_THREADS * CRO_REGFILE_ELEMENTS * r->iterations * (r->ctas - r->unpublished);
    for (const auto& kv : t.per_sm) {
        if (kv.second.mark) {
            if (r->bad_sms < 16) r->bad_sm[r->bad_sms] = (uint16_t)kv.first;
            r->bad_sms++;
        }
        sms->push_back(kv.second);
    }
    *faults = t.recs[0];
    std::stable_sort(faults->begin(), faults->end(), [](const cro_regfile_fault& x, const cro_regfile_fault& y) {
        return std::make_tuple(x.smid, x.iteration, x.element, x.warp, x.lane, x.slot) <
               std::make_tuple(y.smid, y.iteration, y.element, y.warp, y.lane, y.slot);
    });
    const bool all = r->unpublished || (r->failed_sms && r->failed_sms == r->sms_covered);
    const bool any = r->unpublished || r->failed_sms;
    r->verdict = all ? CRO_REGFILE_ALL : any ? CRO_REGFILE_SM : CRO_REGFILE_NONE;
    return r->status = any ? CRO_ERR_CHECKSUM : CRO_OK;
}
}  // namespace

std::string regfile_opts_error(const cro_regfile_opts& o) {
    const uint32_t iters = o.iterations ? o.iterations : kRegfileDefaultIterations;
    const bool inj_ok = !o.test_inject_mask ||
                        (o.test_inject_sm >= -1 && o.test_inject_sm < CRO_REGFILE_MAX_SMS && o.test_inject_warp >= -1 &&
                         o.test_inject_warp < CRO_REGFILE_THREADS / 32 && o.test_inject_lane >= -1 && o.test_inject_lane < 32 &&
                         o.test_inject_slot >= -1 && o.test_inject_slot < CRO_REGFILE_SLOTS &&
                         o.test_inject_element < CRO_REGFILE_ELEMENTS && o.test_inject_iteration < iters);
    if (iters > CRO_REGFILE_MAX_ITERATIONS || o.max_rounds > CRO_REGFILE_MAX_ROUNDS || o.deadline_ms < 0 || !inj_ok)
        return "register-file probe: iterations at most " + std::to_string(CRO_REGFILE_MAX_ITERATIONS) + ", max_rounds at most " +
               std::to_string(CRO_REGFILE_MAX_ROUNDS) + ", deadline_ms not negative, and an injection must name an SM id below " +
               std::to_string(CRO_REGFILE_MAX_SMS) + ", a warp below 8, a lane below 32 and a slot below " +
               std::to_string(CRO_REGFILE_SLOTS) + " (each or -1), element 0 or 1 and an iteration the call runs";
    return "";
}

int ctx_probe_regfile(cro_ctx* c, int idx, const cro_regfile_opts& o, cro_regfile_result* r, std::vector<cro_regfile_sm>* sms,
                      std::vector<cro_regfile_fault>* faults) {
    return probe_cells<RegfileProbe>(c, idx, o, r, sms, faults);
}

int classify_regfile(uint32_t iterations, uint64_t seed, uint32_t sm_count, uint64_t k, uint32_t rounds,
                     const cro_regfile_cta* ctas, uint64_t claims, const cro_regfile_fault* records, cro_regfile_result* r,
                     std::vector<cro_regfile_sm>* sms, std::vector<cro_regfile_fault>* faults) {
    RegfileProbe::Call call;
    call.iterations = iterations;
    return classify_cells<RegfileProbe>(call, seed, sm_count, k, &rounds, ctas, &claims, records, r, sms, faults);
}

int ctx_probe_regfile_uuid(cro_ctx* c, const char* uuid, const cro_regfile_opts& o, cro_regfile_result* r,
                           std::vector<cro_regfile_sm>* sms, std::vector<cro_regfile_fault>* faults, int cap) {
    return probe_cells_uuid<RegfileProbe>(c, uuid, o, r, sms, faults, cap);
}

}  // namespace cro
