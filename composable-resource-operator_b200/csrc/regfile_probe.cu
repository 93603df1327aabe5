// regfile_probe.cu — the register-file probe (cro_probe_regfile, cro_probe_regfile_uuid): every SM's registers held
// as 0 and as 1 across two barriers and checked word by word, and the SRAM ECC record NVML keeps.
#include <map>
#include <set>
#include <tuple>

#include "probe_internal.hpp"

namespace cro {

namespace {
// Iterations per CTA and launches when the caller gives none.  On an H100 80GB HBM3 at a 700 W limit
// (profiles/h100_700w_regfile_rate.jsonl) one iteration takes 51 us and one launch covers all 132 SMs, so 96 iterations
// cost about the SRAM probe's 5 ms (DESIGN.md "The register-file probe").
constexpr uint32_t kRegfileDefaultIterations = 96;
constexpr uint32_t kRegfileDefaultRounds = 4;

// The result of a call that checked nothing: zeroes but for what the call had settled before it stopped.
void blank_result(cro_regfile_result* r, const cro_regfile_result& from, std::vector<cro_regfile_sm>* sms,
                  std::vector<cro_regfile_fault>* faults) {
    const cro_regfile_result keep = from;
    memset(r, 0, sizeof *r);
    r->seed = keep.seed;
    r->call = keep.call;
    r->sm_count = keep.sm_count;
    r->iterations = keep.iterations;
    r->slots = CRO_REGFILE_SLOTS;
    r->threads = CRO_REGFILE_THREADS;
    r->num_regs = keep.num_regs;
    r->regs_per_sm = keep.regs_per_sm;
    r->cuda_error = keep.cuda_error;
    r->before = keep.before;
    r->after = keep.after;
    r->health = keep.health;
    sms->clear();
    faults->clear();
}

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

// What a call's rounds leave for its verdict.
struct RegfileTally {
    std::map<uint32_t, cro_regfile_sm> per_sm;
    std::map<uint32_t, uint64_t> last;                      // per SM: failed compares of the last iteration
    std::set<uint32_t> seen;
    uint32_t fold_sm = ~0u;                                 // the lowest SM seen, whose fold r reports
};

// One round of call k: the grid CTA records hc into r and t.  CRO_ERR_UNSUPPORTED (with the error text) when the device
// reports more SM ids than the result holds.
int take_regfile_round(cro_ctx* c, const cro_regfile_cta* hc, int grid, uint64_t k, cro_regfile_result* r, RegfileTally& t,
                       uint32_t* covered) {
    r->ctas += (uint32_t)grid;
    uint64_t t0 = ~0ull, t1 = 0;
    for (int j = 0; j < grid; ++j) {
        const cro_regfile_cta& x = hc[(size_t)j];
        if (x.stamp != k) {
            r->unpublished++;
            continue;
        }
        if (x.nsmid > CRO_REGFILE_MAX_SMS) {
            set_call_error(c, "register-file probe: the device reports %nsmid = " + std::to_string(x.nsmid) +
                                  ", more SM ids than the " + std::to_string(CRO_REGFILE_MAX_SMS) + " the result holds");
            return CRO_ERR_UNSUPPORTED;
        }
        r->nsmid = x.nsmid;
        t0 = std::min<uint64_t>(t0, x.t0);
        t1 = std::max<uint64_t>(t1, x.t1);
        t.seen.insert(x.smid);
        cro_regfile_sm& S = t.per_sm[x.smid];
        S.smid = x.smid;
        S.ctas++;
        for (int e = 0; e < CRO_REGFILE_ELEMENTS; ++e) {
            S.mismatches[e] += x.count[e];
            r->mismatches[e] += x.count[e];
        }
        t.last[x.smid] += x.last;
        S.ns += x.t1 > x.t0 ? x.t1 - x.t0 : 0;
        S.cycles += x.cycles;
        r->bits_checked += 32ull * CRO_REGFILE_SLOTS * CRO_REGFILE_THREADS * CRO_REGFILE_ELEMENTS * r->iterations;
        const bool fold_bad = x.fold_x != r->expect_xor || x.fold_s != r->expect_sum || x.fold_w != r->expect_wsum;
        S.fold_mismatches += fold_bad ? 1 : 0;
        r->fold_mismatches += fold_bad ? 1 : 0;
        if (x.smid < t.fold_sm) {
            t.fold_sm = x.smid;
            r->fold_xor = x.fold_x;
            r->fold_sum = x.fold_s;
            r->fold_wsum = x.fold_w;
        }
    }
    if (t1 > t0) r->timer_ns += t1 - t0;
    *covered = r->sms_covered = (uint32_t)t.seen.size();
    return CRO_OK;
}

// The call's end: coverage, each SM's mark (persistent: a compare of the last iteration failed; intermittent: only an
// earlier one, or only the fold), the records sorted, the bad SMs and the verdict.
int close_regfile_call(cro_regfile_result* r, RegfileTally& t, uint64_t n_claims, std::vector<cro_regfile_fault>* recs,
                       std::vector<cro_regfile_sm>* sms, std::vector<cro_regfile_fault>* faults) {
    r->complete = r->sms_covered >= r->sm_count ? 1u : 0u;
    for (auto& kv : t.per_sm) {
        cro_regfile_sm& S = kv.second;
        const uint64_t any = S.fold_mismatches + S.mismatches[0] + S.mismatches[1];
        S.mark = t.last[kv.first] ? CRO_REGFILE_PERSISTENT : any ? CRO_REGFILE_INTERMITTENT : 0u;
        if (S.mark) {
            if (r->bad_sms < 16) r->bad_sm[r->bad_sms] = (uint16_t)kv.first;
            r->bad_sms++;
        }
        sms->push_back(S);
    }
    r->failed_sms = r->bad_sms;
    recs->resize((size_t)std::min<uint64_t>(n_claims, CRO_REGFILE_RECORDS));
    *faults = *recs;
    std::stable_sort(faults->begin(), faults->end(), [](const cro_regfile_fault& x, const cro_regfile_fault& y) {
        return std::make_tuple(x.smid, x.iteration, x.element, x.warp, x.lane, x.slot) <
               std::make_tuple(y.smid, y.iteration, y.element, y.warp, y.lane, y.slot);
    });
    const bool all = r->unpublished || (r->failed_sms && r->failed_sms == r->sms_covered);
    const bool any = r->unpublished || r->failed_sms;
    r->verdict = all ? CRO_REGFILE_ALL : any ? CRO_REGFILE_SM : CRO_REGFILE_NONE;
    return r->status = any ? CRO_ERR_CHECKSUM : CRO_OK;
}

// The call's settings before anything runs.
void open_regfile_call(cro_regfile_result* r, uint64_t seed, uint64_t k, uint32_t sm_count, uint32_t iters) {
    r->seed = seed;
    r->call = k;
    r->sm_count = sm_count;
    r->iterations = iters;
    r->slots = CRO_REGFILE_SLOTS;
    r->threads = CRO_REGFILE_THREADS;
    closed_form(seed, iters, r);
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
    const uint64_t t_call = now_ns();
    blank_result(r, cro_regfile_result{}, sms, faults);
    Device* d = dev_at(c, idx);
    if (!d) return r->status = unknown_device(c, idx, "a GPU attached after init is probed through the helper process, cro_probe_regfile_uuid");
    const uint32_t iters = o.iterations ? o.iterations : kRegfileDefaultIterations;
    const uint32_t max_rounds = o.max_rounds ? o.max_rounds : kRegfileDefaultRounds;
    const std::string why = regfile_opts_error(o);
    if (!why.empty()) {
        c->set_error(why);
        return r->status = CRO_ERR_INVALID_ARG;
    }
    DeviceGuard g = enter_device(c, idx);
    if (g.rc) return r->status = g.rc;
    Range nv(c, "cro.probe_regfile");
    const std::string uuid(d->info.gpu_uuid, strnlen(d->info.gpu_uuid, sizeof d->info.gpu_uuid));
    const bool nvml = !(c->opts.flags & CRO_F_NO_NVML);
    RegfileTally t;
    std::vector<cro_regfile_fault> recs;
    uint64_t n_claims = 0;
    bool held = false;
    cudaEvent_t ev[2] = {nullptr, nullptr};                  // the call's own, destroyed on every way out
    int rc = [&]() -> int {
        const int sm_count = d->plan.sm_count;
        cudaFuncAttributes fa{};
        CU_TRY(c, regfile_plan(d->ordinal, &fa));
        int regs = 0;
        CU_TRY(c, cudaDeviceGetAttribute(&regs, cudaDevAttrMaxRegistersPerMultiprocessor, d->ordinal));
        r->num_regs = (uint32_t)fa.numRegs;
        r->regs_per_sm = (uint32_t)regs;
        const uint64_t k = d->regfile_calls++;
        open_regfile_call(r, space_seed(d, kSeedRegfile, k), k, (uint32_t)sm_count, iters);

        // [claims][records][CTA records], allocated per call
        const size_t rec_off = 64, cta_off = (rec_off + CRO_REGFILE_RECORDS * sizeof(cro_regfile_fault) + 63) & ~(size_t)63;
        const size_t cta_bytes = (size_t)sm_count * sizeof(cro_regfile_cta);
        DeviceMem<unsigned char> b;
        CU_TRY(c, cudaMalloc(&b.p, cta_off + cta_bytes));
        for (cudaEvent_t& x : ev) CU_TRY(c, cudaEventCreate(&x));
        cudaStream_t st = d->stream;
        CU_TRY(c, cudaMemsetAsync(b.p, 0, rec_off, st));
        RegfileArgs a{};
        a.claims = reinterpret_cast<unsigned long long*>(b.p);
        a.rec = reinterpret_cast<cro_regfile_fault*>(b.p + rec_off);
        a.cta = reinterpret_cast<cro_regfile_cta*>(b.p + cta_off);
        a.seed = r->seed;
        a.stamp = k;
        a.iterations = iters;
        a.inj_sm = o.test_inject_sm;
        a.inj_warp = o.test_inject_warp;
        a.inj_lane = o.test_inject_lane;
        a.inj_slot = o.test_inject_slot;
        a.inj_element = o.test_inject_element;
        a.inj_iter = o.test_inject_iteration;
        a.inj_mask = o.test_inject_mask;
        std::vector<cro_regfile_cta> hc((size_t)sm_count);
        if (nvml) identity::NvmlSramHealth(uuid, false, &r->before);
        held = true;
        auto launch = [&] { return launch_regfile(a, sm_count, st); };
        auto fetch = [&] { return cudaMemcpyAsync(hc.data(), a.cta, cta_bytes, cudaMemcpyDeviceToHost, st); };
        auto take = [&](uint32_t* covered) { return take_regfile_round(c, hc.data(), sm_count, k, r, t, covered); };
        const int e = coverage_rounds(c, d, ev, a.cta, cta_bytes, (uint32_t)sm_count, max_rounds, &r->rounds, &r->ns, launch, fetch, take);
        if (e) return e;
        CU_TRY(c, cudaMemcpy(&n_claims, a.claims, sizeof n_claims, cudaMemcpyDeviceToHost));
        recs.resize((size_t)std::min<uint64_t>(n_claims, CRO_REGFILE_RECORDS));
        if (!recs.empty()) CU_TRY(c, cudaMemcpy(recs.data(), a.rec, recs.size() * sizeof(cro_regfile_fault), cudaMemcpyDeviceToHost));
        return CRO_OK;
    }();
    for (cudaEvent_t x : ev)
        if (x) cudaEventDestroy(x);
    if (rc == CRO_ERR_CUDA) r->cuda_error = (int32_t)cudaGetLastError();
    if (held && nvml) identity::NvmlSramHealth(uuid, true, &r->after);
    r->health = sram_health(r->before, r->after);
    if (rc) {
        blank_result(r, *r, sms, faults);
        r->wall_ns = now_ns() - t_call;
        return r->status = rc;
    }
    const int status = close_regfile_call(r, t, n_claims, &recs, sms, faults);
    r->wall_ns = now_ns() - t_call;
    return status;
}

int classify_regfile(uint32_t iterations, uint64_t seed, uint32_t sm_count, uint64_t k, uint32_t rounds,
                     const cro_regfile_cta* ctas, uint64_t claims, const cro_regfile_fault* records, cro_regfile_result* r,
                     std::vector<cro_regfile_sm>* sms, std::vector<cro_regfile_fault>* faults) {
    blank_result(r, cro_regfile_result{}, sms, faults);
    open_regfile_call(r, seed, k, sm_count, iterations);
    RegfileTally t;
    for (uint32_t j = 0; j < rounds; ++j, ctas += sm_count) {
        ++r->rounds;
        uint32_t covered = 0;
        const int e = take_regfile_round(nullptr, ctas, (int)sm_count, k, r, t, &covered);
        if (e) {
            blank_result(r, *r, sms, faults);
            return r->status = e;
        }
    }
    std::vector<cro_regfile_fault> recs(records, records + std::min<uint64_t>(claims, CRO_REGFILE_RECORDS));
    return close_regfile_call(r, t, claims, &recs, sms, faults);
}

int ctx_probe_regfile_uuid(cro_ctx* c, const char* uuid, const cro_regfile_opts& o, cro_regfile_result* r,
                           std::vector<cro_regfile_sm>* sms, std::vector<cro_regfile_fault>* faults, int cap) {
    blank_result(r, cro_regfile_result{}, sms, faults);
    if (!uuid) return r->status = CRO_ERR_INVALID_ARG;
    const std::string why = regfile_opts_error(o);
    if (!why.empty()) {
        set_call_error(c, why);
        return r->status = CRO_ERR_INVALID_ARG;
    }
    uint64_t helper_ns = 0;
    if (run_check_helper(c, cro_wire_regfile, uuid, "register-file helper", "cro.probe_regfile.helper", &o, cap, o.deadline_ms,
                         &helper_ns, r, faults, sms) == CRO_OK)
        r->helper_ns = helper_ns;
    return r->status;
}

}  // namespace cro
