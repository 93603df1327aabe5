// cell_report.hpp — the host side the memory-cell probes (the SRAM probe, sram_probe.cu, and the register-file probe,
// regfile_probe.cu) share: each round's CTA records taken into the legs and their SMs, each leg's coverage, records and
// marks, and the in-process, classify and helper forms of a call.  Each CTA publishes its counts per element, its last
// iteration's count and a fold; the device keeps mismatching cells per leg while the leg's record buffer has room.
//
// What a probe P gives the code below (Cta, a leg's totals and an SM's part in a leg have the SRAM probe's field names):
//   Opts, Result, Sm, Fault, Args    its option, result, per-SM, record and kernel argument types
//   Cta, Record                      host mirrors of what the device publishes per CTA and records per cell
//   Call                             what a call settles before its first launch (legs, iterations, ...) and keeps
//   kLegs, kElements, kRecords, kMaxSms, kPersistent, kIntermittent, kDefaultRounds
//   kName                            "<kName> probe" and "<kName> helper" in error texts
//   kId                              "cro.probe_<kId>" and "cro.probe_<kId>.helper" NVTX ranges, cro_probe_<kId>_uuid
//   kWire, kCalls, kSeeds            its helper command (helper_wire.h), call counter in Device and seed space
//   leg(r, l), leg(sm, l)            leg l of a result and of an SM
//   opts_error(o)                    why the in-process form refuses the options ("" when they pass)
//   helper_opts_error(o)             why the helper form refuses them before it spawns ("" leaves them to the helper)
//   plan(c, d, o, r, &call)          the call's launch setup on device d; a CRO error (with its text) when it cannot run
//   open(call, r)                    r's settings beyond seed, call and SM count, and each leg's closed form of the fold
//   grid(call, leg, sm_count)        CTAs per launch of a leg
//   args(o, call, leg, &a)           the leg's own argument fields
//   launch(call, leg, a, round, grid, stream)
//   round(call, R, leg, hc, grid, k)   what a round's CTA records hc add beyond the common fields
//   folds(leg)                       whether the leg's CTAs fold
//   close(r, tally, call, sms, faults)   the call's end: the SM list, faults, bad SMs and verdict
//   keep(r, from)                    the result fields beyond the common ones that a failed call keeps
#pragma once
#include <algorithm>
#include <map>
#include <set>
#include <string>
#include <vector>

#include "probe_internal.hpp"

namespace cro {

// What a call's legs leave for its verdict.
template <class P>
struct CellTally {
    std::map<uint32_t, typename P::Sm> per_sm;
    std::map<uint32_t, uint64_t> last[P::kLegs];            // per leg and SM: failed compares of the last iteration
    std::set<uint32_t> seen[P::kLegs];                      // per leg: distinct SMs; the lowest one's fold is the leg's
    std::vector<typename P::Record> recs[P::kLegs];         // per leg: the records the device kept
};

// One round of leg `leg` of call k: the grid CTA records hc into the leg's totals, t's per-SM and last-iteration counts
// and what P adds; *covered: the distinct SMs the leg has seen so far.  CRO_ERR_UNSUPPORTED (with the error text) when
// the device reports more SM ids than the result holds.
template <class P>
int take_cell_round(cro_ctx* c, const typename P::Cta* hc, int grid, uint64_t k, unsigned leg, typename P::Result* r,
                    CellTally<P>& t, typename P::Call& call, uint32_t* covered) {
    auto& R = P::leg(*r, leg);
    R.ctas += (uint32_t)grid;
    P::round(call, R, leg, hc, grid, k);
    uint64_t t0 = ~0ull, t1 = 0;
    for (int j = 0; j < grid; ++j) {
        const typename P::Cta& x = hc[(size_t)j];
        if (x.stamp != k) {
            R.unpublished++;
            continue;
        }
        if (x.nsmid > P::kMaxSms) {
            set_call_error(c, std::string(P::kName) + " probe: the device reports %nsmid = " + std::to_string(x.nsmid) +
                                  ", more SM ids than the " + std::to_string(P::kMaxSms) + " the result holds");
            return CRO_ERR_UNSUPPORTED;
        }
        r->nsmid = x.nsmid;
        t0 = std::min<uint64_t>(t0, x.t0);
        t1 = std::max<uint64_t>(t1, x.t1);
        const bool lowest = t.seen[leg].empty() || x.smid < *t.seen[leg].begin();
        t.seen[leg].insert(x.smid);
        typename P::Sm& S = t.per_sm[x.smid];
        S.smid = x.smid;
        auto& SL = P::leg(S, leg);
        SL.ctas++;
        for (unsigned e = 0; e < P::kElements; ++e) {
            SL.mismatches[e] += x.count[e];
            R.mismatches[e] += x.count[e];
        }
        t.last[leg][x.smid] += x.last;
        SL.ns += x.t1 > x.t0 ? x.t1 - x.t0 : 0;
        SL.cycles += x.cycles;
        if (!P::folds(leg)) continue;
        const bool fold_bad = x.fold_x != R.expect_xor || x.fold_s != R.expect_sum || x.fold_w != R.expect_wsum;
        SL.fold_mismatches += fold_bad ? 1 : 0;
        R.fold_mismatches += fold_bad ? 1 : 0;
        if (lowest) {
            R.fold_xor = x.fold_x;
            R.fold_sum = x.fold_s;
            R.fold_wsum = x.fold_w;
        }
    }
    if (t1 > t0) R.timer_ns += t1 - t0;
    *covered = R.sms_covered = (uint32_t)t.seen[leg].size();
    return CRO_OK;
}

// A leg after its last round: its coverage of sm_count SMs, the records kept of n_claims and each SM's mark
// (persistent: a compare of the last iteration failed; intermittent: only an earlier one, or only the fold).
template <class P>
void close_cell_leg(typename P::Result* r, unsigned leg, uint32_t sm_count, uint64_t n_claims, CellTally<P>& t) {
    auto& R = P::leg(*r, leg);
    R.complete = R.sms_covered >= sm_count ? 1u : 0u;
    R.recorded = std::min<uint64_t>(n_claims, P::kRecords);
    for (auto& kv : t.per_sm) {
        auto& SL = P::leg(kv.second, leg);
        if (!SL.ctas) continue;
        uint64_t any = SL.fold_mismatches;
        for (uint64_t m : SL.mismatches) any += m;
        SL.mark = t.last[leg][kv.first] ? P::kPersistent : any ? P::kIntermittent : 0u;
        if (SL.mark) R.failed_sms++;
    }
}

// The result of a call that checked nothing: zeroes but for what the call had settled before it stopped (`from`'s
// seed, call number, SM count, CUDA error and NVML health, and what P::keep adds).
template <class P>
void blank_cell_result(typename P::Result* r, const typename P::Result& from, std::vector<typename P::Sm>* sms,
                       std::vector<typename P::Fault>* faults) {
    const typename P::Result keep = from;
    memset(r, 0, sizeof *r);
    r->seed = keep.seed;
    r->call = keep.call;
    r->sm_count = keep.sm_count;
    r->cuda_error = keep.cuda_error;
    r->before = keep.before;
    r->after = keep.after;
    r->health = keep.health;
    P::keep(r, keep);
    sms->clear();
    faults->clear();
}

// The call's settings before anything runs, then P::open's.
template <class P>
void open_cell_call(const typename P::Call& call, uint64_t seed, uint64_t k, uint32_t sm_count, typename P::Result* r) {
    r->seed = seed;
    r->call = k;
    r->sm_count = sm_count;
    P::open(call, r);
}

// The in-process form: the call takes its number k from the device's counter only once P::plan succeeded, and gets
// the seed space_seed(d, P::kSeeds, k); then per leg one launch per coverage round.  NVML's SRAM health is read after
// the call's buffers are set up and before its first launch, and once that was read, after the launches on every way
// out.  Every return past the device guard sets wall_ns.
template <class P>
int probe_cells(cro_ctx* c, int idx, const typename P::Opts& o, typename P::Result* r, std::vector<typename P::Sm>* sms,
                std::vector<typename P::Fault>* faults) {
    using Cta = typename P::Cta;
    using Record = typename P::Record;
    const uint64_t t_call = now_ns();
    blank_cell_result<P>(r, typename P::Result{}, sms, faults);
    const std::string id = P::kId;
    Device* d = dev_at(c, idx);
    if (!d) {
        const std::string why = "a GPU attached after init is probed through the helper process, cro_probe_" + id + "_uuid";
        return r->status = unknown_device(c, idx, why.c_str());
    }
    const uint32_t max_rounds = o.max_rounds ? o.max_rounds : P::kDefaultRounds;
    const std::string why = P::opts_error(o);
    if (!why.empty()) {
        c->set_error(why);
        return r->status = CRO_ERR_INVALID_ARG;
    }
    DeviceGuard g = enter_device(c, idx);
    if (g.rc) return r->status = g.rc;
    Range nv(c, ("cro.probe_" + id).c_str());
    const std::string uuid(d->info.gpu_uuid, strnlen(d->info.gpu_uuid, sizeof d->info.gpu_uuid));
    const bool nvml = !(c->opts.flags & CRO_F_NO_NVML);
    CellTally<P> t;
    typename P::Call call{};
    bool held = false;
    cudaEvent_t ev[2] = {nullptr, nullptr};                  // the call's own, destroyed on every way out
    int rc = [&]() -> int {
        const int sm_count = d->plan.sm_count;
        const int e = P::plan(c, d, o, r, &call);
        if (e) return e;
        int max_grid = sm_count;
        for (unsigned leg = 0; leg < P::kLegs; ++leg)
            if (call.legs >> leg & 1u) max_grid = std::max(max_grid, P::grid(call, leg, sm_count));
        const uint64_t k = (d->*P::kCalls)++;
        open_cell_call<P>(call, space_seed(d, P::kSeeds, k), k, (uint32_t)sm_count, r);

        // [claims per leg][records per leg][CTA records], allocated per call
        const size_t rec_off = 64, rec_bytes = (size_t)P::kLegs * P::kRecords * sizeof(Record);
        const size_t cta_off = (rec_off + rec_bytes + 63) & ~(size_t)63;
        DeviceMem<unsigned char> b;
        CU_TRY(c, cudaMalloc(&b.p, cta_off + (size_t)max_grid * sizeof(Cta)));
        for (cudaEvent_t& x : ev) CU_TRY(c, cudaEventCreate(&x));
        cudaStream_t st = d->stream;
        CU_TRY(c, cudaMemsetAsync(b.p, 0, rec_off, st));
        typename P::Args a{};
        a.cta = reinterpret_cast<decltype(a.cta)>(b.p + cta_off);
        a.seed = r->seed;
        a.stamp = k;
        a.iterations = call.iterations;
        std::vector<Cta> hc((size_t)max_grid);
        if (nvml) identity::NvmlSramHealth(uuid, false, &r->before);
        held = true;

        for (unsigned leg = 0; leg < P::kLegs; ++leg) {
            if (!(call.legs >> leg & 1u)) continue;
            auto& R = P::leg(*r, leg);
            const int grid = P::grid(call, leg, sm_count);
            const size_t cta_bytes = (size_t)grid * sizeof(Cta);
            a.rec = reinterpret_cast<decltype(a.rec)>(b.p + rec_off) + (size_t)leg * P::kRecords;
            a.claims = reinterpret_cast<unsigned long long*>(b.p) + leg;
            P::args(o, call, leg, &a);
            auto launch = [&] { return P::launch(call, leg, a, R.rounds, grid, st); };
            auto fetch = [&] { return cudaMemcpyAsync(hc.data(), a.cta, cta_bytes, cudaMemcpyDeviceToHost, st); };
            auto take = [&](uint32_t* covered) { return take_cell_round<P>(c, hc.data(), grid, k, leg, r, t, call, covered); };
            const int e = coverage_rounds(c, d, ev, a.cta, cta_bytes, (uint32_t)sm_count, max_rounds, &R.rounds, &R.ns, launch, fetch, take);
            if (e) return e;
            unsigned long long n_claims = 0;
            CU_TRY(c, cudaMemcpy(&n_claims, a.claims, sizeof n_claims, cudaMemcpyDeviceToHost));
            close_cell_leg<P>(r, leg, (uint32_t)sm_count, n_claims, t);
            std::vector<Record>& recs = t.recs[leg];
            recs.resize((size_t)R.recorded);
            if (!recs.empty()) CU_TRY(c, cudaMemcpy(recs.data(), a.rec, recs.size() * sizeof(Record), cudaMemcpyDeviceToHost));
        }
        return CRO_OK;
    }();
    for (cudaEvent_t x : ev)
        if (x) cudaEventDestroy(x);
    if (rc == CRO_ERR_CUDA) r->cuda_error = (int32_t)cudaGetLastError();
    if (held && nvml) identity::NvmlSramHealth(uuid, true, &r->after);
    r->health = sram_health(r->before, r->after);
    if (rc) {
        blank_cell_result<P>(r, *r, sms, faults);
        r->wall_ns = now_ns() - t_call;
        return r->status = rc;
    }
    const int status = P::close(r, t, call, sms, faults);
    r->wall_ns = now_ns() - t_call;
    return status;
}

// cro_selftest_<kId>_classify: call k of a device of sm_count SMs (seed `seed`, the rest of its settings in `call`) as
// the in-process call classifies it, from the caller's rounds instead of launches: leg l of call.legs ran rounds[l]
// rounds of P::grid CTA records each, in leg order, and left claims[l] claims and min(claims[l], kRecords) records.
template <class P>
int classify_cells(typename P::Call call, uint64_t seed, uint32_t sm_count, uint64_t k, const uint32_t* rounds,
                   const typename P::Cta* ctas, const uint64_t* claims, const typename P::Record* records, typename P::Result* r,
                   std::vector<typename P::Sm>* sms, std::vector<typename P::Fault>* faults) {
    blank_cell_result<P>(r, typename P::Result{}, sms, faults);
    open_cell_call<P>(call, seed, k, sm_count, r);
    CellTally<P> t;
    for (unsigned leg = 0; leg < P::kLegs; ++leg) {
        if (!(call.legs >> leg & 1u)) continue;
        auto& R = P::leg(*r, leg);
        const int grid = P::grid(call, leg, (int)sm_count);
        for (uint32_t j = 0; j < rounds[leg]; ++j, ctas += grid) {
            ++R.rounds;
            uint32_t covered = 0;
            const int e = take_cell_round<P>(nullptr, ctas, grid, k, leg, r, t, call, &covered);
            if (e) {
                blank_cell_result<P>(r, *r, sms, faults);
                return r->status = e;
            }
        }
        close_cell_leg<P>(r, leg, sm_count, claims[leg], t);
        t.recs[leg].assign(records, records + R.recorded);
        records += R.recorded;
    }
    return P::close(r, t, call, sms, faults);
}

// The helper form: `croprobe-cli <kId>-raw` with the options and cap on argv (run_check_helper; a fresh seed base when
// P::kWire is seeded), once P::helper_opts_error passed them.  helper_ns is set only when run_check_helper returns CRO_OK.
template <class P>
int probe_cells_uuid(cro_ctx* c, const char* uuid, const typename P::Opts& o, typename P::Result* r,
                     std::vector<typename P::Sm>* sms, std::vector<typename P::Fault>* faults, int cap) {
    blank_cell_result<P>(r, typename P::Result{}, sms, faults);
    if (!uuid) return r->status = CRO_ERR_INVALID_ARG;
    const std::string why = P::helper_opts_error(o);
    if (!why.empty()) {
        set_call_error(c, why);
        return r->status = CRO_ERR_INVALID_ARG;
    }
    const std::string id = P::kId;
    uint64_t helper_ns = 0;
    if (run_check_helper(c, P::kWire, uuid, std::string(P::kName) + " helper", ("cro.probe_" + id + ".helper").c_str(), &o, cap,
                         o.deadline_ms, &helper_ns, r, faults, sms) == CRO_OK)
        r->helper_ns = helper_ns;
    return r->status;
}

}  // namespace cro
