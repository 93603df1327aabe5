// sm_legs.hpp — the host side the per-SM arithmetic probes (the compute probe, compute_probe.cu, the precision probe,
// precision_probe.cu, the sparse probe, sparse_probe.cu, and the warp-MMA probe, warpmma_probe.cu) share: what one
// round's CTA records add to a leg and to its SMs, the marks and the slowest SM of a finished leg, the call's verdict,
// and the in-process and helper forms of a call.  Sm is cro_compute_sm, cro_precision_sm, cro_sparse_sm or
// cro_warpmma_sm (smid and leg[], one cro_compute_sm_leg per leg); the leg totals are a cro_compute_leg in all four.
#pragma once
#include <algorithm>
#include <map>
#include <string>
#include <tuple>
#include <vector>

#include "probe_internal.hpp"

namespace cro {

// cro_sm_cta is the public mirror of ComputeCta (cro_selftest_sm_legs_classify hands the records over as they are).
static_assert(sizeof(cro_sm_cta) == sizeof(ComputeCta) && offsetof(cro_sm_cta, stamp) == offsetof(ComputeCta, stamp) &&
                  offsetof(cro_sm_cta, t0) == offsetof(ComputeCta, t0) && offsetof(cro_sm_cta, t1) == offsetof(ComputeCta, t1) &&
                  offsetof(cro_sm_cta, cycles) == offsetof(ComputeCta, cycles) &&
                  offsetof(cro_sm_cta, mismatches) == offsetof(ComputeCta, mismatches) &&
                  offsetof(cro_sm_cta, fold_mismatches) == offsetof(ComputeCta, fold_mismatches) &&
                  offsetof(cro_sm_cta, fold) == offsetof(ComputeCta, fold) && offsetof(cro_sm_cta, smid) == offsetof(ComputeCta, smid) &&
                  offsetof(cro_sm_cta, nsmid) == offsetof(ComputeCta, nsmid),
              "cro_sm_cta mirrors ComputeCta");

// One round of leg `leg` of call k: the CTA records hc (grid of them, each ops / grid operations) into R and per_sm,
// and the round's coverage bitmap (sm_words words) into R.sms_covered and *covered.  A CTA whose stamp is not k did not
// publish.  *fold_sm tracks the lowest SM id seen, whose CTA's fold R.fold reports.  CRO_ERR_UNSUPPORTED (with the
// error text, `who` naming the probe) when the device reports more SM ids than max_sms.
template <class Sm>
int take_leg_round(cro_ctx* c, const char* who, const std::vector<ComputeCta>& hc, uint64_t k, uint32_t leg, uint64_t ops,
                   const unsigned long long* hbits, int sm_words, uint32_t max_sms, cro_compute_leg& R, uint32_t* nsmid,
                   uint32_t* fold_sm, std::map<uint32_t, Sm>& per_sm, uint32_t* covered) {
    R.ctas += (uint32_t)hc.size();
    R.ops += ops;
    uint64_t t0 = ~0ull, t1 = 0;
    for (const ComputeCta& x : hc) {
        if (x.stamp != k) {
            R.unpublished++;
            continue;
        }
        if (x.nsmid > max_sms) {
            set_call_error(c, std::string(who) + ": the device reports %nsmid = " + std::to_string(x.nsmid) +
                                  ", more SM ids than the " + std::to_string(max_sms) + " the coverage bitmaps hold");
            return CRO_ERR_UNSUPPORTED;
        }
        *nsmid = x.nsmid;
        t0 = std::min<uint64_t>(t0, x.t0);
        t1 = std::max<uint64_t>(t1, x.t1);
        Sm& S = per_sm[x.smid];
        S.smid = x.smid;
        cro_compute_sm_leg& SL = S.leg[leg];
        SL.ctas++;
        SL.mismatches += x.mismatches;
        SL.fold_mismatches += x.fold_mismatches;
        SL.ns += x.t1 > x.t0 ? x.t1 - x.t0 : 0;
        SL.cycles += x.cycles;
        R.mismatches += x.mismatches;
        R.fold_mismatches += x.fold_mismatches;
        if (x.smid < *fold_sm) {
            *fold_sm = x.smid;
            R.fold = x.fold;
        }
    }
    if (t1 > t0) R.timer_ns += t1 - t0;
    R.sms_covered = 0;
    for (int w = 0; w < sm_words; ++w) R.sms_covered += (uint32_t)__builtin_popcountll(hbits[w]);
    *covered = R.sms_covered;
    return CRO_OK;
}

// A finished leg: each SM's mark (persistent: the last iteration was wrong; intermittent: only the fold was), the
// failed SMs, and the slowest SM's cycles per iteration against the median SM's.
template <class Sm>
void finish_leg(cro_compute_leg& R, std::map<uint32_t, Sm>& per_sm, uint32_t leg, uint32_t iterations) {
    std::vector<std::pair<uint64_t, uint32_t>> per_iter;
    for (auto& kv : per_sm) {
        cro_compute_sm_leg& SL = kv.second.leg[leg];
        if (!SL.ctas) continue;
        SL.mark = SL.mismatches ? CRO_COMPUTE_PERSISTENT : SL.fold_mismatches ? CRO_COMPUTE_INTERMITTENT : 0u;
        if (SL.mark) R.failed_sms++;
        per_iter.push_back({SL.cycles / ((uint64_t)SL.ctas * iterations), kv.first});
    }
    if (!per_iter.empty()) {
        std::vector<uint64_t> v;
        for (auto& p : per_iter) v.push_back(p.first);
        std::sort(v.begin(), v.end());
        const uint64_t median = v[v.size() / 2];
        auto worst = per_iter.front();
        for (auto& p : per_iter)
            if (p.first > worst.first) worst = p;
        R.slowest_sm = worst.second;
        R.slow_permille = median ? (uint32_t)std::min<uint64_t>(worst.first * 1000 / median, 0xFFFFFFFFu) : 0u;
    }
}

// The call's verdict from its legs (all: a leg with an unpublished CTA or failed on every SM it covered; sm: any other
// failure), the bad SMs, *sms by SM id and *faults by (leg, smid, row, col).  Returns the call's status.
template <class Result, class Sm, class Fault>
int close_call(Result* r, uint32_t n_legs, const std::map<uint32_t, Sm>& per_sm, std::vector<Sm>* sms, std::vector<Fault>* faults) {
    bool all = false, any = false;
    for (uint32_t leg = 0; leg < n_legs; ++leg) {
        const cro_compute_leg& R = r->leg[leg];
        if (!(r->legs >> leg & 1u)) continue;
        if (R.unpublished || (R.failed_sms && R.failed_sms == R.sms_covered)) all = true;
        if (R.unpublished || R.failed_sms) any = true;
    }
    for (auto& kv : per_sm) {
        bool bad = false;
        for (const cro_compute_sm_leg& SL : kv.second.leg) bad = bad || SL.mark != 0;
        if (bad && r->bad_sms < 16) r->bad_sm[r->bad_sms] = (uint16_t)kv.first;
        if (bad) r->bad_sms++;
        sms->push_back(kv.second);
    }
    std::sort(faults->begin(), faults->end(), [](const Fault& x, const Fault& y) {
        return std::make_tuple(x.leg, x.smid, x.row, x.col) < std::make_tuple(y.leg, y.smid, y.row, y.col);
    });
    r->verdict = all ? CRO_COMPUTE_ALL : any ? CRO_COMPUTE_SM : CRO_COMPUTE_NONE;
    return r->status = any ? CRO_ERR_CHECKSUM : CRO_OK;
}

// One leg of call k once it is launched: rounds(take) runs its coverage rounds, calling take(&covered) with each round's
// grid CTA records in hc and its coverage bitmap, then the claims count, in hbits; then the leg's coverage, the records
// copy_faults(dst, n) copies in (the first min(claims, P::kRecords)) and the marks of finish_leg.  The in-process call
// and cro_selftest_sm_legs_classify both run every leg through here.
template <class P, class Rounds, class CopyFaults>
int take_leg(cro_ctx* c, const char* who, const std::vector<ComputeCta>& hc, const unsigned long long* hbits, uint64_t k,
             uint32_t leg, uint32_t iterations, cro_compute_leg& R, uint32_t* nsmid, std::map<uint32_t, typename P::Sm>& per_sm,
             std::vector<typename P::Fault>* faults, Rounds rounds, CopyFaults copy_faults) {
    constexpr int kSmWords = P::kMaxSms / 64;
    const uint32_t grid = (uint32_t)hc.size();
    uint32_t fold_sm = ~0u;
    auto take = [&](uint32_t* covered) -> int {
        return take_leg_round(c, who, hc, k, leg, P::ops(leg) * iterations * (uint64_t)grid, hbits, kSmWords, P::kMaxSms, R,
                              nsmid, &fold_sm, per_sm, covered);
    };
    const int e = rounds(take);
    if (e) return e;
    R.complete = R.sms_covered >= grid ? 1u : 0u;
    R.recorded = std::min<uint64_t>(hbits[kSmWords], P::kRecords);
    if (R.recorded) {
        std::vector<typename P::Fault> f((size_t)R.recorded);
        const int ef = copy_faults(f.data(), f.size());
        if (ef) return ef;
        faults->insert(faults->end(), f.begin(), f.end());
    }
    finish_leg(R, per_sm, leg, iterations);
    return CRO_OK;
}

// What a probe P gives the calls below:
//   Opts, Result, Sm, Fault, Args    its option, result, per-SM, record and kernel argument types
//   Tile                             the element type of its answer tiles (Args::expect points into them)
//   kName                            "compute", "precision", "sparse", "warpmma": "<kName> probe" and "<kName> helper" in
//                                    error texts
//   kWire                            its helper command's argv and frame (helper_wire.h), croprobe-cli <kName>-raw
//   kLegs, kAllLegs, kMaxSms, kRecords, kAnswers, kCalls (its call counter in Device), kSeeds (its seed space)
//   kDefaultIterations, kDefaultRounds, kAluLeg[leg] (the leg runs alu_iterations; with any such leg, Opts has
//                                    alu_iterations and P kDefaultAluIterations)
//   elements(answer), expected(answer, seed, out), fold(answer, tile)   an answer's tile: size, values, the fold one
//                                                                       iteration of a CTA adds when all is right
//   answer(leg), ops(leg)            a leg's answer and operations per CTA and iteration
//   launch(leg, args, grid, stream)  one launch of a leg
//   opts_error(opts)                 why the options are refused ("" when they pass), both forms' argument check
//   test_args(opts, leg, &args)      the launch's test fields beyond the accumulator injection (none: an empty body)

// The result of a call that computed nothing: zeroes but for what the call had settled before it stopped (`from`'s
// seed, call number, SM count and legs).
template <class Result, class Sm, class Fault>
void blank_result(Result* r, const Result from, std::vector<Sm>* sms, std::vector<Fault>* faults) {
    memset(r, 0, sizeof *r);
    r->seed = from.seed;
    r->call = from.call;
    r->sm_count = from.sm_count;
    r->legs = from.legs;
    sms->clear();
    faults->clear();
}

template <class P>
constexpr bool has_alu_legs() {
    for (bool alu : P::kAluLeg)
        if (alu) return true;
    return false;
}

// Iterations per CTA of each leg: the options' or the defaults.
template <class P>
void leg_iterations(const typename P::Opts& o, uint32_t (&iters)[P::kLegs]) {
    const uint32_t ti = o.iterations ? o.iterations : P::kDefaultIterations;
    for (uint32_t l = 0; l < P::kLegs; ++l) iters[l] = ti;
    if constexpr (has_alu_legs<P>()) {
        const uint32_t ai = o.alu_iterations ? o.alu_iterations : P::kDefaultAluIterations;
        for (uint32_t l = 0; l < P::kLegs; ++l)
            if (P::kAluLeg[l]) iters[l] = ai;
    }
}

// The in-process form: call k of the device gets the seed space_seed(d, P::kSeeds, k), its answer tiles computed here
// (timed into host_ref_ns), and one launch per leg and coverage round, one CTA per SM.
template <class P>
int probe_sm_legs(cro_ctx* c, int idx, const typename P::Opts& o, typename P::Result* r, std::vector<typename P::Sm>* sms,
                  std::vector<typename P::Fault>* faults) {
    using Fault = typename P::Fault;
    constexpr int kSmWords = P::kMaxSms / 64;
    blank_result(r, typename P::Result{}, sms, faults);
    Device* d = dev_at(c, idx);
    if (!d) return r->status = unknown_device(c, idx, "a GPU probed through the helper process cannot be given kernels from here");
    const uint32_t legs = o.legs ? o.legs : P::kAllLegs;
    uint32_t iters[P::kLegs];
    leg_iterations<P>(o, iters);
    const bool inj = o.test_inject_mask != 0;
    const std::string why = P::opts_error(o);
    if (!why.empty()) {
        c->set_error(why);
        return r->status = CRO_ERR_INVALID_ARG;
    }
    const uint32_t max_rounds = o.max_rounds ? o.max_rounds : P::kDefaultRounds;
    DeviceGuard g = enter_device(c, idx);
    if (g.rc) return r->status = g.rc;
    const std::string who = std::string(P::kName) + " probe";
    std::map<uint32_t, typename P::Sm> per_sm;
    cudaEvent_t ev[2] = {nullptr, nullptr};     // the call's own, destroyed on every way out
    int rc = [&]() -> int {
        const int grid = d->plan.sm_count;
        const uint64_t k = (d->*P::kCalls)++;
        const uint64_t seed = space_seed(d, P::kSeeds, k);
        r->seed = seed;
        r->call = k;
        r->sm_count = (uint32_t)grid;
        r->legs = legs;
        size_t tile_at[P::kAnswers + 1] = {0};
        for (int a = 0; a < P::kAnswers; ++a) tile_at[a + 1] = tile_at[a] + (size_t)P::elements(a);
        std::vector<typename P::Tile> tiles(tile_at[P::kAnswers]);
        const uint64_t h0 = now_ns();
        for (int a = 0; a < P::kAnswers; ++a) P::expected(a, seed, tiles.data() + tile_at[a]);
        r->host_ref_ns = now_ns() - h0;
        uint64_t fold[P::kAnswers];
        for (int a = 0; a < P::kAnswers; ++a) fold[a] = P::fold(a, tiles.data() + tile_at[a]);

        // [tiles][per leg: sm bitmap, claims][per leg: records][CTA records], allocated per call
        const size_t tile_bytes = tiles.size() * sizeof(typename P::Tile);
        const size_t ctr_off = tile_bytes, ctr_bytes = (size_t)P::kLegs * (kSmWords + 1) * 8;
        const size_t rec_off = ctr_off + ctr_bytes, rec_bytes = (size_t)P::kLegs * P::kRecords * sizeof(Fault);
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

        for (uint32_t leg = 0; leg < P::kLegs; ++leg) {
            if (!(legs >> leg & 1u)) continue;
            cro_compute_leg& R = r->leg[leg];
            const int answer = P::answer(leg);
            typename P::Args a{};
            a.expect = reinterpret_cast<decltype(a.expect)>(b.p) + tile_at[answer];
            a.cta = cta;
            a.sm_bits = ctr + (size_t)leg * (kSmWords + 1);
            a.claims = a.sm_bits + kSmWords;
            a.rec = reinterpret_cast<Fault*>(b.p + rec_off) + (size_t)leg * P::kRecords;
            a.seed = seed;
            a.stamp = k;
            a.iterations = iters[leg];
            a.inj_sm = o.test_inject_sm;
            a.inj_row = o.test_inject_row;
            a.inj_col = o.test_inject_col;
            a.inj_iter = o.test_inject_iteration;
            a.inj_mask = (inj && (uint32_t)o.test_inject_leg == leg) ? o.test_inject_mask : 0;
            P::test_args(o, leg, &a);
            R.iterations = iters[leg];
            R.expect_fold = (uint64_t)iters[leg] * fold[answer];
            auto launch = [&] { return P::launch(leg, a, grid, st); };
            auto fetch = [&] {
                cudaError_t e = cudaMemcpyAsync(hc.data(), cta, cta_bytes, cudaMemcpyDeviceToHost, st);
                return e ? e : cudaMemcpyAsync(hbits, a.sm_bits, sizeof hbits, cudaMemcpyDeviceToHost, st);
            };
            auto rounds = [&](auto take) {
                return coverage_rounds(c, d, ev, cta, cta_bytes, (uint32_t)grid, max_rounds, &R.rounds, &R.ns, launch, fetch, take);
            };
            auto copy_faults = [&](Fault* f, size_t n) -> int {
                CU_TRY(c, cudaMemcpy(f, a.rec, n * sizeof(Fault), cudaMemcpyDeviceToHost));
                return CRO_OK;
            };
            const int e = take_leg<P>(c, who.c_str(), hc, hbits, k, leg, iters[leg], R, &r->nsmid, per_sm, faults, rounds, copy_faults);
            if (e) return e;
        }
        return CRO_OK;
    }();
    for (cudaEvent_t x : ev)
        if (x) cudaEventDestroy(x);
    if (rc) {
        blank_result(r, *r, sms, faults);
        return r->status = rc;
    }
    return close_call(r, P::kLegs, per_sm, sms, faults);
}

// cro_selftest_sm_legs_classify: call k of a device of `grid` SMs as the in-process call classifies it, from the
// caller's rounds instead of launches.  Leg l of `legs` ran rounds[l] rounds (grid records of ctas and kMaxSms / 64
// words of sm_bits each, in leg order) and left claims[l] claims and min(claims[l], kRecords) records.
template <class P>
int classify_sm_legs(uint32_t legs, const uint32_t* iterations, uint32_t grid, uint64_t k, const uint32_t* rounds,
                     const cro_sm_cta* ctas, const uint64_t* sm_bits, const uint64_t* claims, const typename P::Fault* records,
                     typename P::Result* r, std::vector<typename P::Sm>* sms, std::vector<typename P::Fault>* faults) {
    using Fault = typename P::Fault;
    constexpr int kSmWords = P::kMaxSms / 64;
    blank_result(r, typename P::Result{}, sms, faults);
    r->call = k;
    r->sm_count = grid;
    r->legs = legs;
    const std::string who = std::string(P::kName) + " probe";
    std::map<uint32_t, typename P::Sm> per_sm;
    std::vector<ComputeCta> hc((size_t)grid);
    unsigned long long hbits[kSmWords + 1];
    const int rc = [&]() -> int {
        for (uint32_t leg = 0; leg < P::kLegs; ++leg) {
            if (!(legs >> leg & 1u)) continue;
            cro_compute_leg& R = r->leg[leg];
            R.iterations = iterations[leg];
            hbits[kSmWords] = claims[leg];
            auto each_round = [&](auto take) -> int {
                for (uint32_t j = 0; j < rounds[leg]; ++j, ctas += grid, sm_bits += kSmWords) {
                    memcpy(hc.data(), ctas, (size_t)grid * sizeof(ComputeCta));
                    memcpy(hbits, sm_bits, kSmWords * sizeof(uint64_t));
                    ++R.rounds;
                    uint32_t covered = 0;
                    const int e = take(&covered);
                    if (e) return e;
                }
                return CRO_OK;
            };
            auto copy_faults = [&](Fault* f, size_t n) -> int {
                std::copy(records, records + n, f);
                records += n;
                return CRO_OK;
            };
            const int e = take_leg<P>(nullptr, who.c_str(), hc, hbits, k, leg, iterations[leg], R, &r->nsmid, per_sm, faults,
                                      each_round, copy_faults);
            if (e) return e;
        }
        return CRO_OK;
    }();
    if (rc) {
        blank_result(r, *r, sms, faults);
        return r->status = rc;
    }
    return close_call(r, P::kLegs, per_sm, sms, faults);
}

// The helper form: `croprobe-cli <kName>-raw` with a fresh seed base, the options and cap on argv (run_check_helper).
template <class P>
int probe_sm_legs_uuid(cro_ctx* c, const char* uuid, const typename P::Opts& o, int deadline_ms, typename P::Result* r,
                       std::vector<typename P::Sm>* sms, std::vector<typename P::Fault>* faults, int cap, uint64_t* helper_ns) {
    blank_result(r, typename P::Result{}, sms, faults);
    *helper_ns = 0;
    if (!uuid) return r->status = CRO_ERR_INVALID_ARG;
    const std::string why = P::opts_error(o);
    if (!why.empty()) {
        set_call_error(c, why);
        return r->status = CRO_ERR_INVALID_ARG;
    }
    const std::string name = P::kName;
    run_check_helper(c, P::kWire, uuid, name + " helper", ("cro.probe_" + name + ".helper").c_str(), &o, cap, deadline_ms,
                     helper_ns, r, faults, sms);
    return r->status;
}

}  // namespace cro
