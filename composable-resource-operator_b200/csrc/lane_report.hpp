// lane_report.hpp — the host half of the per-thread report path the cross-lane and ALU probes share
// (xlane_probe.cu, alu_probe.cu): each launch's CTA entries and per-thread entries taken round by round, then the
// call's coverage, marks, sorted and capped records and verdict.  The device half is lane_tally.cuh.
//
// P names the probe's types and constants: Result, Sm, Fault, Thread, Cta; kLegs, kThreads, kThreadRecs, kRecords,
// kMaxSms, kPersistent, kIntermittent, kNone, kSm, kAll; kName (for errors) and ops(leg).  Result, Sm and the entries
// have the cross-lane probe's field names.
#pragma once
#include <algorithm>
#include <map>
#include <set>
#include <string>
#include <tuple>
#include <vector>

#include "probe_internal.hpp"

namespace cro {

// What a call's rounds leave for its verdict.
template <class P>
struct LaneTally {
    std::map<uint32_t, typename P::Sm> per_sm;
    std::map<uint32_t, uint64_t> last;                      // per SM: failed compares of the last iteration
    std::set<uint32_t> seen[P::kLegs];
    uint32_t fold_sm[P::kLegs];                             // the lowest SM seen per leg, whose fold r reports
    std::vector<typename P::Fault> recs;
    LaneTally() { std::fill(fold_sm, fold_sm + P::kLegs, ~0u); }
};

template <class P>
bool lane_any_failed(const typename P::Thread* ht, int grid, uint64_t k) {
    for (size_t i = 0; i < (size_t)grid * P::kThreads; ++i)
        if (ht[i].stamp == k && ht[i].count) return true;
    return false;
}

// One round of leg `leg` of call k: the grid CTAs' entries hc, their threads' entries ht and records hr (read only for
// threads that failed).  CRO_ERR_UNSUPPORTED (with the error text) when the device reports more SM ids than the
// result holds.
template <class P>
int take_lane_round(cro_ctx* c, unsigned leg, const typename P::Cta* hc, const typename P::Thread* ht, const typename P::Fault* hr,
                    int grid, uint64_t k, typename P::Result* r, LaneTally<P>& t, uint32_t* covered) {
    const uint32_t bit = 1u << leg;
    r->ctas += (uint32_t)grid;
    uint64_t t0 = ~0ull, t1 = 0;
    for (int j = 0; j < grid; ++j) {
        const typename P::Cta& x = hc[(size_t)j];
        if (x.stamp != k) {
            r->unpublished++;
            r->failed_legs |= bit;
            continue;
        }
        if (x.nsmid > P::kMaxSms) {
            set_call_error(c, std::string(P::kName) + ": the device reports %nsmid = " + std::to_string(x.nsmid) + ", more SM ids than the " +
                                  std::to_string(P::kMaxSms) + " the result holds");
            return CRO_ERR_UNSUPPORTED;
        }
        r->nsmid = x.nsmid;
        t0 = std::min<uint64_t>(t0, x.t0);
        t1 = std::max<uint64_t>(t1, x.t1);
        t.seen[leg].insert(x.smid);
        typename P::Sm& S = t.per_sm[x.smid];
        S.smid = x.smid;
        S.ctas++;
        S.ns += x.t1 > x.t0 ? x.t1 - x.t0 : 0;
        S.cycles += x.cycles;
        uint64_t fx = 0, fs = 0, fw = 0, n = 0;
        bool silent = false;
        for (size_t q = 0; q < P::kThreads; ++q) {
            const size_t i = (size_t)j * P::kThreads + q;
            const typename P::Thread& e = ht[i];
            if (e.stamp != k) {
                r->threads_unpublished++;
                silent = true;
                continue;
            }
            n += e.count;
            t.last[x.smid] += e.last;
            fx ^= e.fold_x;
            fs += e.fold_s;
            fw += e.fold_w;
            for (size_t m = 0; m < std::min<uint64_t>(e.count, P::kThreadRecs); ++m) t.recs.push_back(hr[i * P::kThreadRecs + m]);
        }
        S.mismatches[leg] += n;
        r->mismatches[leg] += n;
        r->ops_checked[leg] += (uint64_t)P::ops(leg) * P::kThreads * r->iterations;
        const bool fold_bad = !silent && (fx != r->expect[leg][0] || fs != r->expect[leg][1] || fw != r->expect[leg][2]);
        S.fold_mismatches += fold_bad ? 1 : 0;
        r->fold_mismatches[leg] += fold_bad ? 1 : 0;
        if (n || fold_bad || silent) {
            S.failed_legs |= bit;
            r->failed_legs |= bit;
        }
        if (x.smid < t.fold_sm[leg]) {
            t.fold_sm[leg] = x.smid;
            r->fold[leg][0] = fx;
            r->fold[leg][1] = fs;
            r->fold[leg][2] = fw;
        }
    }
    if (t1 > t0) r->timer_ns += t1 - t0;
    *covered = (uint32_t)t.seen[leg].size();
    return CRO_OK;
}

// The call's end: coverage, each SM's mark (persistent: a compare of the last iteration failed; intermittent: only an
// earlier one, only the fold, or a thread that did not publish), the records sorted and capped, the bad SMs and the
// verdict.
template <class P>
int close_lane_call(typename P::Result* r, LaneTally<P>& t, std::vector<typename P::Sm>* sms, std::vector<typename P::Fault>* faults) {
    uint32_t covered = ~0u;
    for (unsigned leg = 0; leg < P::kLegs; ++leg)
        if (r->legs >> leg & 1u) covered = std::min<uint32_t>(covered, (uint32_t)t.seen[leg].size());
    r->sms_covered = covered == ~0u ? 0 : covered;
    r->complete = r->sms_covered >= r->sm_count ? 1u : 0u;
    for (auto& kv : t.per_sm) {
        typename P::Sm& S = kv.second;
        S.mark = t.last[kv.first] ? P::kPersistent : S.failed_legs ? P::kIntermittent : 0u;
        if (S.mark) {
            if (r->bad_sms < 16) r->bad_sm[r->bad_sms] = (uint16_t)kv.first;
            r->bad_sms++;
        }
        sms->push_back(S);
    }
    r->failed_sms = r->bad_sms;
    *faults = std::move(t.recs);
    using F = typename P::Fault;
    std::stable_sort(faults->begin(), faults->end(), [](const F& x, const F& y) {
        return std::make_tuple(x.leg, x.smid, x.iteration, x.op, x.warp, x.lane) <
               std::make_tuple(y.leg, y.smid, y.iteration, y.op, y.warp, y.lane);
    });
    if (faults->size() > P::kRecords) faults->resize(P::kRecords);
    const bool silent = r->unpublished || r->threads_unpublished;
    const bool all = silent || (r->failed_sms && r->failed_sms == t.per_sm.size());
    const bool any = silent || r->failed_sms;
    r->verdict = all ? P::kAll : any ? P::kSm : P::kNone;
    return r->status = any ? CRO_ERR_CHECKSUM : CRO_OK;
}

}  // namespace cro
