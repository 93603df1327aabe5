// sm_legs.hpp — the per-leg bookkeeping of the per-SM arithmetic probes (the compute probe, compute_probe.cu, and the
// precision probe, precision_probe.cu): what one round's CTA records add to a leg and to its SMs, the marks and the
// slowest SM of a finished leg, and the call's verdict.  Sm is cro_compute_sm or cro_precision_sm (smid and leg[],
// one cro_compute_sm_leg per leg); the leg totals are a cro_compute_leg in both.
#pragma once
#include <algorithm>
#include <map>
#include <tuple>
#include <vector>

#include "probe_internal.hpp"

namespace cro {

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
            c->set_error(std::string(who) + ": the device reports %nsmid = " + std::to_string(x.nsmid) + ", more SM ids than the " +
                         std::to_string(max_sms) + " the coverage bitmaps hold");
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

}  // namespace cro
