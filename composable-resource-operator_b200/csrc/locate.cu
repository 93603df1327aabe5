// locate.cu — the fault locator (cro_locate_faults): names the words behind a failed probe.
#include <map>

#include "probe_internal.hpp"

namespace cro {

namespace {
constexpr int kLocateSlots = 2 * CRO_LOCATE_PASSES + CRO_LOCATE_PASSES;   // [2p + h] compare sweeps, then closed forms

// The report of a call that located nothing: zeroes but for the sweep size it got to (0 before it knew it).
void blank_report(cro_fault_report* rep, std::vector<cro_fault_word>* words, uint64_t sweep_bytes) {
    memset(rep, 0, sizeof *rep);
    rep->sweep_bytes = sweep_bytes;
    words->clear();
}

// The seeds whose closed forms a call generates: one per distinct seed of a compared half, in pass then half order.
// Closed form k sits in slot 2 * CRO_LOCATE_PASSES + k.
std::vector<uint64_t> closed_form_seeds(const cro_fault_report& rep) {
    std::vector<uint64_t> seeds;
    for (uint32_t p = 0; p < rep.n_passes; ++p)
        for (int h = 0; h < 2; ++h)
            if ((rep.pass[p].halves >> h & 1u) && std::find(seeds.begin(), seeds.end(), rep.pass[p].seed[h]) == seeds.end())
                seeds.push_back(rep.pass[p].seed[h]);
    return seeds;
}

// The report from what a call's compare passes wrote (hv, the host mirror after the fetch): per pass its counts, bit
// flips, granules and folds, the merged word list, and whether the recorded words explain each compared half's fold
// exactly.  rep already holds the call's setup: sweep_bytes, n_passes and each pass's halves, skipped, seeds and invert.
void collect_faults(const MismatchView& hv, cro_fault_report* rep, std::vector<cro_fault_word>* words) {
    const uint64_t n = rep->sweep_bytes / 8;
    const std::vector<uint64_t> cf_seeds = closed_form_seeds(*rep);
    std::map<uint64_t, cro_fault_word> merged;
    bool complete = true;
    for (uint32_t p = 0; p < rep->n_passes; ++p) {
        cro_locate_pass& P = rep->pass[p];
        P.mismatches = hv.ctr[p].mismatches;
        P.recorded = std::min<uint64_t>(hv.ctr[p].claims, kLocateRecords);
        if (P.recorded != P.mismatches) complete = false;
        for (int b = 0; b < 64; ++b) rep->bit_flips[b] += hv.ctr[p].bits[b];
        for (uint64_t k = 0; k < hv.gran_words; ++k) P.granules += (uint64_t)__builtin_popcountll(hv.gran[p * hv.gran_words + k]);
        uint64_t dx[2] = {0, 0}, ds[2] = {0, 0}, dw[2] = {0, 0};
        for (uint64_t k = 0; k < P.recorded; ++k) {
            const LocateRecord& R = hv.rec[(size_t)p * kLocateRecords + k];
            const int h = R.word >= n ? 1 : 0;
            const uint64_t i = R.word - h * n, delta = R.actual - R.expected;
            dx[h] ^= R.actual ^ R.expected;
            ds[h] += delta;
            dw[h] += delta * (2 * i + 1);
            auto it = merged.find(R.word);
            if (it == merged.end()) merged[R.word] = cro_fault_word{R.word, R.expected, R.actual, 1u << p, 0};
            else it->second.passes |= 1u << p;
        }
        for (int h = 0; h < 2; ++h) {
            if (!(P.halves >> h & 1u)) continue;
            const SweepOut& s = hv.slots[2 * p + h];
            P.words_scanned += s.n_words;
            P.scan_ns += s.t1 - s.t0;
            P.fold_xor[h] = s.x;
            P.fold_sum[h] = s.s;
            P.fold_wsum[h] = s.w;
            const size_t k = (size_t)(std::find(cf_seeds.begin(), cf_seeds.end(), P.seed[h]) - cf_seeds.begin());
            SweepOut cf = hv.slots[2 * CRO_LOCATE_PASSES + k];
            if (P.invert) cf = complement_fold(cf, n);
            if ((s.x ^ cf.x) != dx[h] || s.s - cf.s != ds[h] || s.w - cf.w != dw[h]) complete = false;
        }
    }
    for (int b = 0; b < 64; ++b)
        if (rep->bit_flips[b]) rep->flip_or |= 1ull << b;
    rep->located = merged.size();
    for (const auto& kv : merged) words->push_back(kv.second);
    rep->complete = complete ? 1u : 0u;
}

// The verdict of a collected report, and its status: CRO_ERR_CHECKSUM when any pass mismatched.
int fault_status(cro_fault_report* rep) {
    rep->verdict = fault_verdict(*rep);
    bool any = false;
    for (uint32_t p = 0; p < rep->n_passes; ++p) any |= rep->pass[p].mismatches != 0;
    return rep->status = any ? CRO_ERR_CHECKSUM : CRO_OK;
}
}  // namespace

uint32_t fault_verdict(const cro_fault_report& r) {
    const uint32_t np = std::min<uint32_t>(r.n_passes, CRO_LOCATE_PASSES);
    for (uint32_t p = 1; p < np; ++p)
        if (r.pass[p].mismatches) return CRO_FAULTS_PERSISTENT;
    if (np == 0 || r.pass[0].mismatches == 0) return CRO_FAULTS_NONE;
    return np > 1 ? CRO_FAULTS_NOT_REPRODUCED : CRO_FAULTS_UNCLASSIFIED;
}

int selftest_locate_collect(uint64_t sweep_bytes, const cro_locate_pass* passes, uint32_t n_passes, const cro_locate_counters* ctr,
                            const cro_locate_record* records, const uint64_t* granules, uint64_t granule_words,
                            const cro_sweep_slot* slots, cro_fault_report* rep, std::vector<cro_fault_word>* words) {
    blank_report(rep, words, sweep_bytes);
    rep->n_passes = n_passes;
    for (uint32_t p = 0; p < n_passes; ++p) {
        cro_locate_pass& P = rep->pass[p];
        P.halves = passes[p].halves;
        P.skipped = passes[p].skipped;
        P.seed[0] = passes[p].seed[0];
        P.seed[1] = passes[p].seed[1];
        P.invert = passes[p].invert;
    }
    if (closed_form_seeds(*rep).size() > CRO_LOCATE_PASSES) {    // more closed forms than the call has slots for
        blank_report(rep, words, sweep_bytes);
        return rep->status = CRO_ERR_INVALID_ARG;
    }
    // the device's layout: kLocateRecords records per pass, the compare slots then the closed forms
    std::vector<LocateCounters> c(CRO_LOCATE_PASSES);
    std::vector<LocateRecord> rec((size_t)CRO_LOCATE_PASSES * kLocateRecords);
    std::vector<unsigned long long> gran(CRO_LOCATE_PASSES * granule_words);
    std::vector<SweepOut> s(kLocateSlots);
    memcpy(c.data(), ctr, n_passes * sizeof *ctr);
    for (uint32_t p = 0; p < n_passes; ++p) {
        const uint64_t k = std::min<uint64_t>(ctr[p].claims, kLocateRecords);
        if (k) memcpy(&rec[(size_t)p * kLocateRecords], records, k * sizeof *records);
        records += k;
    }
    if (granule_words) memcpy(gran.data(), granules, n_passes * granule_words * 8);
    memcpy(s.data(), slots, kLocateSlots * sizeof *slots);
    collect_faults(MismatchView{c.data(), gran.data(), s.data(), rec.data(), nullptr, granule_words}, rep, words);
    return fault_status(rep);
}

int ctx_locate(cro_ctx* c, int idx, const cro_locate_opts& o, cro_fault_report* rep, std::vector<cro_fault_word>* words) {
    blank_report(rep, words, 0);
    Device* d = dev_at(c, idx);
    if (!d) return rep->status = unknown_device(c, idx, "a GPU probed through the helper process has no resident region to locate faults in");
    if (o.flags & ~CRO_LOCATE_RETEST) return rep->status = CRO_ERR_INVALID_ARG;
    DeviceGuard g = enter_device(c, idx);
    if (g.rc) return rep->status = g.rc;
    int rc = [&]() -> int {
        int r = ensure_region(c, d);
        if (r) return r;
        const uint64_t S = d->sweep_bytes, n = S / 8;
        if (o.test_force_count && (o.test_force_first >= 2 * n || o.test_force_count > 2 * n - o.test_force_first))
            return CRO_ERR_INVALID_ARG;
        if (!d->locate) d->locate.reset(new MismatchBuffer);
        MismatchBuffer& mb = *d->locate;
        const SweepScratch& sc = mb.scratch[0];
        if ((r = mb.ensure(c, CRO_LOCATE_PASSES, 2 * S, kLocateSlots, 0, std::max({d->plan.locate.grid, d->plan.expect.grid, 1}), 1)))
            return r;
        if ((r = mb.zero(c, d->stream))) return r;
        const MismatchView dv = mb.dev();

        const bool retest = (o.flags & CRO_LOCATE_RETEST) != 0;
        const uint32_t np = retest ? CRO_LOCATE_PASSES : 1;
        const uint64_t rseed = space_seed(d, kSeedRetest, 0);
        rep->sweep_bytes = S;
        rep->n_passes = np;
        rep->retest_seed = retest ? rseed : 0;
        unsigned char* half[2] = {d->region, d->region + S};
        for (uint32_t p = 0; p < np; ++p) {
            cro_locate_pass& P = rep->pass[p];
            P.invert = p == 2 ? ~0ull : 0ull;
            if (p == 0) {
                for (int h = 0; h < 2; ++h) {
                    if (d->half_known[h]) { P.halves |= 1u << h; P.seed[h] = d->half_seed[h]; }
                    else P.skipped |= 1u << h;
                }
            } else {
                P.halves = 3;
                P.seed[0] = P.seed[1] = rseed;
                const Params fp{ProbeParams{rseed, d->nonce_cur}, nullptr};
                for (int h = 0; h < 2; ++h)
                    CU_TRY(c, launch_fill(d->plan, half[h], S, fp, sc, nullptr, d->stream, p == 2));
                CU_TRY(c, launch_force_words(d->region, o.test_force_first, o.test_force_count, o.test_force_and,
                                             o.test_force_or, d->plan.sm_count, d->stream));
                c->launches += 2 + (o.test_force_count ? 1 : 0);
                d->half_known[0] = d->half_known[1] = false;   // the probe's pattern is gone
                d->filled = false;
            }
            for (int h = 0; h < 2; ++h) {
                if (!(P.halves >> h & 1u)) continue;
                CU_TRY(c, launch_locate(d->plan, half[h], S, h * n, P.seed[h], P.invert, dv.check((int)p), sc, &dv.slots[2 * p + h],
                                        d->stream));
                c->launches++;
            }
        }
        const std::vector<uint64_t> cf_seeds = closed_form_seeds(*rep);
        for (size_t k = 0; k < cf_seeds.size(); ++k) {
            CU_TRY(c, launch_expected(d->plan, S, Params{ProbeParams{cf_seeds[k], d->nonce_cur}, nullptr}, sc,
                                      &dv.slots[2 * CRO_LOCATE_PASSES + k], d->stream));
            c->launches++;
        }
        if ((r = mb.fetch(c, d->stream)) || (r = wait_stream(c, d))) return r;
        collect_faults(mb.host(), rep, words);
        return CRO_OK;
    }();
    if (rc) {
        blank_report(rep, words, rep->sweep_bytes);
        return rep->status = rc;
    }
    return fault_status(rep);
}

}  // namespace cro
