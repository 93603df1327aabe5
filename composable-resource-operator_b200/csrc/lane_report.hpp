// lane_report.hpp — the host side the per-thread SM probes (the cross-lane probe, xlane_probe.cu, the ALU probe,
// alu_probe.cu, and the barrier probe, barrier_probe.cu) share: each launch's CTA entries and per-thread entries taken
// round by round, the call's coverage, marks, sorted and capped records and verdict, and the in-process, classify and
// helper forms of a call.  The device half is lane_tally.cuh.
//
// What a probe P gives the code below (Result, Sm and the entries have the cross-lane probe's field names):
//   Opts, Result, Sm, Fault, Thread, Cta, Args   its option, result, per-SM, record, entry and kernel argument types
//   Tables                           the call's host tables (an empty struct when it has none)
//   kLegs, kAllLegs, kThreads, kThreadRecs, kRecords, kMaxSms, kMaxIterations, kMaxRounds
//   kPersistent, kIntermittent, kNone, kSm, kAll   its marks and verdicts
//   kName                            "<kName> probe" and "<kName> helper" in error texts
//   kId                              "cro.probe_<kId>" and "cro.probe_<kId>.helper" NVTX ranges, cro_probe_<kId>_uuid
//   kWire                            its helper command's argv and frame (helper_wire.h), croprobe-cli <kId>-raw
//   kCalls, kSeeds                   its call counter in Device and its seed space
//   kDefaultIterations, kDefaultRounds
//   kBlobs                           host blobs each leg uploads (0 when it has no tables)
//   ops(leg)                         checks per thread and iteration of a leg
//   opts_error(o)                    why the options are refused ("" when they pass), both forms' argument check
//   plan(device, leg)                a leg's launch setup
//   grids(c, o, legs, sm_count, grid)   each run leg's grid; a CRO error (with its text) when a leg cannot run
//   launch(o, leg, args, grid, stream)  one launch of a leg
//   open(o, r, tables, timed)        the tables and r->expect (the closed form of every CTA's fold); with timed, the
//                                    tables' build time where the result keeps it
//   blobs(tables, leg)               the leg's blobs to upload, {host pointer, bytes} each
//   args(o, r, leg, blobs, &args)    the leg's own argument fields (blobs: where its blobs sit on the device)
//   no_new_sm_ends(leg)              a round of the leg that reaches no new SM ends the leg
//   close(r, tally, sms, faults)     the call's end: close_lane_call, or that and the probe's own
//   keep(r, from)                    the result fields beyond the common ones that a failed call keeps
#pragma once
#include <algorithm>
#include <array>
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
            set_call_error(c, std::string(P::kName) + " probe: the device reports %nsmid = " + std::to_string(x.nsmid) +
                                  ", more SM ids than the " + std::to_string(P::kMaxSms) + " the result holds");
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

template <class P>
uint32_t lane_legs(const typename P::Opts& o) {
    return o.legs ? o.legs : P::kAllLegs;
}
template <class P>
uint32_t lane_iterations(const typename P::Opts& o) {
    return o.iterations ? o.iterations : P::kDefaultIterations;
}

// The option limits every lane probe has: iterations, legs and max_rounds at most P's, deadline_ms not negative, and
// an injection that names a leg the call runs, an SM id below kMaxSms, a warp and a lane of the CTA (each or -1), an op
// of the leg and an iteration the call runs.
template <class P>
bool lane_opts_ok(const typename P::Opts& o) {
    const uint32_t iters = lane_iterations<P>(o);
    const int leg = o.test_inject_leg;
    const bool inj_ok = !o.test_inject_mask ||
                        (leg >= 0 && leg < (int)P::kLegs && (lane_legs<P>(o) >> leg & 1u) && o.test_inject_sm >= -1 &&
                         o.test_inject_sm < (int)P::kMaxSms && o.test_inject_warp >= -1 && o.test_inject_warp < (int)P::kThreads / 32 &&
                         o.test_inject_lane >= -1 && o.test_inject_lane < 32 && o.test_inject_op < P::ops(leg) &&
                         o.test_inject_iteration < iters);
    return iters <= P::kMaxIterations && o.legs <= P::kAllLegs && o.max_rounds <= P::kMaxRounds && o.deadline_ms >= 0 && inj_ok;
}

// The result of a call that checked nothing: zeroes but for what the call had settled before it stopped (`from`'s
// seed, call number, SM count, legs, iterations and CUDA error, and what P::keep adds).
template <class P>
void blank_lane_result(typename P::Result* r, const typename P::Result& from, std::vector<typename P::Sm>* sms,
                       std::vector<typename P::Fault>* faults) {
    const typename P::Result keep = from;
    memset(r, 0, sizeof *r);
    r->seed = keep.seed;
    r->call = keep.call;
    r->sm_count = keep.sm_count;
    r->legs = keep.legs;
    r->iterations = keep.iterations;
    r->cuda_error = keep.cuda_error;
    P::keep(r, keep);
    sms->clear();
    faults->clear();
}

// The call's settings before anything runs, then its tables and closed forms (P::open).
template <class P>
void open_lane_call(const typename P::Opts& o, uint64_t seed, uint64_t k, uint32_t sm_count, typename P::Result* r,
                    typename P::Tables& tb, bool timed) {
    r->seed = seed;
    r->call = k;
    r->sm_count = sm_count;
    r->legs = lane_legs<P>(o);
    r->iterations = lane_iterations<P>(o);
    P::open(o, r, tb, timed);
}

// A host blob a leg uploads, and where it sits in the call's device block.
struct LaneBlob {
    const void* p;
    size_t bytes;
    size_t at = 0;
};

// The in-process form: the call takes its number k from the device's counter only once every leg's plan and grid
// succeeded, and gets the seed space_seed(d, P::kSeeds, k); then per leg one launch per coverage round.  Every return
// past the device guard sets wall_ns.
template <class P>
int probe_lane_legs(cro_ctx* c, int idx, const typename P::Opts& o, typename P::Result* r, std::vector<typename P::Sm>* sms,
                    std::vector<typename P::Fault>* faults) {
    using Cta = typename P::Cta;
    using Thread = typename P::Thread;
    using Fault = typename P::Fault;
    const uint64_t t_call = now_ns();
    blank_lane_result<P>(r, typename P::Result{}, sms, faults);
    const std::string id = P::kId;
    Device* d = dev_at(c, idx);
    if (!d) {
        const std::string why = "a GPU attached after init is probed through the helper process, cro_probe_" + id + "_uuid";
        return r->status = unknown_device(c, idx, why.c_str());
    }
    const uint32_t iters = lane_iterations<P>(o);
    const uint32_t max_rounds = o.max_rounds ? o.max_rounds : P::kDefaultRounds;
    const uint32_t legs = lane_legs<P>(o);
    const std::string why = P::opts_error(o);
    if (!why.empty()) {
        c->set_error(why);
        return r->status = CRO_ERR_INVALID_ARG;
    }
    DeviceGuard g = enter_device(c, idx);
    if (g.rc) return r->status = g.rc;
    Range nv(c, ("cro.probe_" + id).c_str());
    LaneTally<P> t;
    cudaEvent_t ev[2] = {nullptr, nullptr};                  // the call's own, destroyed on every way out
    int rc = [&]() -> int {
        const int sm_count = d->plan.sm_count;
        for (unsigned leg = 0; leg < P::kLegs; ++leg)
            if (legs >> leg & 1u) CU_TRY(c, P::plan(d->ordinal, leg));
        int grid[P::kLegs] = {};
        const int eg = P::grids(c, o, legs, sm_count, grid);
        if (eg) return eg;
        int max_grid = sm_count;
        for (unsigned leg = 0; leg < P::kLegs; ++leg)
            if (legs >> leg & 1u) max_grid = std::max(max_grid, grid[leg]);
        const uint64_t k = (d->*P::kCalls)++;
        typename P::Tables tb;
        open_lane_call<P>(o, space_seed(d, P::kSeeds, k), k, (uint32_t)sm_count, r, tb, true);

        // [CTA entries][thread entries] (armed together every round), then [records], then each leg's blobs, allocated
        // per call
        const size_t n_thr = (size_t)max_grid * P::kThreads;
        const size_t cta_bytes = (size_t)max_grid * sizeof(Cta), thr_bytes = n_thr * sizeof(Thread);
        const size_t rec_off = (cta_bytes + thr_bytes + 255) & ~(size_t)255, rec_bytes = n_thr * P::kThreadRecs * sizeof(Fault);
        std::array<LaneBlob, P::kBlobs> blob[P::kLegs];
        size_t end = rec_off + rec_bytes;
        for (unsigned leg = 0; leg < P::kLegs; ++leg) {
            blob[leg] = P::blobs(tb, leg);
            for (LaneBlob& x : blob[leg]) {
                x.at = (end + 255) & ~(size_t)255;
                end = x.at + x.bytes;
            }
        }
        DeviceMem<unsigned char> b;
        CU_TRY(c, cudaMalloc(&b.p, end));
        for (const auto& of_leg : blob)
            for (const LaneBlob& x : of_leg)
                if (x.bytes) CU_TRY(c, cudaMemcpyAsync(b.p + x.at, x.p, x.bytes, cudaMemcpyHostToDevice, d->stream));
        for (cudaEvent_t& x : ev) CU_TRY(c, cudaEventCreate(&x));
        cudaStream_t st = d->stream;
        typename P::Args a{};
        a.cta = reinterpret_cast<Cta*>(b.p);
        a.rec = reinterpret_cast<Fault*>(b.p + rec_off);
        a.stamp = k;
        a.iterations = iters;
        a.inj_sm = o.test_inject_sm;
        a.inj_warp = o.test_inject_warp;
        a.inj_lane = o.test_inject_lane;
        a.inj_op = o.test_inject_op;
        a.inj_iter = o.test_inject_iteration;
        std::vector<unsigned char> head(cta_bytes + thr_bytes);
        std::vector<Fault> hr(n_thr * P::kThreadRecs);
        for (unsigned leg = 0; leg < P::kLegs; ++leg) {
            if (!(legs >> leg & 1u)) continue;
            const int n = grid[leg];
            // The round's entries sit where the grid's CTA and thread entries end: CTA entries first, then threads.
            const size_t cb = (size_t)n * sizeof(Cta), tbytes = (size_t)n * P::kThreads * sizeof(Thread);
            a.thr = reinterpret_cast<Thread*>(b.p + cb);
            const auto* hc = reinterpret_cast<const Cta*>(head.data());
            const auto* ht = reinterpret_cast<const Thread*>(head.data() + cb);
            std::array<const void*, P::kBlobs> on_dev;
            std::transform(blob[leg].begin(), blob[leg].end(), on_dev.begin(),
                           [&](const LaneBlob& x) -> const void* { return b.p + x.at; });
            P::args(o, *r, leg, on_dev, &a);
            a.inj_mask = o.test_inject_mask && o.test_inject_leg == (int)leg ? o.test_inject_mask : 0ull;
            auto launch = [&] { return P::launch(o, leg, a, n, st); };
            auto fetch = [&] { return cudaMemcpyAsync(head.data(), b.p, cb + tbytes, cudaMemcpyDeviceToHost, st); };
            auto take = [&](uint32_t* covered) -> int {
                if (lane_any_failed<P>(ht, n, k))
                    CU_TRY(c, cudaMemcpy(hr.data(), a.rec, (size_t)n * P::kThreads * P::kThreadRecs * sizeof(Fault),
                                         cudaMemcpyDeviceToHost));
                const size_t before = t.seen[leg].size();
                const int e = take_lane_round<P>(c, leg, hc, ht, hr.data(), n, k, r, t, covered);
                if (P::no_new_sm_ends(leg) && t.seen[leg].size() == before) *covered = (uint32_t)sm_count;
                return e;
            };
            uint32_t rounds = 0;
            const int e = coverage_rounds(c, d, ev, b.p, cb + tbytes, (uint32_t)sm_count, max_rounds, &rounds, &r->leg_ns[leg], launch,
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
        blank_lane_result<P>(r, *r, sms, faults);
        r->wall_ns = now_ns() - t_call;
        return r->status = rc;
    }
    const int status = P::close(r, t, sms, faults);
    r->wall_ns = now_ns() - t_call;
    return status;
}

// cro_selftest_<kId>_classify: call k of a device of sm_count SMs with the options o (legs and iterations given) and
// seed `seed` as the in-process call classifies it, from the caller's rounds instead of launches: `rounds` rounds per
// leg of o's legs, in leg order, each sm_count CTA entries, sm_count * kThreads thread entries and kThreadRecs records
// per thread entry.  table_ns stays 0.
template <class P>
int classify_lane_legs(const typename P::Opts& o, uint64_t seed, uint32_t sm_count, uint64_t k, uint32_t rounds,
                       const typename P::Cta* ctas, const typename P::Thread* threads, const typename P::Fault* records,
                       typename P::Result* r, std::vector<typename P::Sm>* sms, std::vector<typename P::Fault>* faults) {
    blank_lane_result<P>(r, typename P::Result{}, sms, faults);
    typename P::Tables tb;
    open_lane_call<P>(o, seed, k, sm_count, r, tb, false);
    LaneTally<P> t;
    const size_t n_thr = (size_t)sm_count * P::kThreads;
    for (unsigned leg = 0; leg < P::kLegs; ++leg) {
        if (!(r->legs >> leg & 1u)) continue;
        for (uint32_t j = 0; j < rounds; ++j, ctas += sm_count, threads += n_thr, records += n_thr * P::kThreadRecs) {
            ++r->rounds;
            uint32_t covered = 0;
            const int e = take_lane_round<P>(nullptr, leg, ctas, threads, records, (int)sm_count, k, r, t, &covered);
            if (e) {
                blank_lane_result<P>(r, *r, sms, faults);
                return r->status = e;
            }
        }
    }
    return P::close(r, t, sms, faults);
}

// The helper form: `croprobe-cli <kId>-raw` with a fresh seed base, the options and cap on argv (run_check_helper).
// helper_ns is set only when run_check_helper returns CRO_OK.
template <class P>
int probe_lane_legs_uuid(cro_ctx* c, const char* uuid, const typename P::Opts& o, typename P::Result* r,
                         std::vector<typename P::Sm>* sms, std::vector<typename P::Fault>* faults, int cap) {
    blank_lane_result<P>(r, typename P::Result{}, sms, faults);
    if (!uuid) return r->status = CRO_ERR_INVALID_ARG;
    const std::string why = P::opts_error(o);
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
