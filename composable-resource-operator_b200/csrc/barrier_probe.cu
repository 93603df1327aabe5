// barrier_probe.cu — the barrier probe (cro_probe_barrier, cro_probe_barrier_uuid): every SM's named barriers, mbarrier
// phases and transaction counts, and cluster barriers with async remote stores, one launch per leg.  The host builds
// the call's table here; every check it lists is exact and independent of the order the threads ran in.
#include "barrier_kernels.cuh"
#include "lane_report.hpp"

namespace cro {

namespace barrier {
namespace {

typedef uint64_t u64;
constexpr unsigned kT = CRO_BARRIER_THREADS;

// The seeded word k (0 .. 3) of (leg, row, thread).
u64 word(u64 seed, unsigned leg, unsigned row, unsigned k, unsigned t) {
    return pattern_word(seed, ((((u64)leg * 256 + row) * 4 + k) << 8) | t);
}
// nw of the 8 warps, in a seeded order: the first nw of a Fisher-Yates shuffle.
void warp_order(u64 seed, unsigned leg, unsigned row, unsigned (&perm)[8]) {
    for (unsigned i = 0; i < 8; ++i) perm[i] = i;
    for (unsigned i = 7; i > 0; --i) std::swap(perm[i], perm[word(seed, leg, row, 2, i) % (i + 1)]);
}
uint32_t mask_of(const unsigned (&perm)[8], unsigned from, unsigned to) {
    uint32_t m = 0;
    for (unsigned i = from; i < to; ++i) m |= 1u << perm[i];
    return m;
}
// The sel-th thread (ascending) of the warps in mask.
unsigned nth_thread(uint32_t warps, unsigned sel) {
    for (unsigned t = 0; t < kT; ++t)
        if (warps >> (t >> 5) & 1u) {
            if (sel == 0) return t;
            --sel;
        }
    return 0;
}
bool in(uint32_t warps, unsigned t) { return warps >> (t >> 5) & 1u; }

void bar_row(u64 seed, unsigned r, cro_barrier_row& R, u64* w) {
    const unsigned leg = CRO_BARRIER_LEG_BAR;
    unsigned perm[8];
    warp_order(seed, leg, r, perm);
    R.form = CRO_BARRIER_FORM_POPC + r / 16;
    R.bar = r % 16;
    if (R.form == CRO_BARRIER_FORM_ARRIVE) {
        const unsigned nw = 2 + r % 7, np = 1 + (unsigned)(word(seed, leg, r, 3, 1) % (nw - 1));
        R.producers = mask_of(perm, 0, np);
        R.warps = mask_of(perm, np, nw);
        R.count = 32 * nw;
        for (unsigned t = 0; t < kT; ++t)
            if (in(R.producers, t)) w[2 * t] = (word(seed, leg, r, 0, t) & 0xFFFFFF00ull) | (r + 1);
        return;
    }
    const unsigned nw = 1 + r % 8;
    R.warps = mask_of(perm, 0, nw);
    R.count = 32 * nw;
    const unsigned kind = r % 5, one = nth_thread(R.warps, (unsigned)(word(seed, leg, r, 3, 0) % R.count));
    unsigned ones = 0;
    for (unsigned t = 0; t < kT; ++t) {
        if (!in(R.warps, t)) continue;
        const unsigned p = kind == 0 ? 1u : kind == 1 ? 0u : kind == 2 ? (t == one) : kind == 3 ? (t != one) : (unsigned)(word(seed, leg, r, 1, t) & 1u);
        R.pred[t >> 5] |= p << (t & 31);
        ones += p;
    }
    R.expect = R.form == CRO_BARRIER_FORM_POPC ? ones : R.form == CRO_BARRIER_FORM_AND ? (ones == R.count) : (ones > 0);
}

void mbar_row(u64 seed, unsigned r, cro_barrier_row& R, u64* w) {
    const unsigned leg = CRO_BARRIER_LEG_MBAR;
    unsigned perm[8];
    warp_order(seed, leg, r, perm);
    R.form = CRO_BARRIER_FORM_TICKET + r / 2;
    const unsigned nw = 1 + (unsigned)(word(seed, leg, r, 3, 0) % 8), n = 32 * nw;
    R.warps = mask_of(perm, 0, nw);
    R.held = nth_thread(R.warps, (unsigned)(word(seed, leg, r, 3, 1) % n));
    R.phases = 1;
    switch (R.form) {
        case CRO_BARRIER_FORM_TICKET:
            R.held = (unsigned)(word(seed, leg, r, 3, 1) % kT);
            R.count = n + 1;
            break;
        case CRO_BARRIER_FORM_COUNT:
            R.phases = 2 + (unsigned)(word(seed, leg, r, 3, 2) % 7);
            for (unsigned t = 0; t < kT; ++t)
                if (in(R.warps, t)) {
                    w[2 * t] = 1 + word(seed, leg, r, 0, t) % 4;
                    R.count += (uint32_t)w[2 * t];
                }
            break;
        case CRO_BARRIER_FORM_DROP:
            R.phases = 2;
            R.count = n;
            for (unsigned t = 0; t < kT; ++t)
                if (in(R.warps, t) && t != R.held) w[2 * t] = word(seed, leg, r, 0, t) & 1u;
            break;
        default:   // TX
            R.phases = 1 + (unsigned)(word(seed, leg, r, 3, 2) % 4);
            R.count = 1;
            R.arriver = (unsigned)(word(seed, leg, r, 3, 3) % kT);
            for (unsigned t = 0; t < kT; ++t)
                if (in(R.warps, t)) {
                    w[2 * t] = 1 + word(seed, leg, r, 0, t) % 64;
                    R.expect += w[2 * t];
                }
            break;
    }
}

void cluster_row(u64 seed, unsigned r, unsigned cluster, cro_barrier_row& R, u64* w) {
    const unsigned leg = CRO_BARRIER_LEG_CLUSTER;
    const u64 M32 = 0xFFFFFFFFull;
    R.form = r < kCbarRows ? CRO_BARRIER_FORM_CBAR : CRO_BARRIER_FORM_ST_B32 + (r - kCbarRows);
    if (R.form == CRO_BARRIER_FORM_CBAR) {
        for (unsigned k = 0; k < cluster; ++k) R.next_rank[k] = (uint8_t)((k + 1) % cluster);
        for (unsigned t = 0; t < kT; ++t) w[2 * t] = (word(seed, leg, r, 0, t) & 0xFFFFFF00ull) | (r + 1);
        return;
    }
    if (R.form <= CRO_BARRIER_FORM_ST_V4) {
        static const unsigned kBytes[4] = {4, 8, 8, 16};
        R.count = kT * kBytes[R.form - CRO_BARRIER_FORM_ST_B32];
        for (unsigned t = 0; t < kT; ++t) {
            const u64 a = word(seed, leg, r, 0, t), b = word(seed, leg, r, 1, t);
            w[2 * t] = R.form == CRO_BARRIER_FORM_ST_B32 ? a & M32 : a;
            w[2 * t + 1] = R.form == CRO_BARRIER_FORM_ST_V4 ? b : 0;
        }
        return;
    }
    const unsigned f = R.form, slots = 1 + (unsigned)(word(seed, leg, r, 3, 0) % 8);
    const bool wide = f == CRO_BARRIER_FORM_RED_ADD64;
    R.arriver = slots;
    R.count = kT * (wide ? 8 : 4);
    unsigned per[8] = {0};
    for (unsigned t = 0; t < kT; ++t) per[t % slots]++;
    const u64 bound = 2000 + word(seed, leg, r, 3, 1) % 1000;   // inc / dec: one bound for every thread
    for (unsigned s = 0; s < slots; ++s) {
        const u64 x = word(seed, leg, r, 1, s);
        R.slot_init[s] = f == CRO_BARRIER_FORM_RED_INC ? x % 1000 : f == CRO_BARRIER_FORM_RED_DEC ? per[s] + x % 1000 : wide ? x : x & M32;
    }
    for (unsigned s = 0; s < slots; ++s) R.slot_expect[s] = R.slot_init[s];
    for (unsigned t = 0; t < kT; ++t) {
        const u64 a = word(seed, leg, r, 0, t), b = word(seed, leg, r, 2, t) & M32;
        u64 v = wide ? a : a & M32;
        if (f == CRO_BARRIER_FORM_RED_AND) v |= b;
        if (f == CRO_BARRIER_FORM_RED_OR) v &= b;
        if (f == CRO_BARRIER_FORM_RED_INC || f == CRO_BARRIER_FORM_RED_DEC) v = bound;
        w[2 * t] = v;
        u64& d = R.slot_expect[t % slots];
        const int32_t sd = (int32_t)(uint32_t)d, sv = (int32_t)(uint32_t)v;
        switch (f) {
            case CRO_BARRIER_FORM_RED_ADD: d = (d + v) & M32; break;
            case CRO_BARRIER_FORM_RED_ADD64: d += v; break;
            case CRO_BARRIER_FORM_RED_MIN: d = std::min(d, v); break;
            case CRO_BARRIER_FORM_RED_MAX: d = std::max(d, v); break;
            case CRO_BARRIER_FORM_RED_MINS: d = (uint32_t)std::min(sd, sv); break;
            case CRO_BARRIER_FORM_RED_MAXS: d = (uint32_t)std::max(sd, sv); break;
            case CRO_BARRIER_FORM_RED_AND: d &= v; break;
            case CRO_BARRIER_FORM_RED_OR: d |= v; break;
            case CRO_BARRIER_FORM_RED_XOR: d ^= v; break;
            case CRO_BARRIER_FORM_RED_INC: d = d >= v ? 0 : d + 1; break;
            default: d = (d == 0 || d > v) ? v : d - 1; break;
        }
    }
}

}  // namespace

void table(unsigned leg, u64 seed, unsigned cluster, cro_barrier_row* rows, u64* words) {
    for (unsigned r = 0; r < kOps[leg]; ++r) {
        rows[r] = cro_barrier_row{};
        u64* w = words + (size_t)r * kT * 2;
        std::fill(w, w + kT * 2, 0ull);
        if (leg == CRO_BARRIER_LEG_BAR) bar_row(seed, r, rows[r], w);
        else if (leg == CRO_BARRIER_LEG_MBAR) mbar_row(seed, r, rows[r], w);
        else cluster_row(seed, r, cluster, rows[r], w);
    }
}

// Every value thread t folds in row r, in the device's order (rank: the CTA's cluster rank; getctarank is not folded).
template <class F>
void folded(unsigned leg, const cro_barrier_row& R, const u64* w, unsigned t, F f) {
    switch (R.form) {
        case CRO_BARRIER_FORM_ARRIVE:
            if (in(R.warps, t))
                for (unsigned p = 0; p < kT; ++p)
                    if (in(R.producers, p)) f(w[2 * p]);
            return;
        case CRO_BARRIER_FORM_POPC: case CRO_BARRIER_FORM_AND: case CRO_BARRIER_FORM_OR:
            if (in(R.warps, t)) f(R.expect);
            return;
        case CRO_BARRIER_FORM_CBAR: f(w[2 * t]); return;
        default: break;
    }
    if (leg == CRO_BARRIER_LEG_MBAR) {
        for (unsigned j = 0; j < R.phases; ++j) {
            if (R.form == CRO_BARRIER_FORM_TICKET && in(R.warps, t)) {
                f(1);
                f(t);
            }
            f(0);
            f(1);
            f(1);
        }
        return;
    }
    f(1);
    if (R.form <= CRO_BARRIER_FORM_ST_V4) {
        f(w[2 * t]);
        f(w[2 * t + 1]);
    } else if (t < R.arriver) {
        f(R.slot_expect[t]);
    }
}

}  // namespace barrier

namespace {
// Iterations per CTA and leg when the caller gives none, and launches per leg.  On an H100 80GB HBM3 at a 700 W limit
// (profiles/h100_700w_barrier_rate.jsonl) one iteration of the three legs takes about 0.28 ms of launches (BAR 244 us,
// MBAR 10 us, CLUSTER 27 us), so 16 iterations cost about the 5 ms the SRAM, register-file, cross-lane and ALU probes take.
constexpr uint32_t kBarrierDefaultIterations = 16;
constexpr uint32_t kBarrierDefaultRounds = 4;
constexpr uint32_t kBarrierDefaultCluster = 2;
constexpr size_t kThreadRecs = CRO_BARRIER_THREAD_RECORDS;

// The barrier probe's types and constants for the shared report path (lane_report.hpp).
struct BarrierReport {
    using Result = cro_barrier_result;
    using Sm = cro_barrier_sm;
    using Fault = cro_barrier_fault;
    using Thread = cro_barrier_thread;
    using Cta = cro_barrier_cta;
    static constexpr unsigned kLegs = CRO_BARRIER_LEGS, kThreads = CRO_BARRIER_THREADS, kThreadRecs = CRO_BARRIER_THREAD_RECORDS,
                              kRecords = CRO_BARRIER_RECORDS, kMaxSms = CRO_BARRIER_MAX_SMS, kPersistent = CRO_BARRIER_PERSISTENT,
                              kIntermittent = CRO_BARRIER_INTERMITTENT, kNone = CRO_BARRIER_NONE, kSm = CRO_BARRIER_SM,
                              kAll = CRO_BARRIER_ALL;
    static constexpr const char* kName = "barrier probe";
    static unsigned ops(unsigned leg) { return barrier::kOps[leg]; }
};

uint32_t legs_of(const cro_barrier_opts& o) { return o.legs ? o.legs : CRO_BARRIER_ALL_LEGS; }
uint32_t cluster_of(const cro_barrier_opts& o) { return o.cluster ? o.cluster : kBarrierDefaultCluster; }

void blank_result(cro_barrier_result* r, const cro_barrier_result& from, std::vector<cro_barrier_sm>* sms,
                  std::vector<cro_barrier_fault>* faults) {
    const cro_barrier_result keep = from;
    memset(r, 0, sizeof *r);
    r->seed = keep.seed;
    r->call = keep.call;
    r->sm_count = keep.sm_count;
    r->legs = keep.legs;
    r->iterations = keep.iterations;
    r->cluster = keep.cluster;
    r->cuda_error = keep.cuda_error;
    r->table_ns = keep.table_ns;
    sms->clear();
    faults->clear();
}

struct Tables {
    std::vector<cro_barrier_row> rows[CRO_BARRIER_LEGS];
    std::vector<uint64_t> words[CRO_BARRIER_LEGS];
};

// The legs' tables and the closed form of every CTA's fold.
void open_barrier_call(cro_barrier_result* r, uint64_t seed, uint64_t k, uint32_t sm_count, uint32_t legs, uint32_t iters,
                       uint32_t cluster, Tables& tb) {
    const uint64_t t0 = now_ns();
    r->seed = seed;
    r->call = k;
    r->sm_count = sm_count;
    r->legs = legs;
    r->iterations = iters;
    r->cluster = cluster;
    for (unsigned leg = 0; leg < CRO_BARRIER_LEGS; ++leg) {
        if (!(legs >> leg & 1u)) continue;
        const unsigned n = barrier::kOps[leg];
        tb.rows[leg].resize(n);
        tb.words[leg].resize((size_t)n * CRO_BARRIER_THREADS * 2);
        barrier::table(leg, seed, cluster, tb.rows[leg].data(), tb.words[leg].data());
        uint64_t x = 0, s = 0, f = 0;
        for (uint64_t op = 0; op < n; ++op)
            for (unsigned t = 0; t < CRO_BARRIER_THREADS; ++t)
                barrier::folded(leg, tb.rows[leg][op], tb.words[leg].data() + op * CRO_BARRIER_THREADS * 2, t, [&](uint64_t v) {
                    x ^= v;
                    s += v;
                    f += v * (2 * op + 1);
                });
        r->expect[leg][0] = x;
        r->expect[leg][1] = s;
        r->expect[leg][2] = f;
    }
    r->table_ns = now_ns() - t0;
}

// The report path's verdict, then the barrier probe's own: the kept timeout records, the coverage, the (SM, peer SM)
// pairs of every kept CLUSTER record (taken before the records are sorted and capped, so BAR and MBAR records cannot
// crowd them out), and LINK when only CLUSTER checks failed on a strict subset of the SMs.  A cluster cannot use an SM
// whose GPC has no room for the whole cluster, so the call's coverage is the CTA-local legs' when one ran, and the
// CLUSTER leg's own is cluster_sms.
int close_barrier_call(cro_barrier_result* r, LaneTally<BarrierReport>& t, std::vector<cro_barrier_sm>* sms,
                       std::vector<cro_barrier_fault>* faults) {
    std::set<std::pair<uint32_t, uint32_t>> pairs;
    for (const cro_barrier_fault& f : t.recs) {
        r->timeouts += f.kind == CRO_BARRIER_KIND_TIMEOUT ? 1 : 0;
        if (f.leg == CRO_BARRIER_LEG_CLUSTER) pairs.insert({f.smid, f.peer_smid});
    }
    r->cluster_sms = (uint32_t)t.seen[CRO_BARRIER_LEG_CLUSTER].size();
    const int status = close_lane_call<BarrierReport>(r, t, sms, faults);
    if (r->legs & ~(1u << CRO_BARRIER_LEG_CLUSTER)) {
        uint32_t covered = ~0u;
        for (unsigned leg = 0; leg < CRO_BARRIER_LEG_CLUSTER; ++leg)
            if (r->legs >> leg & 1u) covered = std::min<uint32_t>(covered, (uint32_t)t.seen[leg].size());
        r->sms_covered = covered;
        r->complete = r->sms_covered >= r->sm_count ? 1u : 0u;
    }
    for (const auto& p : pairs) {
        if (r->bad_pairs < CRO_BARRIER_MAX_PAIRS) r->bad_pair[r->bad_pairs] = cro_barrier_pair{(uint16_t)p.first, (uint16_t)p.second};
        r->bad_pairs++;
    }
    bool only_cluster = r->verdict == CRO_BARRIER_SM;
    for (const cro_barrier_sm& s : *sms)
        if (s.mark && s.failed_legs != 1u << CRO_BARRIER_LEG_CLUSTER) only_cluster = false;
    if (only_cluster) r->verdict = CRO_BARRIER_LINK;
    return status;
}
}  // namespace

void barrier_expected(unsigned leg, uint64_t seed, uint32_t cluster, cro_barrier_row* rows, uint64_t* words) {
    barrier::table(leg, seed, cluster, rows, words);
}

std::string barrier_opts_error(const cro_barrier_opts& o) {
    const uint32_t iters = o.iterations ? o.iterations : kBarrierDefaultIterations, cluster = cluster_of(o);
    const int leg = o.test_inject_leg;
    const bool inj_ok = !o.test_inject_mask ||
                        (leg >= 0 && leg < CRO_BARRIER_LEGS && (legs_of(o) >> leg & 1u) && o.test_inject_sm >= -1 &&
                         o.test_inject_sm < CRO_BARRIER_MAX_SMS && o.test_inject_warp >= -1 && o.test_inject_warp < CRO_BARRIER_WARPS &&
                         o.test_inject_lane >= -1 && o.test_inject_lane < 32 && o.test_inject_op < barrier::kOps[leg] &&
                         o.test_inject_iteration < iters);
    if (iters > CRO_BARRIER_MAX_ITERATIONS || o.legs > CRO_BARRIER_ALL_LEGS || o.max_rounds > CRO_BARRIER_MAX_ROUNDS || o.deadline_ms < 0 ||
        (cluster != 2 && cluster != 4 && cluster != 8) || !inj_ok)
        return "barrier probe: iterations at most " + std::to_string(CRO_BARRIER_MAX_ITERATIONS) + ", legs at most 0x7, max_rounds at most " +
               std::to_string(CRO_BARRIER_MAX_ROUNDS) + ", deadline_ms not negative, cluster 2, 4 or 8, and an injection must name a "
               "leg the call runs, an SM id below " + std::to_string(CRO_BARRIER_MAX_SMS) + ", a warp below 8 and a lane below 32 "
               "(each or -1), a row of the leg and an iteration the call runs";
    return "";
}

int ctx_probe_barrier(cro_ctx* c, int idx, const cro_barrier_opts& o, cro_barrier_result* r, std::vector<cro_barrier_sm>* sms,
                      std::vector<cro_barrier_fault>* faults) {
    const uint64_t t_call = now_ns();
    blank_result(r, cro_barrier_result{}, sms, faults);
    Device* d = dev_at(c, idx);
    if (!d)
        return r->status = unknown_device(c, idx, "a GPU attached after init is probed through the helper process, cro_probe_barrier_uuid");
    const uint32_t iters = o.iterations ? o.iterations : kBarrierDefaultIterations;
    const uint32_t max_rounds = o.max_rounds ? o.max_rounds : kBarrierDefaultRounds;
    const uint32_t legs = legs_of(o), cluster = cluster_of(o);
    const std::string why = barrier_opts_error(o);
    if (!why.empty()) {
        c->set_error(why);
        return r->status = CRO_ERR_INVALID_ARG;
    }
    DeviceGuard g = enter_device(c, idx);
    if (g.rc) return r->status = g.rc;
    Range nv(c, "cro.probe_barrier");
    LaneTally<BarrierReport> t;
    cudaEvent_t ev[2] = {nullptr, nullptr};                  // the call's own, destroyed on every way out
    int rc = [&]() -> int {
        const int sm_count = d->plan.sm_count;
        for (unsigned leg = 0; leg < CRO_BARRIER_LEGS; ++leg)
            if (legs >> leg & 1u) CU_TRY(c, barrier_plan(d->ordinal, leg));
        int net_grid = 0;
        if (legs >> CRO_BARRIER_LEG_CLUSTER & 1u) {
            CU_TRY(c, barrier_cluster_grid(cluster, &net_grid));
            if (net_grid < (int)cluster) {
                c->set_error("barrier probe: the device cannot place one cluster of " + std::to_string(cluster) + " CTAs");
                return CRO_ERR_UNSUPPORTED;
            }
        }
        const int max_grid = std::max(sm_count, net_grid);
        const uint64_t k = d->barrier_calls++;
        Tables tb;
        open_barrier_call(r, space_seed(d, kSeedBarrier, k), k, (uint32_t)sm_count, legs, iters, cluster, tb);

        // [CTA entries][thread entries] (armed together every round), then [records], then [rows][words] per leg
        const size_t n_thr = (size_t)max_grid * CRO_BARRIER_THREADS;
        const size_t cta_bytes = (size_t)max_grid * sizeof(cro_barrier_cta), thr_bytes = n_thr * sizeof(cro_barrier_thread);
        const size_t rec_off = (cta_bytes + thr_bytes + 255) & ~(size_t)255, rec_bytes = n_thr * kThreadRecs * sizeof(cro_barrier_fault);
        size_t row_off[CRO_BARRIER_LEGS], word_off[CRO_BARRIER_LEGS], end = (rec_off + rec_bytes + 255) & ~(size_t)255;
        for (unsigned leg = 0; leg < CRO_BARRIER_LEGS; ++leg) {
            row_off[leg] = end;
            end = (end + tb.rows[leg].size() * sizeof(cro_barrier_row) + 255) & ~(size_t)255;
            word_off[leg] = end;
            end += tb.words[leg].size() * sizeof(uint64_t);
        }
        DeviceMem<unsigned char> b;
        CU_TRY(c, cudaMalloc(&b.p, end));
        for (unsigned leg = 0; leg < CRO_BARRIER_LEGS; ++leg)
            if (!tb.rows[leg].empty()) {
                CU_TRY(c, cudaMemcpyAsync(b.p + row_off[leg], tb.rows[leg].data(), tb.rows[leg].size() * sizeof(cro_barrier_row),
                                          cudaMemcpyHostToDevice, d->stream));
                CU_TRY(c, cudaMemcpyAsync(b.p + word_off[leg], tb.words[leg].data(), tb.words[leg].size() * sizeof(uint64_t),
                                          cudaMemcpyHostToDevice, d->stream));
            }
        for (cudaEvent_t& x : ev) CU_TRY(c, cudaEventCreate(&x));
        cudaStream_t st = d->stream;
        BarrierArgs a{};
        a.cta = reinterpret_cast<cro_barrier_cta*>(b.p);
        a.thr = reinterpret_cast<cro_barrier_thread*>(b.p + cta_bytes);
        a.rec = reinterpret_cast<cro_barrier_fault*>(b.p + rec_off);
        a.stamp = k;
        a.iterations = iters;
        a.inj_sm = o.test_inject_sm;
        a.inj_warp = o.test_inject_warp;
        a.inj_lane = o.test_inject_lane;
        a.inj_op = o.test_inject_op;
        a.inj_iter = o.test_inject_iteration;
        std::vector<unsigned char> head(cta_bytes + thr_bytes);
        std::vector<cro_barrier_fault> hr(n_thr * kThreadRecs);
        for (unsigned leg = 0; leg < CRO_BARRIER_LEGS; ++leg) {
            if (!(legs >> leg & 1u)) continue;
            const int grid = leg == CRO_BARRIER_LEG_CLUSTER ? net_grid : sm_count;
            // The round's entries sit where the grid's CTA and thread entries end: CTA entries first, then threads.
            const size_t cb = (size_t)grid * sizeof(cro_barrier_cta), tbytes = (size_t)grid * CRO_BARRIER_THREADS * sizeof(cro_barrier_thread);
            a.thr = reinterpret_cast<cro_barrier_thread*>(b.p + cb);
            const auto* hc = reinterpret_cast<const cro_barrier_cta*>(head.data());
            const auto* ht = reinterpret_cast<const cro_barrier_thread*>(head.data() + cb);
            a.rows = reinterpret_cast<const cro_barrier_row*>(b.p + row_off[leg]);
            a.words = reinterpret_cast<const unsigned long long*>(b.p + word_off[leg]);
            a.inj_mask = o.test_inject_mask && o.test_inject_leg == (int)leg ? o.test_inject_mask : 0ull;
            auto launch = [&] { return launch_barrier(leg, a, grid, cluster, st); };
            auto fetch = [&] { return cudaMemcpyAsync(head.data(), b.p, cb + tbytes, cudaMemcpyDeviceToHost, st); };
            auto take = [&](uint32_t* covered) -> int {
                if (lane_any_failed<BarrierReport>(ht, grid, k))
                    CU_TRY(c, cudaMemcpy(hr.data(), a.rec, (size_t)grid * CRO_BARRIER_THREADS * kThreadRecs * sizeof(cro_barrier_fault),
                                         cudaMemcpyDeviceToHost));
                const uint32_t before = (uint32_t)t.seen[leg].size();
                const int e = take_lane_round<BarrierReport>(c, leg, hc, ht, hr.data(), grid, k, r, t, covered);
                // A CLUSTER round that reached no new SM ends the leg: the SMs left cannot host a whole cluster.
                if (leg == CRO_BARRIER_LEG_CLUSTER && t.seen[leg].size() == before) *covered = (uint32_t)sm_count;
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
        blank_result(r, *r, sms, faults);
        r->wall_ns = now_ns() - t_call;
        return r->status = rc;
    }
    const int status = close_barrier_call(r, t, sms, faults);
    r->wall_ns = now_ns() - t_call;
    return status;
}

int classify_barrier(uint32_t legs, uint32_t iterations, uint64_t seed, uint32_t cluster, uint32_t sm_count, uint64_t k, uint32_t rounds,
                     const cro_barrier_cta* ctas, const cro_barrier_thread* threads, const cro_barrier_fault* records,
                     cro_barrier_result* r, std::vector<cro_barrier_sm>* sms, std::vector<cro_barrier_fault>* faults) {
    blank_result(r, cro_barrier_result{}, sms, faults);
    Tables tb;
    open_barrier_call(r, seed, k, sm_count, legs, iterations, cluster, tb);
    r->table_ns = 0;
    LaneTally<BarrierReport> t;
    const size_t n_thr = (size_t)sm_count * CRO_BARRIER_THREADS;
    for (unsigned leg = 0; leg < CRO_BARRIER_LEGS; ++leg) {
        if (!(legs >> leg & 1u)) continue;
        for (uint32_t j = 0; j < rounds; ++j, ctas += sm_count, threads += n_thr, records += n_thr * kThreadRecs) {
            ++r->rounds;
            uint32_t covered = 0;
            const int e = take_lane_round<BarrierReport>(nullptr, leg, ctas, threads, records, (int)sm_count, k, r, t, &covered);
            if (e) {
                blank_result(r, *r, sms, faults);
                return r->status = e;
            }
        }
    }
    return close_barrier_call(r, t, sms, faults);
}

int ctx_probe_barrier_uuid(cro_ctx* c, const char* uuid, const cro_barrier_opts& o, cro_barrier_result* r,
                           std::vector<cro_barrier_sm>* sms, std::vector<cro_barrier_fault>* faults, int cap) {
    blank_result(r, cro_barrier_result{}, sms, faults);
    if (!uuid) return r->status = CRO_ERR_INVALID_ARG;
    const std::string why = barrier_opts_error(o);
    if (!why.empty()) {
        set_call_error(c, why);
        return r->status = CRO_ERR_INVALID_ARG;
    }
    uint64_t helper_ns = 0;
    if (run_check_helper(c, cro_wire_barrier, uuid, "barrier helper", "cro.probe_barrier.helper", &o, cap, o.deadline_ms, &helper_ns, r,
                         faults, sms) == CRO_OK)
        r->helper_ns = helper_ns;
    return r->status;
}

}  // namespace cro
