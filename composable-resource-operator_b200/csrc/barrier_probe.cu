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
constexpr uint32_t kBarrierDefaultCluster = 2;

uint32_t cluster_of(const cro_barrier_opts& o) { return o.cluster ? o.cluster : kBarrierDefaultCluster; }

// What the lane probes' host driver (lane_report.hpp) needs of the barrier probe: per leg a table of rows and words
// built on the host, and a CLUSTER leg that launches clusters of o.cluster CTAs.
struct BarrierProbe {
    using Opts = cro_barrier_opts;
    using Result = cro_barrier_result;
    using Sm = cro_barrier_sm;
    using Fault = cro_barrier_fault;
    using Thread = cro_barrier_thread;
    using Cta = cro_barrier_cta;
    using Args = BarrierArgs;
    struct Tables {
        std::vector<cro_barrier_row> rows[CRO_BARRIER_LEGS];
        std::vector<uint64_t> words[CRO_BARRIER_LEGS];
    };
    static constexpr unsigned kLegs = CRO_BARRIER_LEGS, kAllLegs = CRO_BARRIER_ALL_LEGS, kThreads = CRO_BARRIER_THREADS,
                              kThreadRecs = CRO_BARRIER_THREAD_RECORDS, kRecords = CRO_BARRIER_RECORDS, kMaxSms = CRO_BARRIER_MAX_SMS,
                              kMaxIterations = CRO_BARRIER_MAX_ITERATIONS, kMaxRounds = CRO_BARRIER_MAX_ROUNDS,
                              kPersistent = CRO_BARRIER_PERSISTENT, kIntermittent = CRO_BARRIER_INTERMITTENT, kNone = CRO_BARRIER_NONE,
                              kSm = CRO_BARRIER_SM, kAll = CRO_BARRIER_ALL;
    static constexpr const char* kName = "barrier";
    static constexpr const char* kId = "barrier";
    static constexpr const cro_wire& kWire = cro_wire_barrier;
    static constexpr uint64_t Device::*kCalls = &Device::barrier_calls;
    static constexpr SeedSpace kSeeds = kSeedBarrier;
    // Iterations per CTA and leg when the caller gives none, and launches per leg.  On an H100 80GB HBM3 at a 700 W
    // limit (profiles/h100_700w_barrier_rate.jsonl) one iteration of the three legs takes about 0.28 ms of launches
    // (BAR 244 us, MBAR 10 us, CLUSTER 27 us), so 16 iterations cost about the 5 ms the SRAM, register-file, cross-lane
    // and ALU probes take.
    static constexpr uint32_t kDefaultIterations = 16, kDefaultRounds = 4;
    static constexpr unsigned kBlobs = 2;       // rows, words

    static unsigned ops(unsigned leg) { return barrier::kOps[leg]; }
    static std::string opts_error(const cro_barrier_opts& o) { return barrier_opts_error(o); }
    static cudaError_t plan(int device, unsigned leg) { return barrier_plan(device, leg); }
    // BAR and MBAR: one CTA per SM; CLUSTER: as many clusters as the device holds at once.
    static int grids(cro_ctx* c, const cro_barrier_opts& o, uint32_t legs, int sm_count, int (&grid)[kLegs]) {
        std::fill(grid, grid + kLegs, sm_count);
        if (!(legs >> CRO_BARRIER_LEG_CLUSTER & 1u)) return CRO_OK;
        const uint32_t cluster = cluster_of(o);
        CU_TRY(c, barrier_cluster_grid(cluster, &grid[CRO_BARRIER_LEG_CLUSTER]));
        if (grid[CRO_BARRIER_LEG_CLUSTER] < (int)cluster) {
            c->set_error("barrier probe: the device cannot place one cluster of " + std::to_string(cluster) + " CTAs");
            return CRO_ERR_UNSUPPORTED;
        }
        return CRO_OK;
    }
    static cudaError_t launch(const cro_barrier_opts& o, unsigned leg, const BarrierArgs& a, int grid, cudaStream_t st) {
        return launch_barrier(leg, a, grid, cluster_of(o), st);
    }
    // The legs' tables and the closed form of every CTA's fold.
    static void open(const cro_barrier_opts& o, cro_barrier_result* r, Tables& tb, bool timed) {
        const uint64_t t0 = now_ns();
        r->cluster = cluster_of(o);
        for (unsigned leg = 0; leg < CRO_BARRIER_LEGS; ++leg) {
            if (!(r->legs >> leg & 1u)) continue;
            const unsigned n = barrier::kOps[leg];
            tb.rows[leg].resize(n);
            tb.words[leg].resize((size_t)n * CRO_BARRIER_THREADS * 2);
            barrier::table(leg, r->seed, r->cluster, tb.rows[leg].data(), tb.words[leg].data());
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
        if (timed) r->table_ns = now_ns() - t0;
    }
    static std::array<LaneBlob, kBlobs> blobs(const Tables& tb, unsigned leg) {
        return {LaneBlob{tb.rows[leg].data(), tb.rows[leg].size() * sizeof(cro_barrier_row)},
                LaneBlob{tb.words[leg].data(), tb.words[leg].size() * sizeof(uint64_t)}};
    }
    static void args(const cro_barrier_opts&, const cro_barrier_result&, unsigned, const std::array<const void*, kBlobs>& on_dev,
                     BarrierArgs* a) {
        a->rows = static_cast<const cro_barrier_row*>(on_dev[0]);
        a->words = static_cast<const unsigned long long*>(on_dev[1]);
    }
    // A CLUSTER round that reached no new SM ends the leg: the SMs left cannot host a whole cluster.
    static bool no_new_sm_ends(unsigned leg) { return leg == CRO_BARRIER_LEG_CLUSTER; }
    static int close(cro_barrier_result* r, LaneTally<BarrierProbe>& t, std::vector<cro_barrier_sm>* sms,
                     std::vector<cro_barrier_fault>* faults);
    static void keep(cro_barrier_result* r, const cro_barrier_result& from) {
        r->cluster = from.cluster;
        r->table_ns = from.table_ns;
    }
};

// The report path's verdict, then the barrier probe's own: the kept timeout records, the coverage, the (SM, peer SM)
// pairs of every kept CLUSTER record (taken before the records are sorted and capped, so BAR and MBAR records cannot
// crowd them out), and LINK when only CLUSTER checks failed on a strict subset of the SMs.  A cluster cannot use an SM
// whose GPC has no room for the whole cluster, so the call's coverage is the CTA-local legs' when one ran, and the
// CLUSTER leg's own is cluster_sms.
int BarrierProbe::close(cro_barrier_result* r, LaneTally<BarrierProbe>& t, std::vector<cro_barrier_sm>* sms,
                        std::vector<cro_barrier_fault>* faults) {
    std::set<std::pair<uint32_t, uint32_t>> pairs;
    for (const cro_barrier_fault& f : t.recs) {
        r->timeouts += f.kind == CRO_BARRIER_KIND_TIMEOUT ? 1 : 0;
        if (f.leg == CRO_BARRIER_LEG_CLUSTER) pairs.insert({f.smid, f.peer_smid});
    }
    r->cluster_sms = (uint32_t)t.seen[CRO_BARRIER_LEG_CLUSTER].size();
    const int status = close_lane_call<BarrierProbe>(r, t, sms, faults);
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
    const uint32_t cluster = cluster_of(o);
    if (!lane_opts_ok<BarrierProbe>(o) || (cluster != 2 && cluster != 4 && cluster != 8))
        return "barrier probe: iterations at most " + std::to_string(CRO_BARRIER_MAX_ITERATIONS) + ", legs at most 0x7, max_rounds at most " +
               std::to_string(CRO_BARRIER_MAX_ROUNDS) + ", deadline_ms not negative, cluster 2, 4 or 8, and an injection must name a "
               "leg the call runs, an SM id below " + std::to_string(CRO_BARRIER_MAX_SMS) + ", a warp below 8 and a lane below 32 "
               "(each or -1), a row of the leg and an iteration the call runs";
    return "";
}

int ctx_probe_barrier(cro_ctx* c, int idx, const cro_barrier_opts& o, cro_barrier_result* r, std::vector<cro_barrier_sm>* sms,
                      std::vector<cro_barrier_fault>* faults) {
    return probe_lane_legs<BarrierProbe>(c, idx, o, r, sms, faults);
}

int classify_barrier(uint32_t legs, uint32_t iterations, uint64_t seed, uint32_t cluster, uint32_t sm_count, uint64_t k, uint32_t rounds,
                     const cro_barrier_cta* ctas, const cro_barrier_thread* threads, const cro_barrier_fault* records,
                     cro_barrier_result* r, std::vector<cro_barrier_sm>* sms, std::vector<cro_barrier_fault>* faults) {
    cro_barrier_opts o{};
    o.legs = legs;
    o.iterations = iterations;
    o.cluster = cluster;
    return classify_lane_legs<BarrierProbe>(o, seed, sm_count, k, rounds, ctas, threads, records, r, sms, faults);
}

int ctx_probe_barrier_uuid(cro_ctx* c, const char* uuid, const cro_barrier_opts& o, cro_barrier_result* r,
                           std::vector<cro_barrier_sm>* sms, std::vector<cro_barrier_fault>* faults, int cap) {
    return probe_lane_legs_uuid<BarrierProbe>(c, uuid, o, r, sms, faults, cap);
}

}  // namespace cro
