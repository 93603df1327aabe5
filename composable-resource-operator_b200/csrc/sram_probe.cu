// sram_probe.cu — the SRAM probe (cro_probe_sram, cro_probe_sram_uuid): every SM's shared memory marched as 0 and as
// 1, the SM-to-SM network of a cluster written and read across, and the SRAM ECC record NVML keeps for them.
#include <map>
#include <set>
#include <tuple>

#include "probe_internal.hpp"

namespace cro {

namespace {
// Iterations per CTA and launches per leg when the caller gives none.  On an H100 80GB HBM3 at a 400 W limit
// (profiles/h100_400w_sram_rate.jsonl) a local launch of 64 iterations takes 2.9 ms and a network launch at C = 2
// 1.8 ms, and one round of each covers all 132 SMs: about 5 ms a call for every cell written and read back 64 times
// each way.  The time grows linearly with iterations (DESIGN.md "The SRAM probe").
constexpr uint32_t kSramDefaultIterations = 64;
constexpr uint32_t kSramDefaultRounds = 4;
constexpr uint32_t kSramDefaultCluster = 2;

// The result of a call that marched nothing: zeroes but for what the call had settled before it stopped.
void blank_result(cro_sram_result* r, const cro_sram_result& from, std::vector<cro_sram_sm>* sms, std::vector<cro_sram_fault>* faults) {
    const cro_sram_result keep = from;
    memset(r, 0, sizeof *r);
    r->seed = keep.seed;
    r->call = keep.call;
    r->sm_count = keep.sm_count;
    r->legs = keep.legs;
    r->bytes_per_sm = keep.bytes_per_sm;
    r->cuda_error = keep.cuda_error;
    r->before = keep.before;
    r->after = keep.after;
    r->health = keep.health;
    sms->clear();
    faults->clear();
}

// What every CTA's M5 fold must be: the read-sweep checksum of pattern_word(seed, 0 .. n) once per iteration (xor of
// the iterations' folds, sums summed).
void closed_form(uint64_t seed, uint32_t n, uint32_t iterations, cro_sram_leg* L) {
    uint64_t x = 0, s = 0, w = 0;
    for (uint64_t i = 0; i < n; ++i) {
        const uint64_t v = pattern_word(seed, i);
        x ^= v;
        s += v;
        w += v * (2 * i + 1);
    }
    L->expect_xor = (iterations & 1) ? x : 0;
    L->expect_sum = s * iterations;
    L->expect_wsum = w * iterations;
}

bool valid_injection(const cro_sram_opts& o, uint32_t iterations) {
    if (!o.test_inject_mask) return true;
    const bool el = o.test_inject_leg == CRO_SRAM_SMEM ? (o.test_inject_element >= 1 && o.test_inject_element <= 5)
                    : o.test_inject_leg == CRO_SRAM_DSMEM ? (o.test_inject_element == 1 || o.test_inject_element == 2)
                                                          : false;
    return el && o.test_inject_sm >= -1 && o.test_inject_sm < CRO_SRAM_MAX_SMS && o.test_inject_iteration < iterations &&
           o.test_inject_word >= -1;
}

// cro_sram_cta and cro_sram_record are the public mirrors of SramCta and SramRecord (cro_selftest_sram_classify).
#define CRO_SAME_AT(a, b, f) (offsetof(a, f) == offsetof(b, f))
static_assert(sizeof(cro_sram_cta) == sizeof(SramCta) && CRO_SAME_AT(cro_sram_cta, SramCta, stamp) &&
                  CRO_SAME_AT(cro_sram_cta, SramCta, t0) && CRO_SAME_AT(cro_sram_cta, SramCta, t1) &&
                  CRO_SAME_AT(cro_sram_cta, SramCta, cycles) && CRO_SAME_AT(cro_sram_cta, SramCta, count) &&
                  CRO_SAME_AT(cro_sram_cta, SramCta, last) && CRO_SAME_AT(cro_sram_cta, SramCta, fold_x) &&
                  CRO_SAME_AT(cro_sram_cta, SramCta, fold_s) && CRO_SAME_AT(cro_sram_cta, SramCta, fold_w) &&
                  CRO_SAME_AT(cro_sram_cta, SramCta, smid) && CRO_SAME_AT(cro_sram_cta, SramCta, nsmid) &&
                  CRO_SAME_AT(cro_sram_cta, SramCta, rank) && CRO_SAME_AT(cro_sram_cta, SramCta, block),
              "cro_sram_cta mirrors SramCta");
static_assert(sizeof(cro_sram_record) == sizeof(SramRecord) && CRO_SAME_AT(cro_sram_record, SramRecord, element) &&
                  CRO_SAME_AT(cro_sram_record, SramRecord, iteration) && CRO_SAME_AT(cro_sram_record, SramRecord, smid) &&
                  CRO_SAME_AT(cro_sram_record, SramRecord, peer_block) && CRO_SAME_AT(cro_sram_record, SramRecord, round) &&
                  CRO_SAME_AT(cro_sram_record, SramRecord, word) && CRO_SAME_AT(cro_sram_record, SramRecord, expected) &&
                  CRO_SAME_AT(cro_sram_record, SramRecord, actual),
              "cro_sram_record mirrors SramRecord");
#undef CRO_SAME_AT

// What a call's legs leave for its verdict.
struct SramTally {
    std::map<uint32_t, cro_sram_sm> per_sm;
    std::map<uint32_t, uint64_t> last[CRO_SRAM_LEGS];       // per SM: failed compares of the last iteration
    std::vector<SramRecord> recs[CRO_SRAM_LEGS];
    std::vector<std::vector<uint32_t>> block_smid;          // network leg, per round: blockIdx.x -> %smid (~0u: silent)
};
// What one leg keeps across its rounds.
struct SramLegRounds {
    std::set<uint32_t> seen;                                // distinct SMs
    uint32_t fold_sm = ~0u;                                 // the lowest of them, whose fold R reports
};

// A leg before its first round: its iterations, cluster and (local) the closed form of the fold.  Returns the bytes
// each of its CTAs reads and writes: local M0 and M5 touch every word once, M1 .. M4 twice; network D0, D2, D3 once
// and D1 once per peer.
uint64_t open_sram_leg(cro_sram_leg& R, bool net, uint64_t seed, uint32_t n_words, uint32_t iters, uint32_t cluster) {
    R.iterations = iters;
    R.cluster = net ? cluster : 0u;
    if (!net) closed_form(seed, n_words, iters, &R);
    return 8ull * n_words * iters * (net ? cluster + 2 : 10);
}

// One round of leg `leg` of call k: the grid CTA records hc (each CTA moved cta_bytes_moved bytes) into r->leg[leg],
// t's per-SM and last-iteration counts and, on the network leg, the round's block map; *covered: the distinct SMs the
// leg has seen so far.  CRO_ERR_UNSUPPORTED (with the error text) when the device reports more SM ids than the result
// holds.
int take_sram_round(cro_ctx* c, const SramCta* hc, int grid, uint64_t k, uint32_t leg, uint64_t cta_bytes_moved,
                    cro_sram_result* r, SramTally& t, SramLegRounds& lr, uint32_t* covered) {
    cro_sram_leg& R = r->leg[leg];
    const bool net = leg == CRO_SRAM_DSMEM;
    R.ctas += (uint32_t)grid;
    R.bytes += cta_bytes_moved * (uint64_t)grid;
    if (net) t.block_smid.emplace_back((size_t)grid, ~0u);
    uint64_t t0 = ~0ull, t1 = 0;
    for (int j = 0; j < grid; ++j) {
        const SramCta& x = hc[(size_t)j];
        if (x.stamp != k) {
            R.unpublished++;
            continue;
        }
        if (x.nsmid > CRO_SRAM_MAX_SMS) {
            set_call_error(c, "SRAM probe: the device reports %nsmid = " + std::to_string(x.nsmid) + ", more SM ids than the " +
                                  std::to_string(CRO_SRAM_MAX_SMS) + " the result holds");
            return CRO_ERR_UNSUPPORTED;
        }
        r->nsmid = x.nsmid;
        t0 = std::min<uint64_t>(t0, x.t0);
        t1 = std::max<uint64_t>(t1, x.t1);
        if (net) t.block_smid.back()[(size_t)j] = x.smid;
        lr.seen.insert(x.smid);
        cro_sram_sm& S = t.per_sm[x.smid];
        S.smid = x.smid;
        cro_sram_sm_leg& SL = S.leg[leg];
        SL.ctas++;
        for (int e = 0; e < CRO_SRAM_ELEMENTS; ++e) {
            SL.mismatches[e] += x.count[e];
            R.mismatches[e] += x.count[e];
        }
        t.last[leg][x.smid] += x.last;
        SL.ns += x.t1 > x.t0 ? x.t1 - x.t0 : 0;
        SL.cycles += x.cycles;
        if (net) continue;
        const bool fold_bad = x.fold_x != R.expect_xor || x.fold_s != R.expect_sum || x.fold_w != R.expect_wsum;
        SL.fold_mismatches += fold_bad ? 1 : 0;
        R.fold_mismatches += fold_bad ? 1 : 0;
        if (x.smid < lr.fold_sm) {
            lr.fold_sm = x.smid;
            R.fold_xor = x.fold_x;
            R.fold_sum = x.fold_s;
            R.fold_wsum = x.fold_w;
        }
    }
    if (t1 > t0) R.timer_ns += t1 - t0;
    *covered = R.sms_covered = (uint32_t)lr.seen.size();
    return CRO_OK;
}

// A leg after its last round: its coverage of sm_count SMs, the records kept of n_claims and each SM's mark
// (persistent: a compare of the last iteration failed; intermittent: only an earlier one, or only the fold).
void close_sram_leg(cro_sram_result* r, uint32_t leg, uint32_t sm_count, uint64_t n_claims, SramTally& t) {
    cro_sram_leg& R = r->leg[leg];
    R.complete = R.sms_covered >= sm_count ? 1u : 0u;
    R.recorded = std::min<uint64_t>(n_claims, CRO_SRAM_RECORDS);
    for (auto& kv : t.per_sm) {
        cro_sram_sm_leg& SL = kv.second.leg[leg];
        if (!SL.ctas) continue;
        uint64_t any = SL.fold_mismatches;
        for (uint64_t m : SL.mismatches) any += m;
        SL.mark = t.last[leg][kv.first] ? CRO_SRAM_PERSISTENT : any ? CRO_SRAM_INTERMITTENT : 0u;
        if (SL.mark) R.failed_sms++;
    }
}

// The call's end: the word records with the owner or writer resolved from the CTAs' own records of the same round,
// the SMs that failed the local leg, the network pairs between SMs that passed it, and the verdict.
int close_sram_call(cro_sram_result* r, const SramTally& t, std::vector<cro_sram_sm>* sms, std::vector<cro_sram_fault>* faults) {
    for (uint32_t leg = 0; leg < CRO_SRAM_LEGS; ++leg)
        for (const SramRecord& q : t.recs[leg]) {
            cro_sram_fault f{};
            f.leg = leg;
            f.element = q.element;
            f.iteration = q.iteration;
            f.smid = q.smid;
            f.word = q.word;
            f.expected = q.expected;
            f.actual = q.actual;
            if (leg == CRO_SRAM_SMEM) {
                f.peer_smid = q.smid;
                f.direction = CRO_SRAM_DIR_LOCAL;
            } else {
                f.direction = q.element == 1 ? CRO_SRAM_DIR_READ : CRO_SRAM_DIR_WRITE;
                f.peer_smid = q.round < t.block_smid.size() && q.peer_block < t.block_smid[q.round].size()
                                  ? t.block_smid[q.round][q.peer_block]
                                  : ~0u;
            }
            faults->push_back(f);
        }
    std::sort(faults->begin(), faults->end(), [](const cro_sram_fault& x, const cro_sram_fault& y) {
        return std::make_tuple(x.leg, x.element, x.smid, x.iteration, x.word) < std::make_tuple(y.leg, y.element, y.smid, y.iteration, y.word);
    });

    // verdict: SMs that failed the local leg, then network pairs between SMs that passed it
    std::set<uint32_t> local_bad;
    for (auto& kv : t.per_sm) {
        if (kv.second.leg[CRO_SRAM_SMEM].mark) local_bad.insert(kv.first);
        sms->push_back(kv.second);
    }
    std::set<std::tuple<uint32_t, uint32_t, uint32_t>> pairs;      // (direction, from, owner)
    for (const cro_sram_fault& f : *faults) {
        if (f.leg != CRO_SRAM_DSMEM || local_bad.count(f.smid) || local_bad.count(f.peer_smid)) continue;
        if (f.direction == CRO_SRAM_DIR_READ) pairs.insert({f.direction, f.smid, f.peer_smid});
        else pairs.insert({f.direction, f.peer_smid, f.smid});
    }
    bool all = false, any = false;
    for (uint32_t leg = 0; leg < CRO_SRAM_LEGS; ++leg) {
        const cro_sram_leg& R = r->leg[leg];
        if (!(r->legs >> leg & 1u)) continue;
        if (R.unpublished || (R.failed_sms && R.failed_sms == R.sms_covered)) all = true;
        if (R.unpublished || R.failed_sms) any = true;
    }
    for (uint32_t s : local_bad) {
        if (r->bad_sms < 16) r->bad_sm[r->bad_sms] = (uint16_t)s;
        r->bad_sms++;
    }
    for (const auto& p : pairs) {
        if (r->bad_pairs < CRO_SRAM_MAX_PAIRS)
            r->bad_pair[r->bad_pairs] = cro_sram_pair{(uint16_t)std::get<1>(p), (uint16_t)std::get<2>(p), std::get<0>(p)};
        r->bad_pairs++;
    }
    r->verdict = all ? CRO_SRAM_ALL : !local_bad.empty() ? CRO_SRAM_SM : any ? CRO_SRAM_LINK : CRO_SRAM_NONE;
    return r->status = any ? CRO_ERR_CHECKSUM : CRO_OK;
}
}  // namespace

uint32_t sram_health(const cro_sram_health& b, const cro_sram_health& a) {
    uint32_t h = 0;
    if ((b.nvml & a.nvml & CRO_SRAM_NVML_ECC_CORRECTED) && a.ecc_corrected > b.ecc_corrected) h |= CRO_SRAM_HEALTH_CORRECTED_DURING;
    if ((b.nvml & a.nvml & CRO_SRAM_NVML_ECC_UNCORRECTED) && a.ecc_uncorrected > b.ecc_uncorrected) h |= CRO_SRAM_HEALTH_UNCORRECTED_DURING;
    if ((a.nvml & CRO_SRAM_NVML_STATUS) && a.threshold_exceeded) h |= CRO_SRAM_HEALTH_THRESHOLD_EXCEEDED;
    return h;
}

int ctx_probe_sram(cro_ctx* c, int idx, const cro_sram_opts& o, cro_sram_result* r, std::vector<cro_sram_sm>* sms,
                   std::vector<cro_sram_fault>* faults) {
    const uint64_t t_call = now_ns();
    blank_result(r, cro_sram_result{}, sms, faults);
    Device* d = dev_at(c, idx);
    if (!d) return r->status = unknown_device(c, idx, "a GPU attached after init is probed through the helper process, cro_probe_sram_uuid");
    const uint32_t legs = o.legs ? o.legs : CRO_SRAM_ALL_LEGS;
    const uint32_t iters = o.iterations ? o.iterations : kSramDefaultIterations;
    const uint32_t cluster = o.cluster ? o.cluster : kSramDefaultCluster;
    const uint32_t max_rounds = o.max_rounds ? o.max_rounds : kSramDefaultRounds;
    if ((legs & ~CRO_SRAM_ALL_LEGS) || iters > CRO_SRAM_MAX_ITERATIONS || (cluster != 2 && cluster != 4 && cluster != 8) ||
        max_rounds > CRO_SRAM_MAX_ROUNDS || !valid_injection(o, iters)) {
        c->set_error("SRAM probe: legs must be CRO_SRAM_ALL_LEGS bits, iterations at most " + std::to_string(CRO_SRAM_MAX_ITERATIONS) +
                     ", cluster 2, 4 or 8, max_rounds at most " + std::to_string(CRO_SRAM_MAX_ROUNDS) +
                     ", and an injection must name a leg, an element it has (local 1 .. 5, network 1 or 2), an SM id below " +
                     std::to_string(CRO_SRAM_MAX_SMS) + " (or -1), an iteration the call runs and a word (or -1)");
        return r->status = CRO_ERR_INVALID_ARG;
    }
    DeviceGuard g = enter_device(c, idx);
    if (g.rc) return r->status = g.rc;
    Range nv(c, "cro.probe_sram");
    const std::string uuid(d->info.gpu_uuid, strnlen(d->info.gpu_uuid, sizeof d->info.gpu_uuid));
    const bool nvml = !(c->opts.flags & CRO_F_NO_NVML);
    SramTally t;
    bool marched = false;
    cudaEvent_t ev[2] = {nullptr, nullptr};                  // the call's own, destroyed on every way out
    int rc = [&]() -> int {
        const int sm_count = d->plan.sm_count;
        unsigned n_words = 0;
        CU_TRY(c, sram_plan(d->ordinal, &n_words));
        if (o.test_inject_mask && o.test_inject_word >= (int)n_words) {
            c->set_error("SRAM probe: injection word " + std::to_string(o.test_inject_word) + " is past the " +
                         std::to_string(n_words) + " words each CTA marches");
            return CRO_ERR_INVALID_ARG;
        }
        int clusters = 0;
        if (legs & CRO_SRAM_LEG_DSMEM) {
            CU_TRY(c, sram_max_clusters(cluster, n_words, &clusters));
            if (clusters < 1) {
                c->set_error("SRAM probe: the device cannot place one cluster of " + std::to_string(cluster) + " CTAs with " +
                             std::to_string(8ull * n_words) + " bytes of shared memory each");
                return CRO_ERR_UNSUPPORTED;
            }
        }
        const int net_grid = clusters * (int)cluster, max_grid = std::max(sm_count, net_grid);
        const uint64_t k = d->sram_calls++;
        const uint64_t seed = space_seed(d, kSeedSram, k);     // rank r's: seed + r * kNonceStride
        r->seed = seed;
        r->call = k;
        r->sm_count = (uint32_t)sm_count;
        r->legs = legs;
        r->bytes_per_sm = 8ull * n_words;

        // [claims per leg][records per leg][CTA records], allocated per call
        const size_t rec_off = 64, rec_bytes = (size_t)CRO_SRAM_LEGS * CRO_SRAM_RECORDS * sizeof(SramRecord);
        const size_t cta_off = (rec_off + rec_bytes + 63) & ~(size_t)63;
        DeviceMem<unsigned char> b;
        CU_TRY(c, cudaMalloc(&b.p, cta_off + (size_t)max_grid * sizeof(SramCta)));
        for (cudaEvent_t& x : ev) CU_TRY(c, cudaEventCreate(&x));
        cudaStream_t st = d->stream;
        CU_TRY(c, cudaMemsetAsync(b.p, 0, rec_off, st));
        unsigned long long* claims = reinterpret_cast<unsigned long long*>(b.p);
        SramRecord* rec = reinterpret_cast<SramRecord*>(b.p + rec_off);
        SramCta* cta = reinterpret_cast<SramCta*>(b.p + cta_off);
        std::vector<SramCta> hc((size_t)max_grid);
        if (nvml) identity::NvmlSramHealth(uuid, false, &r->before);
        marched = true;

        for (uint32_t leg = 0; leg < CRO_SRAM_LEGS; ++leg) {
            if (!(legs >> leg & 1u)) continue;
            cro_sram_leg& R = r->leg[leg];
            const bool net = leg == CRO_SRAM_DSMEM;
            const int grid = net ? net_grid : sm_count;
            SramArgs a{};
            a.cta = cta;
            a.rec = rec + (size_t)leg * CRO_SRAM_RECORDS;
            a.claims = claims + leg;
            a.seed = seed;
            a.stamp = k;
            a.n_words = n_words;
            a.iterations = iters;
            a.inj_sm = o.test_inject_sm;
            a.inj_word = o.test_inject_word;
            a.inj_element = o.test_inject_element;
            a.inj_iter = o.test_inject_iteration;
            a.inj_mask = o.test_inject_leg == (int)leg ? o.test_inject_mask : 0ull;
            const uint64_t cta_bytes_moved = open_sram_leg(R, net, seed, n_words, iters, cluster);
            const size_t cta_bytes = (size_t)grid * sizeof(SramCta);
            SramLegRounds lr;
            auto launch = [&] {
                a.round = R.rounds;
                return net ? launch_sram_dsmem(a, grid, cluster, st) : launch_sram_smem(a, grid, st);
            };
            auto fetch = [&] { return cudaMemcpyAsync(hc.data(), cta, cta_bytes, cudaMemcpyDeviceToHost, st); };
            auto take = [&](uint32_t* covered) -> int {
                return take_sram_round(c, hc.data(), grid, k, leg, cta_bytes_moved, r, t, lr, covered);
            };
            const int e = coverage_rounds(c, d, ev, cta, cta_bytes, (uint32_t)sm_count, max_rounds, &R.rounds, &R.ns, launch, fetch, take);
            if (e) return e;
            unsigned long long n_claims = 0;
            CU_TRY(c, cudaMemcpy(&n_claims, a.claims, sizeof n_claims, cudaMemcpyDeviceToHost));
            close_sram_leg(r, leg, (uint32_t)sm_count, n_claims, t);
            t.recs[leg].resize((size_t)R.recorded);
            if (R.recorded) CU_TRY(c, cudaMemcpy(t.recs[leg].data(), a.rec, t.recs[leg].size() * sizeof(SramRecord), cudaMemcpyDeviceToHost));
        }
        return CRO_OK;
    }();
    for (cudaEvent_t x : ev)
        if (x) cudaEventDestroy(x);
    if (rc == CRO_ERR_CUDA) r->cuda_error = (int32_t)cudaGetLastError();
    if (marched && nvml) identity::NvmlSramHealth(uuid, true, &r->after);
    r->health = sram_health(r->before, r->after);
    if (rc) {
        blank_result(r, *r, sms, faults);
        r->wall_ns = now_ns() - t_call;
        return r->status = rc;
    }

    const int status = close_sram_call(r, t, sms, faults);
    r->wall_ns = now_ns() - t_call;
    return status;
}

int classify_sram(uint32_t legs, uint32_t iterations, uint32_t n_words, uint64_t seed, uint32_t cluster, uint32_t sm_count,
                  uint32_t net_grid, uint64_t k, const uint32_t* rounds, const cro_sram_cta* ctas, const uint64_t* claims,
                  const cro_sram_record* records, cro_sram_result* r, std::vector<cro_sram_sm>* sms,
                  std::vector<cro_sram_fault>* faults) {
    blank_result(r, cro_sram_result{}, sms, faults);
    r->seed = seed;
    r->call = k;
    r->sm_count = sm_count;
    r->legs = legs;
    r->bytes_per_sm = 8ull * n_words;
    SramTally t;
    const int rc = [&]() -> int {
        for (uint32_t leg = 0; leg < CRO_SRAM_LEGS; ++leg) {
            if (!(legs >> leg & 1u)) continue;
            cro_sram_leg& R = r->leg[leg];
            const bool net = leg == CRO_SRAM_DSMEM;
            const int grid = (int)(net ? net_grid : sm_count);
            const uint64_t cta_bytes_moved = open_sram_leg(R, net, seed, n_words, iterations, cluster);
            std::vector<SramCta> hc((size_t)grid);
            SramLegRounds lr;
            for (uint32_t j = 0; j < rounds[leg]; ++j, ctas += grid) {
                memcpy(hc.data(), ctas, hc.size() * sizeof(SramCta));
                ++R.rounds;
                uint32_t covered = 0;
                const int e = take_sram_round(nullptr, hc.data(), grid, k, leg, cta_bytes_moved, r, t, lr, &covered);
                if (e) return e;
            }
            close_sram_leg(r, leg, sm_count, claims[leg], t);
            t.recs[leg].resize((size_t)R.recorded);
            if (R.recorded) memcpy(t.recs[leg].data(), records, t.recs[leg].size() * sizeof(SramRecord));
            records += R.recorded;
        }
        return CRO_OK;
    }();
    if (rc) {
        blank_result(r, *r, sms, faults);
        return r->status = rc;
    }
    return close_sram_call(r, t, sms, faults);
}

namespace {
uint64_t sram_tail_count(const unsigned char* head) {
    return reinterpret_cast<const cro_sram_result*>(head)->recorded;
}
}  // namespace

int ctx_probe_sram_uuid(cro_ctx* c, const char* uuid, const cro_sram_opts& o, cro_sram_result* r, std::vector<cro_sram_sm>* sms,
                        std::vector<cro_sram_fault>* faults, int cap) {
    blank_result(r, cro_sram_result{}, sms, faults);
    if (!uuid) return r->status = CRO_ERR_INVALID_ARG;
    const std::string want = uuid;
    auto num = [](int64_t v) { return std::to_string(v); };
    const std::vector<std::string> args = {"sram-raw", want, num(o.legs), num(o.iterations), num(o.cluster), num(o.max_rounds),
                                           num(o.test_inject_leg), num(o.test_inject_sm), num(o.test_inject_element),
                                           num(o.test_inject_iteration), num(o.test_inject_word), std::to_string(o.test_inject_mask),
                                           num(cap)};
    const size_t head = sizeof *r + CRO_SRAM_MAX_SMS * sizeof(cro_sram_sm);
    std::string got;
    uint64_t helper_ns = 0;
    const int rc = run_probe_helper(c, want, "SRAM helper", "cro.probe_sram.helper", args, o.deadline_ms, head,
                                    sizeof(cro_sram_fault), (size_t)cap, sram_tail_count, &got, &helper_ns);
    if (rc != CRO_OK) return r->status = rc;
    memcpy(r, got.data(), sizeof *r);
    const cro_sram_sm* s = reinterpret_cast<const cro_sram_sm*>(got.data() + sizeof *r);
    sms->assign(s, s + std::min<uint32_t>(r->sms_listed, CRO_SRAM_MAX_SMS));
    const cro_sram_fault* f = reinterpret_cast<const cro_sram_fault*>(got.data() + head);
    faults->assign(f, f + r->recorded);
    r->helper_ns = helper_ns;
    return r->status;
}

}  // namespace cro
