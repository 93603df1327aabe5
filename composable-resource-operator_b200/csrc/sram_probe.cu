// sram_probe.cu — the SRAM probe (cro_probe_sram, cro_probe_sram_uuid): every SM's shared memory marched as 0 and as
// 1, the SM-to-SM network of a cluster written and read across, and the SRAM ECC record NVML keeps for them.
#include <set>
#include <tuple>

#include "cell_report.hpp"

namespace cro {

namespace {
// Iterations per CTA and launches per leg when the caller gives none.  On an H100 80GB HBM3 at a 400 W limit
// (profiles/h100_400w_sram_rate.jsonl) a local launch of 64 iterations takes 2.9 ms and a network launch at C = 2
// 1.8 ms, and one round of each covers all 132 SMs: about 5 ms a call for every cell written and read back 64 times
// each way.  The time grows linearly with iterations (DESIGN.md "The SRAM probe").
constexpr uint32_t kSramDefaultIterations = 64;
constexpr uint32_t kSramDefaultRounds = 4;
constexpr uint32_t kSramDefaultCluster = 2;

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

// What the memory-cell probes' host driver (cell_report.hpp) needs of the SRAM probe.  The host reads the device's
// SramCta and SramRecord through their public mirrors.
struct SramProbe {
    using Opts = cro_sram_opts;
    using Result = cro_sram_result;
    using Sm = cro_sram_sm;
    using Fault = cro_sram_fault;
    using Cta = cro_sram_cta;
    using Record = cro_sram_record;
    using Args = SramArgs;
    struct Call {
        uint32_t legs, iterations, n_words, cluster;
        int net_grid;                                       // network leg: CTAs per launch
        std::vector<std::vector<uint32_t>> block_smid;      // network leg, per round: blockIdx.x -> %smid (~0u: silent)
    };
    static constexpr unsigned kLegs = CRO_SRAM_LEGS, kElements = CRO_SRAM_ELEMENTS, kRecords = CRO_SRAM_RECORDS,
                              kMaxSms = CRO_SRAM_MAX_SMS, kPersistent = CRO_SRAM_PERSISTENT, kIntermittent = CRO_SRAM_INTERMITTENT,
                              kDefaultRounds = kSramDefaultRounds;
    static constexpr const char* kName = "SRAM";
    static constexpr const char* kId = "sram";
    static constexpr const cro_wire& kWire = cro_wire_sram;
    static constexpr auto kCalls = &Device::sram_calls;
    static constexpr SeedSpace kSeeds = kSeedSram;

    static cro_sram_leg& leg(cro_sram_result& r, unsigned l) { return r.leg[l]; }
    static cro_sram_sm_leg& leg(cro_sram_sm& s, unsigned l) { return s.leg[l]; }
    static std::string opts_error(const cro_sram_opts& o) { return sram_opts_error(o); }
    // The helper refuses the options itself.
    static std::string helper_opts_error(const cro_sram_opts&) { return ""; }

    // The words each CTA marches, an injection word among them, and for the network leg as many clusters as the device
    // places at once.
    static int plan(cro_ctx* c, Device* d, const cro_sram_opts& o, cro_sram_result*, Call* call) {
        call->legs = o.legs ? o.legs : CRO_SRAM_ALL_LEGS;
        call->iterations = o.iterations ? o.iterations : kSramDefaultIterations;
        const uint32_t cluster = call->cluster = o.cluster ? o.cluster : kSramDefaultCluster;
        unsigned n_words = 0;
        CU_TRY(c, sram_plan(d->ordinal, &n_words));
        call->n_words = n_words;
        if (o.test_inject_mask && o.test_inject_word >= (int)n_words) {
            c->set_error("SRAM probe: injection word " + std::to_string(o.test_inject_word) + " is past the " +
                         std::to_string(n_words) + " words each CTA marches");
            return CRO_ERR_INVALID_ARG;
        }
        int clusters = 0;
        if (call->legs & CRO_SRAM_LEG_DSMEM) {
            CU_TRY(c, sram_max_clusters(cluster, n_words, &clusters));
            if (clusters < 1) {
                c->set_error("SRAM probe: the device cannot place one cluster of " + std::to_string(cluster) + " CTAs with " +
                             std::to_string(8ull * n_words) + " bytes of shared memory each");
                return CRO_ERR_UNSUPPORTED;
            }
        }
        call->net_grid = clusters * (int)cluster;
        return CRO_OK;
    }
    static void open(const Call& call, cro_sram_result* r) {
        r->legs = call.legs;
        r->bytes_per_sm = 8ull * call.n_words;
        for (unsigned l = 0; l < kLegs; ++l) {
            if (!(call.legs >> l & 1u)) continue;
            const bool net = l == CRO_SRAM_DSMEM;
            r->leg[l].iterations = call.iterations;
            r->leg[l].cluster = net ? call.cluster : 0u;
            if (!net) closed_form(r->seed, call.n_words, call.iterations, &r->leg[l]);
        }
    }
    static int grid(const Call& call, unsigned leg, int sm_count) { return leg == CRO_SRAM_DSMEM ? call.net_grid : sm_count; }
    static void args(const cro_sram_opts& o, const Call& call, unsigned leg, SramArgs* a) {
        a->n_words = call.n_words;
        a->inj_sm = o.test_inject_sm;
        a->inj_word = o.test_inject_word;
        a->inj_element = o.test_inject_element;
        a->inj_iter = o.test_inject_iteration;
        a->inj_mask = o.test_inject_leg == (int)leg ? o.test_inject_mask : 0ull;
    }
    static cudaError_t launch(const Call& call, unsigned leg, SramArgs& a, uint32_t round, int grid, cudaStream_t st) {
        a.round = round;
        return leg == CRO_SRAM_DSMEM ? launch_sram_dsmem(a, grid, call.cluster, st) : launch_sram_smem(a, grid, st);
    }
    // Each CTA reads and writes its words: local M0 and M5 every word once, M1 .. M4 twice; network D0, D2, D3 once and
    // D1 once per peer.  The network leg maps each round's blocks to their SMs, to name the peer of its records.
    static void round(Call& call, cro_sram_leg& R, unsigned leg, const cro_sram_cta* hc, int grid, uint64_t k) {
        const bool net = leg == CRO_SRAM_DSMEM;
        R.bytes += 8ull * call.n_words * call.iterations * (net ? call.cluster + 2 : 10) * (uint64_t)grid;
        if (!net) return;
        std::vector<uint32_t>& m = call.block_smid.emplace_back((size_t)grid);
        for (int j = 0; j < grid; ++j) m[(size_t)j] = hc[j].stamp == k ? hc[j].smid : ~0u;
    }
    static bool folds(unsigned leg) { return leg == CRO_SRAM_SMEM; }

    static int close(cro_sram_result* r, const CellTally<SramProbe>& t, const Call& call, std::vector<cro_sram_sm>* sms,
                     std::vector<cro_sram_fault>* faults);
    static void keep(cro_sram_result* r, const cro_sram_result& from) {
        r->legs = from.legs;
        r->bytes_per_sm = from.bytes_per_sm;
    }
};

// The call's end: the word records with the owner or writer resolved from the CTAs' own records of the same round,
// the SMs that failed the local leg, the network pairs between SMs that passed it, and the verdict.
int SramProbe::close(cro_sram_result* r, const CellTally<SramProbe>& t, const Call& call, std::vector<cro_sram_sm>* sms,
                     std::vector<cro_sram_fault>* faults) {
    for (uint32_t leg = 0; leg < CRO_SRAM_LEGS; ++leg)
        for (const cro_sram_record& q : t.recs[leg]) {
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
                f.peer_smid = q.round < call.block_smid.size() && q.peer_block < call.block_smid[q.round].size()
                                  ? call.block_smid[q.round][q.peer_block]
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

std::string sram_opts_error(const cro_sram_opts& o) {
    const uint32_t legs = o.legs ? o.legs : CRO_SRAM_ALL_LEGS;
    const uint32_t iters = o.iterations ? o.iterations : kSramDefaultIterations;
    const uint32_t cluster = o.cluster ? o.cluster : kSramDefaultCluster;
    const uint32_t max_rounds = o.max_rounds ? o.max_rounds : kSramDefaultRounds;
    if ((legs & ~CRO_SRAM_ALL_LEGS) || iters > CRO_SRAM_MAX_ITERATIONS || (cluster != 2 && cluster != 4 && cluster != 8) ||
        max_rounds > CRO_SRAM_MAX_ROUNDS || !valid_injection(o, iters))
        return "SRAM probe: legs must be CRO_SRAM_ALL_LEGS bits, iterations at most " + std::to_string(CRO_SRAM_MAX_ITERATIONS) +
               ", cluster 2, 4 or 8, max_rounds at most " + std::to_string(CRO_SRAM_MAX_ROUNDS) +
               ", and an injection must name a leg, an element it has (local 1 .. 5, network 1 or 2), an SM id below " +
               std::to_string(CRO_SRAM_MAX_SMS) + " (or -1), an iteration the call runs and a word (or -1)";
    return "";
}

int ctx_probe_sram(cro_ctx* c, int idx, const cro_sram_opts& o, cro_sram_result* r, std::vector<cro_sram_sm>* sms,
                   std::vector<cro_sram_fault>* faults) {
    return probe_cells<SramProbe>(c, idx, o, r, sms, faults);
}

int classify_sram(uint32_t legs, uint32_t iterations, uint32_t n_words, uint64_t seed, uint32_t cluster, uint32_t sm_count,
                  uint32_t net_grid, uint64_t k, const uint32_t* rounds, const cro_sram_cta* ctas, const uint64_t* claims,
                  const cro_sram_record* records, cro_sram_result* r, std::vector<cro_sram_sm>* sms,
                  std::vector<cro_sram_fault>* faults) {
    return classify_cells<SramProbe>({legs, iterations, n_words, cluster, (int)net_grid, {}}, seed, sm_count, k, rounds, ctas, claims,
                                     records, r, sms, faults);
}

int ctx_probe_sram_uuid(cro_ctx* c, const char* uuid, const cro_sram_opts& o, cro_sram_result* r, std::vector<cro_sram_sm>* sms,
                        std::vector<cro_sram_fault>* faults, int cap) {
    return probe_cells_uuid<SramProbe>(c, uuid, o, r, sms, faults, cap);
}

}  // namespace cro
