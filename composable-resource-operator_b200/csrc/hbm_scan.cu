// hbm_scan.cu — the whole-HBM scan (cro_scan_hbm, cro_scan_hbm_uuid): every byte of a GPU's memory that nobody holds,
// written and read back as 0 and as 1 with the probe's own fill and the locator's compare, and the DRAM health record
// NVML keeps for it.
#include <unistd.h>

#include <atomic>
#include <map>

#include "probe_internal.hpp"

namespace cro {

uint64_t fresh_seed() {
    static std::atomic<uint64_t> calls{0};
    const uint64_t t = (uint64_t)std::chrono::system_clock::now().time_since_epoch().count();
    const uint64_t s = pattern_word(t ^ ((uint64_t)getpid() << 40), calls.fetch_add(1) * kNonceStride);
    return s ? s : 1;     // 0 asks for a fresh seed: never report it as the one used
}

namespace {
constexpr int kCfSlot0 = CRO_SCAN_PASSES * CRO_SCAN_MAX_CHUNKS;   // slots [p * MAX + k] compare folds, then closed forms

void blank_report(cro_scan_report* rep, std::vector<cro_fault_word>* words) {
    memset(rep, 0, sizeof *rep);
    words->clear();
}

// The chunks of one call, freed on every way out.
struct Chunks {
    std::vector<unsigned char*> p;
    void release() {
        for (unsigned char* q : p) cudaFree(q);
        p.clear();
    }
    ~Chunks() { release(); }
};

struct Events {
    cudaEvent_t ev[CRO_SCAN_ELEMENTS + 1] = {};
    ~Events() {
        for (cudaEvent_t e : ev)
            if (e) cudaEventDestroy(e);
    }
};

// One element over every chunk: E0 / E2 fill the pattern / its complement (then the test force), E1 / E3 compare.
cudaError_t launch_element(cro_ctx* c, Device* d, int e, const cro_scan_report& rep, const Chunks& ch, const cro_scan_opts& o,
                           const MismatchView& dv, const SweepScratch& sc) {
    const uint64_t first = o.test_force_first, last = o.test_force_first + o.test_force_count;
    for (uint32_t k = 0; k < rep.n_chunks; ++k) {
        const cro_scan_chunk& K = rep.chunk[k];
        const uint64_t seed = rep.seed + K.word0, n = K.bytes / 8;
        cudaError_t ce;
        if (e % 2 == 0) {
            if ((ce = launch_fill(d->plan, ch.p[k], K.bytes, Params{ProbeParams{seed, 0}, nullptr}, sc, nullptr, d->stream, e == 2)))
                return ce;
            c->launches++;
            const uint64_t lo = std::max(first, K.word0), hi = std::min(last, K.word0 + n);
            if (o.test_force_count && lo < hi) {
                if ((ce = launch_force_words(ch.p[k], lo - K.word0, hi - lo, o.test_force_and, o.test_force_or, d->plan.sm_count,
                                             d->stream)))
                    return ce;
                c->launches++;
            }
        } else {
            const int p = e / 2;
            if ((ce = launch_locate(d->plan, ch.p[k], K.bytes, K.word0, seed, p ? ~0ull : 0ull, dv.check(p), sc,
                                    &dv.slots[p * CRO_SCAN_MAX_CHUNKS + k], d->stream)))
                return ce;
            c->launches++;
        }
    }
    return cudaSuccess;
}

// Per pass: counts, bit flips, granules and the records merged by scan index; per chunk its folds and whether the
// recorded deltas reproduce fold minus closed form.  Passes whose compare element did not complete stay blank.
void collect(const MismatchView& hv, bool have_cf, cro_scan_report* rep, std::vector<cro_fault_word>* words) {
    std::map<uint64_t, cro_fault_word> merged;
    bool complete = have_cf && rep->elements_done == CRO_SCAN_ELEMENTS;
    const uint32_t nc = rep->n_chunks;
    std::vector<uint64_t> starts(nc);
    for (uint32_t k = 0; k < nc; ++k) starts[k] = rep->chunk[k].word0;
    for (int p = 0; p < CRO_SCAN_PASSES; ++p) {
        if ((uint32_t)(2 * p + 1) >= rep->elements_done) break;
        cro_scan_pass& P = rep->pass[p];
        P.invert = p ? ~0ull : 0ull;
        P.mismatches = hv.ctr[p].mismatches;
        P.recorded = std::min<uint64_t>(hv.ctr[p].claims, kLocateRecords);
        if (P.recorded != P.mismatches) complete = false;
        for (int b = 0; b < 64; ++b) P.bit_flips[b] = hv.ctr[p].bits[b];
        for (uint64_t w = 0; w < hv.gran_words; ++w) P.granules += (uint64_t)__builtin_popcountll(hv.gran[p * hv.gran_words + w]);
        std::vector<uint64_t> dx(nc), ds(nc), dw(nc);
        for (uint64_t j = 0; j < P.recorded; ++j) {
            const LocateRecord& R = hv.rec[(size_t)p * kLocateRecords + j];
            const uint32_t k = (uint32_t)(std::upper_bound(starts.begin(), starts.end(), R.word) - starts.begin()) - 1;
            const uint64_t i = R.word - starts[k], delta = R.actual - R.expected;
            dx[k] ^= R.actual ^ R.expected;
            ds[k] += delta;
            dw[k] += delta * (2 * i + 1);
            rep->flip_or |= R.actual ^ R.expected;
            auto it = merged.find(R.word);
            if (it == merged.end()) merged[R.word] = cro_fault_word{R.word, R.expected, R.actual, 1u << p, k};
            else it->second.passes |= 1u << p;
        }
        for (uint32_t k = 0; k < nc; ++k) {
            cro_scan_chunk& K = rep->chunk[k];
            const SweepOut& s = hv.slots[p * CRO_SCAN_MAX_CHUNKS + k];
            P.words_scanned += s.n_words;
            K.fold_xor[p] = s.x;
            K.fold_sum[p] = s.s;
            K.fold_wsum[p] = s.w;
            if (!have_cf) continue;
            SweepOut cf = hv.slots[kCfSlot0 + k];
            if (p == 0) { K.expect_xor = cf.x; K.expect_sum = cf.s; K.expect_wsum = cf.w; }
            else cf = complement_fold(cf, K.bytes / 8);
            if ((s.x ^ cf.x) != dx[k] || s.s - cf.s != ds[k] || s.w - cf.w != dw[k]) complete = false;
        }
    }
    rep->located = merged.size();
    for (const auto& kv : merged) words->push_back(kv.second);
    rep->complete = complete ? 1u : 0u;
}
}  // namespace

uint32_t scan_health(const cro_hbm_health& b, const cro_hbm_health& a) {
    uint32_t h = 0;
    if ((b.nvml & a.nvml & CRO_HBM_NVML_ECC_CORRECTED) && a.ecc_corrected > b.ecc_corrected) h |= CRO_SCAN_HEALTH_ECC_CORRECTED_DURING;
    if ((b.nvml & a.nvml & CRO_HBM_NVML_ECC_UNCORRECTED) && a.ecc_uncorrected > b.ecc_uncorrected)
        h |= CRO_SCAN_HEALTH_ECC_UNCORRECTED_DURING;
    const cro_hbm_health& r = (a.nvml & CRO_HBM_NVML_REMAP) ? a : b;      // the latest remap state NVML gave
    if ((r.nvml & CRO_HBM_NVML_REMAP) && r.remap_pending) h |= CRO_SCAN_HEALTH_REMAP_PENDING;
    if ((r.nvml & CRO_HBM_NVML_REMAP) && r.remap_failure) h |= CRO_SCAN_HEALTH_REMAP_FAILURE;
    return h;
}

int ctx_scan_hbm(cro_ctx* c, int idx, const cro_scan_opts& o, cro_scan_report* rep, std::vector<cro_fault_word>* words) {
    const uint64_t t_call = now_ns();
    blank_report(rep, words);
    Device* d = dev_at(c, idx);
    if (!d) return rep->status = unknown_device(c, idx, "a GPU attached after init is scanned through the helper process, cro_scan_hbm_uuid");
    const uint64_t chunk_bytes = o.test_chunk_bytes ? o.test_chunk_bytes : CRO_SCAN_CHUNK_BYTES;
    if (chunk_bytes % 16 || o.reserved0) {
        c->set_error("scan chunk size must be a multiple of 16 bytes and reserved0 zero");
        return rep->status = CRO_ERR_INVALID_ARG;
    }
    DeviceGuard g = enter_device(c, idx);
    if (g.rc) return rep->status = g.rc;
    Range nv(c, "cro.scan_hbm");
    const std::string uuid(d->info.gpu_uuid, strnlen(d->info.gpu_uuid, sizeof d->info.gpu_uuid));
    Chunks ch;
    cudaError_t elem_err = cudaSuccess;
    int rc = [&]() -> int {
        size_t free_b = 0, total_b = 0;
        CU_TRY(c, cudaMemGetInfo(&free_b, &total_b));
        rep->free_bytes = free_b;
        rep->total_bytes = total_b;
        rep->held_bytes = d->region ? 2 * d->sweep_bytes : 0;
        const uint64_t reserve = o.reserve_bytes ? o.reserve_bytes : CRO_SCAN_RESERVE_BYTES;
        uint64_t target = free_b > reserve ? free_b - reserve : 0;
        if (o.max_bytes) target = std::min<uint64_t>(target, o.max_bytes);
        target &= ~(uint64_t)15;
        if (target == 0) {
            c->set_error("no room for one scan chunk: " + std::to_string(free_b) + " bytes free, " + std::to_string(reserve) +
                         " reserved");
            return CRO_ERR_OOM;
        }
        rep->seed = o.seed ? o.seed : fresh_seed();
        // the bookkeeping first, so that it does not compete with the chunks for the last free bytes
        MismatchBuffer mb;
        int r;
        if ((r = mb.ensure(c, CRO_SCAN_PASSES, target, kCfSlot0 + CRO_SCAN_MAX_CHUNKS, 0,
                           std::max({d->plan.locate.grid, d->plan.expect.grid, 1}), 1)))
            return r;
        Events ev;
        for (cudaEvent_t& e : ev.ev) CU_TRY(c, cudaEventCreate(&e));
        const uint64_t t_alloc = now_ns();
        uint64_t covered = 0;
        while (covered < target && ch.p.size() < CRO_SCAN_MAX_CHUNKS) {
            const uint64_t want = std::min(chunk_bytes, target - covered);
            unsigned char* q = nullptr;
            if (cudaMalloc(&q, want) != cudaSuccess) {     // the allocation phase ends here
                cudaGetLastError();
                break;
            }
            cro_scan_chunk& K = rep->chunk[ch.p.size()];
            K.word0 = covered / 8;
            K.bytes = want;
            ch.p.push_back(q);
            covered += want;
        }
        rep->alloc_ns = now_ns() - t_alloc;
        rep->n_chunks = (uint32_t)ch.p.size();
        rep->covered_bytes = covered;
        if (ch.p.empty()) {
            c->set_error("not one scan chunk of " + std::to_string(std::min(chunk_bytes, target)) + " bytes could be allocated");
            return CRO_ERR_OOM;
        }
        const uint64_t n_words = covered / 8;
        if (o.test_force_count && (o.test_force_first >= n_words || o.test_force_count > n_words - o.test_force_first)) {
            c->set_error("test force range lies outside the " + std::to_string(n_words) + " scan words");
            return CRO_ERR_INVALID_ARG;
        }
        const bool nvml = !(c->opts.flags & CRO_F_NO_NVML);
        uint64_t t_nvml = now_ns();
        if (nvml) identity::NvmlHbmHealth(uuid, false, &rep->before);
        rep->nvml_ns = now_ns() - t_nvml;

        const SweepScratch& sc = mb.scratch[0];
        const MismatchView dv = mb.dev();
        CU_TRY(c, cudaGetLastError());
        if ((r = mb.zero(c, d->stream))) return r;
        int e = 0;
        for (; e < CRO_SCAN_ELEMENTS; ++e) {
            cudaError_t ce = cudaEventRecord(ev.ev[e], d->stream);
            if (!ce) ce = launch_element(c, d, e, *rep, ch, o, dv, sc);
            if (!ce) ce = cudaEventRecord(ev.ev[e + 1], d->stream);
            if (!ce) ce = cudaEventSynchronize(ev.ev[e + 1]);
            if (ce) {
                elem_err = ce;
                c->set_error("scan element E" + std::to_string(e) + ": " + cudaGetErrorString(ce));
                break;
            }
            float ms = 0;
            cudaEventElapsedTime(&ms, ev.ev[e], ev.ev[e + 1]);
            rep->element_ns[e] = ms_to_ns(ms);
        }
        rep->elements_done = (uint32_t)e;
        t_nvml = now_ns();
        if (nvml) identity::NvmlHbmHealth(uuid, true, &rep->after);
        rep->nvml_ns += now_ns() - t_nvml;
        rep->health = scan_health(rep->before, rep->after);

        // the closed forms (ALU only) once every element ran; the counters as far as the scan got
        bool have_cf = false;
        if (!elem_err) {
            for (uint32_t k = 0; k < rep->n_chunks && !elem_err; ++k) {
                elem_err = launch_expected(d->plan, rep->chunk[k].bytes, Params{ProbeParams{rep->seed + rep->chunk[k].word0, 0}, nullptr},
                                           sc, &dv.slots[kCfSlot0 + k], d->stream);
                c->launches++;
            }
            have_cf = !elem_err;
        }
        if (elem_err && rep->elements_done < 2) return CRO_OK;
        if (mb.fetch(c, d->stream) != CRO_OK || cudaStreamSynchronize(d->stream) != cudaSuccess) {
            if (!elem_err) elem_err = cudaGetLastError();
            if (!elem_err) elem_err = cudaErrorUnknown;
            return CRO_OK;
        }
        collect(mb.host(), have_cf, rep, words);
        return CRO_OK;
    }();
    const uint64_t t_free = now_ns();
    ch.release();
    rep->alloc_ns += now_ns() - t_free;
    if (!rc && elem_err) {
        rep->cuda_error = (int32_t)elem_err;
        rc = CRO_ERR_CUDA;
    }
    if (!rc) {
        for (const cro_scan_pass& P : rep->pass) rc = rc ? rc : (P.mismatches ? CRO_ERR_CHECKSUM : CRO_OK);
    }
    if (rc == CRO_ERR_OOM || rc == CRO_ERR_INVALID_ARG) {
        // nothing was scanned: keep what says why (the sizes), drop the rest
        const cro_scan_report keep = *rep;
        blank_report(rep, words);
        rep->free_bytes = keep.free_bytes;
        rep->total_bytes = keep.total_bytes;
        rep->held_bytes = keep.held_bytes;
    }
    rep->wall_ns = now_ns() - t_call;
    return rep->status = rc;
}

namespace {
uint64_t scan_tail_count(const unsigned char* head) {
    return reinterpret_cast<const cro_scan_report*>(head)->recorded;
}
}  // namespace

int ctx_scan_hbm_uuid(cro_ctx* c, const char* uuid, const cro_scan_opts& o, cro_scan_report* rep, std::vector<cro_fault_word>* words,
                      int cap) {
    blank_report(rep, words);
    if (!uuid) return rep->status = CRO_ERR_INVALID_ARG;
    const std::string want = uuid;
    auto num = [](uint64_t v) { return std::to_string(v); };
    const std::vector<std::string> args = {"scan-raw", want, num(o.max_bytes), num(o.reserve_bytes), num(o.seed), num(o.test_chunk_bytes),
                                           num(o.test_force_first), num(o.test_force_count), num(o.test_force_and),
                                           num(o.test_force_or), num((uint64_t)cap)};
    std::string got;
    uint64_t helper_ns = 0;
    const int rc = run_probe_helper(c, want, "scan helper", "cro.scan_hbm.helper", args, o.deadline_ms, sizeof *rep,
                                    sizeof(cro_fault_word), (size_t)cap, scan_tail_count, &got, &helper_ns);
    if (rc != CRO_OK) return rep->status = rc;
    memcpy(rep, got.data(), sizeof *rep);
    const cro_fault_word* w = reinterpret_cast<const cro_fault_word*>(got.data() + sizeof *rep);
    words->assign(w, w + rep->recorded);
    rep->helper_ns = helper_ns;
    return rep->status;
}

}  // namespace cro
