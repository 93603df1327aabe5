// l2_probe.cu — the L2 probe (cro_probe_l2): an L2-resident buffer marched from SM to SM, the L2 atomic units checked
// against answers computed without atomics, and the SRAM / L2 ECC record NVML keeps.
#include <map>
#include <set>
#include <tuple>

#include "l2_kernels.cuh"
#include "probe_internal.hpp"

namespace cro {

namespace {
// W and iterations when the caller gives none.  On an H100 80GB HBM3 at a 700 W limit (profiles/h100_700w_l2_rate.jsonl)
// the read-and-write elements M1 .. M4 move 4.1-4.3 TB/s at W = 24 and 32 MiB, and M1, M2 and M4 fall to 2.7-2.8 TB/s
// at 48 and 64 MiB, under the 3.1 TB/s the locator reads HBM at: 32 MiB is the largest measured size that stays in the
// 50 MB L2.  24 iterations of it make a default call of 5.4 ms, about the SRAM probe's (DESIGN.md "The L2 probe").
constexpr uint64_t kL2DefaultBytes = 32ull << 20;
constexpr uint32_t kL2DefaultIterations = 24;
constexpr uint32_t kL2DefaultA1 = 65536;
constexpr uint32_t kL2DefaultA2 = 1024;

// The result of a call that marched nothing: zeroes but for what the call had settled before it stopped.
void blank_result(cro_l2_result* r, const cro_l2_result& from, std::vector<cro_l2_sm>* sms, std::vector<cro_l2_fault>* faults) {
    const cro_l2_result keep = from;
    memset(r, 0, sizeof *r);
    r->seed = keep.seed;
    r->seed_atomic = keep.seed_atomic;
    r->call = keep.call;
    r->bytes = keep.bytes;
    r->sm_count = keep.sm_count;
    r->ctas = keep.ctas;
    r->blocks = keep.blocks;
    r->delta = keep.delta;
    r->iterations = keep.iterations;
    r->a1_counters = keep.a1_counters;
    r->a2_counters = keep.a2_counters;
    r->a2_tickets = keep.a2_tickets;
    r->l2_bytes = keep.l2_bytes;
    r->cuda_error = keep.cuda_error;
    r->before = keep.before;
    r->after = keep.after;
    r->health = keep.health;
    sms->clear();
    faults->clear();
}

// Blocks CTA j handles in element el: those b < blocks with (b + el * delta) mod G == j.
uint64_t blocks_of(uint32_t j, uint32_t el, uint32_t blocks, uint32_t G, uint32_t delta) {
    const uint32_t b0 = (uint32_t)((j + G - (uint64_t)el * delta % G) % G);
    return b0 < blocks ? (blocks - 1 - b0) / G + 1 : 0;
}
}  // namespace

// The rotation step: M1 .. M5 of a word run on CTAs b + delta, ..., b + 5 * delta (mod G), distinct when no k * delta
// with k = 1 .. 4 is a multiple of G.  delta = G / 5 keeps 4 * delta below G; G < 5 has no such step.
uint32_t l2_delta(uint32_t G) { return G < 5 ? 0u : G / 5; }

bool l2_check_args(const cro_l2_opts& o, uint64_t l2_size, bool helper, L2Settings* p, std::string* why) {
    p->bytes = o.bytes ? o.bytes : kL2DefaultBytes;
    p->iterations = o.iterations ? o.iterations : kL2DefaultIterations;
    p->a1 = o.a1_counters ? o.a1_counters : kL2DefaultA1;
    p->a2 = o.a2_counters ? o.a2_counters : kL2DefaultA2;
    const uint64_t max_bytes = l2_size ? (uint64_t)CRO_L2_MAX_L2_MULTIPLE * l2_size : ~0ull;
    bool ok = p->bytes % CRO_L2_BLOCK_BYTES == 0 && p->bytes >= CRO_L2_MIN_BYTES && p->bytes <= max_bytes &&
              p->iterations <= CRO_L2_MAX_ITERATIONS && p->a1 <= CRO_L2_MAX_A1_COUNTERS && p->a2 <= CRO_L2_MAX_A2_COUNTERS &&
              (helper ? o.deadline_ms >= 0 : o.deadline_ms == 0);
    if (ok && o.test_inject_mask) {
        const int64_t w = o.test_inject_word;
        switch (o.test_inject_leg) {
            case CRO_L2_MARCH:
                ok = o.test_inject_sm >= -1 && o.test_inject_sm < CRO_L2_MAX_SMS &&
                     (o.test_inject_element == -1 || (o.test_inject_element >= 1 && o.test_inject_element <= 5)) &&
                     o.test_inject_iteration < p->iterations && w >= -1 && w < (int64_t)(p->bytes / 8);
                break;
            case CRO_L2_A1: ok = w >= 0 && w < (int64_t)p->a1; break;
            case CRO_L2_A2: ok = w >= 0 && w < (int64_t)p->a2 && (uint32_t)o.test_inject_mask != 0; break;
            default: ok = false;
        }
    }
    if (!ok)
        *why = "L2 probe: bytes must be a multiple of " + std::to_string(CRO_L2_BLOCK_BYTES) + " from " +
               std::to_string(CRO_L2_MIN_BYTES) + (l2_size ? " to " + std::to_string(max_bytes) : std::string()) +
               " (8 times the L2), iterations at most " + std::to_string(CRO_L2_MAX_ITERATIONS) + ", a1_counters at most " +
               std::to_string(CRO_L2_MAX_A1_COUNTERS) + ", a2_counters at most " + std::to_string(CRO_L2_MAX_A2_COUNTERS) +
               (helper ? ", deadline_ms not negative" : ", deadline_ms 0 (only the helper form has a deadline of its own)") +
               ", and an injection must name a leg and, for the march, an SM id below " + std::to_string(CRO_L2_MAX_SMS) +
               " (or -1), an element 1 .. 5 (or -1), an iteration the call runs and a word of the buffer (or -1); for A1 or "
               "A2 a counter the leg has, and for A2 a mask with a bit in its low 32";
    return ok;
}

uint32_t l2_health(const cro_l2_health& b, const cro_l2_health& a) {
    uint32_t h = 0;
    const uint32_t both = b.nvml & a.nvml;
    if ((both & CRO_L2_NVML_SRAM_CORRECTED) && a.sram_corrected > b.sram_corrected) h |= CRO_L2_HEALTH_SRAM_CORRECTED_DURING;
    if ((both & CRO_L2_NVML_SRAM_UNCORRECTED) && a.sram_uncorrected > b.sram_uncorrected) h |= CRO_L2_HEALTH_SRAM_UNCORRECTED_DURING;
    if ((both & CRO_L2_NVML_L2_CORRECTED) && a.l2_corrected > b.l2_corrected) h |= CRO_L2_HEALTH_L2_CORRECTED_DURING;
    if ((both & CRO_L2_NVML_L2_UNCORRECTED) && a.l2_uncorrected > b.l2_uncorrected) h |= CRO_L2_HEALTH_L2_UNCORRECTED_DURING;
    if ((a.nvml & CRO_L2_NVML_STATUS) && a.threshold_exceeded) h |= CRO_L2_HEALTH_THRESHOLD_EXCEEDED;
    if ((a.nvml & CRO_L2_NVML_STATUS) && a.unc_bucket_l2) h |= CRO_L2_HEALTH_L2_BUCKET;
    return h;
}

void l2_classify(cro_l2_result* r, cro_l2_sm* sms, size_t n_sms, cro_l2_fault* f, size_t n) {
    std::map<uint64_t, std::set<uint32_t>> readers;          // word -> the SMs that saw it wrong
    for (size_t i = 0; i < n; ++i) readers[f[i].word].insert(f[i].smid);
    std::set<uint32_t> bad;
    std::vector<uint64_t> lines;
    for (const auto& kv : readers) {
        if (kv.second.size() >= 2) lines.push_back(kv.first);
        else bad.insert(*kv.second.begin());
    }
    for (size_t i = 0; i < n; ++i) f[i].line = readers[f[i].word].size() >= 2 ? 1u : 0u;
    // Common cause: every SM that read words in an element where some read went wrong saw a wrong word.  Only the
    // elements' readers count: with fewer blocks than CTAs, an SM whose CTA owns no block in an element reads nothing
    // there and cannot fail it.
    bool failed_el[CRO_L2_ELEMENTS] = {};
    uint64_t total = 0;
    for (size_t i = 0; i < n_sms; ++i)
        for (int e = 0; e < CRO_L2_ELEMENTS; ++e) {
            failed_el[e] = failed_el[e] || sms[i].mismatches[e];
            total += sms[i].mismatches[e];
        }
    bool every = total != 0;
    for (size_t i = 0; i < n_sms; ++i) {
        uint64_t any = 0;
        bool reader = false;
        for (int e = 0; e < CRO_L2_ELEMENTS; ++e) {
            any += sms[i].mismatches[e];
            reader = reader || (failed_el[e] && sms[i].words_read[e]);
        }
        if (reader && !any) every = false;
        sms[i].mark = sms[i].last ? CRO_L2_PERSISTENT : any ? CRO_L2_INTERMITTENT : 0u;
    }
    r->bad_sms = (uint32_t)bad.size();
    memset(r->bad_sm, 0, sizeof r->bad_sm);
    uint32_t j = 0;
    for (uint32_t s : bad)
        if (j < 16) r->bad_sm[j++] = (uint16_t)s;
    r->bad_lines = (uint32_t)lines.size();
    memset(r->bad_line, 0, sizeof r->bad_line);
    for (size_t i = 0; i < lines.size() && i < CRO_L2_MAX_LINES; ++i) r->bad_line[i] = 8 * lines[i];
    const bool all = r->unpublished || every || (!r->fold_ok && !r->mismatches[5]) ||
                     (total && !n);                           // mismatches counted but none recorded: nothing to name
    r->verdict = all ? CRO_L2_ALL : !lines.empty() ? CRO_L2_LINE : !bad.empty() ? CRO_L2_SM
                 : (r->a1_bad || r->a2_bad) ? CRO_L2_ATOMIC : CRO_L2_NONE;
    r->status = r->verdict == CRO_L2_NONE ? CRO_OK : CRO_ERR_CHECKSUM;
}

int ctx_probe_l2(cro_ctx* c, int idx, const cro_l2_opts& o, cro_l2_result* r, std::vector<cro_l2_sm>* sms,
                 std::vector<cro_l2_fault>* faults) {
    const uint64_t t_call = now_ns();
    blank_result(r, cro_l2_result{}, sms, faults);
    Device* d = dev_at(c, idx);
    if (!d) return r->status = unknown_device(c, idx, "the L2 probe runs on a device of this context");
    int l2_size = 0;
    const cudaError_t ae = cudaDeviceGetAttribute(&l2_size, cudaDevAttrL2CacheSize, d->ordinal);
    if (ae != cudaSuccess) {
        c->set_error(std::string("L2 probe: cudaDeviceGetAttribute(cudaDevAttrL2CacheSize): ") + cudaGetErrorString(ae));
        r->cuda_error = (int32_t)ae;
        return r->status = CRO_ERR_CUDA;
    }
    L2Settings p;
    std::string why;
    if (!l2_check_args(o, (uint64_t)l2_size, false, &p, &why)) {
        c->set_error(why);
        return r->status = CRO_ERR_INVALID_ARG;
    }
    DeviceGuard g = enter_device(c, idx);
    if (g.rc) return r->status = g.rc;
    Range nv(c, "cro.probe_l2");
    const std::string uuid(d->info.gpu_uuid, strnlen(d->info.gpu_uuid, sizeof d->info.gpu_uuid));
    const bool nvml = !(c->opts.flags & CRO_F_NO_NVML);
    std::map<uint32_t, cro_l2_sm> per_sm;
    bool ran = false;
    cudaEvent_t ev[6] = {};                                    // the call's own, destroyed on every way out
    int rc = [&]() -> int {
        const uint32_t G = (uint32_t)d->plan.sm_count, delta = l2_delta(G);
        if (!delta) {
            c->set_error("L2 probe: the device has " + std::to_string(G) + " SMs; the rotation needs at least 5");
            return CRO_ERR_UNSUPPORTED;
        }
        size_t dyn = 0;
        CU_TRY(c, l2_plan(d->ordinal, &dyn));
        const uint64_t k = d->l2_calls++;
        const uint64_t launches = (uint64_t)p.iterations * CRO_L2_ELEMENTS;
        r->seed = space_seed(d, kSeedL2, k, 0);
        r->seed_atomic = space_seed(d, kSeedL2, k, 1);
        r->call = k;
        r->bytes = p.bytes;
        r->sm_count = G;
        r->ctas = G;
        r->blocks = (uint32_t)(p.bytes / CRO_L2_BLOCK_BYTES);
        r->delta = delta;
        r->iterations = p.iterations;
        r->a1_counters = p.a1;
        r->a2_counters = p.a2;
        r->a2_tickets = 32 * G;
        r->l2_bytes = (uint64_t)l2_size;

        // [claims, closed form][records][CTA records][A1 sums][A1 xors][A2 counters][tickets][presence][A1 bad][A2 bad][partials],
        // allocated per call
        const uint64_t per = 32ull * G;
        auto up = [](size_t x) { return (x + 255) & ~(size_t)255; };
        const size_t o_rec = 256, o_cta = up(o_rec + CRO_L2_RECORDS * sizeof(cro_l2_fault));
        const size_t o_sum = up(o_cta + launches * G * sizeof(L2Cta)), o_xor = up(o_sum + 8ull * p.a1);
        const size_t o_ctr = up(o_xor + 8ull * p.a1), o_tk = up(o_ctr + 128ull * p.a2);
        const size_t o_pr = up(o_tk + 4 * per * p.a2), o_b1 = up(o_pr + per * p.a2), o_b2 = up(o_b1 + p.a1);
        const unsigned c1 = l2_a1_check_ctas(p.a1), c2 = l2_a2_check_ctas(p.a2);
        const size_t o_p1 = up(o_b2 + p.a2), o_p2 = up(o_p1 + 8ull * c1), total = o_p2 + 16ull * c2;
        DeviceMem<unsigned char> buf, b;
        CU_TRY(c, cudaMalloc(&buf.p, p.bytes));
        CU_TRY(c, cudaMalloc(&b.p, total));
        for (cudaEvent_t& x : ev) CU_TRY(c, cudaEventCreate(&x));
        cudaStream_t st = d->stream;
        CU_TRY(c, cudaMemsetAsync(b.p, 0, o_rec, st));
        CU_TRY(c, cudaMemsetAsync(b.p + o_cta, 0xFF, o_sum - o_cta, st));          // armed: a silent CTA stays all ones
        CU_TRY(c, cudaMemsetAsync(b.p + o_sum, 0, o_tk - o_sum, st));
        CU_TRY(c, cudaMemsetAsync(b.p + o_pr, 0, o_b1 - o_pr, st));
        CU_TRY(c, cudaMemsetAsync(b.p + o_p1, 0xFF, total - o_p1, st));
        // what the combined M5 fold must be: the read-sweep closed form of pattern_word(seed, 0 .. W / 8), once per
        // iteration (the probe's own generator, on the stream's scratch, which the guard keeps to this call)
        SweepOut* cf = reinterpret_cast<SweepOut*>(b.p + 64);
        CU_TRY(c, launch_expected(d->plan, p.bytes, Params{ProbeParams{r->seed, 0}, nullptr}, d->scratch, cf, st));
        c->launches++;
        if (nvml) identity::NvmlL2Health(uuid, false, &r->before);
        ran = true;

        L2Args a{};
        a.buf = reinterpret_cast<ulonglong2*>(buf.p);
        a.cta = reinterpret_cast<L2Cta*>(b.p + o_cta);
        a.rec = reinterpret_cast<cro_l2_fault*>(b.p + o_rec);
        a.claims = reinterpret_cast<unsigned long long*>(b.p);
        a.seed = r->seed;
        a.stamp = k;
        a.blocks = r->blocks;
        a.G = G;
        a.delta = delta;
        const bool march_inj = o.test_inject_mask && o.test_inject_leg == CRO_L2_MARCH;
        a.inj_sm = o.test_inject_sm;
        a.inj_element = o.test_inject_element;
        a.inj_iter = o.test_inject_iteration;
        a.inj_word = o.test_inject_word;
        a.inj_mask = march_inj ? o.test_inject_mask : 0ull;
        L2AtomicArgs t{};
        t.a1_sum = reinterpret_cast<unsigned long long*>(b.p + o_sum);
        t.a1_xor = reinterpret_cast<unsigned long long*>(b.p + o_xor);
        t.a2_ctr = reinterpret_cast<unsigned*>(b.p + o_ctr);
        t.tickets = reinterpret_cast<unsigned*>(b.p + o_tk);
        t.present = b.p + o_pr;
        t.a1_bad = b.p + o_b1;
        t.a2_bad = b.p + o_b2;
        t.a1_partial = reinterpret_cast<unsigned long long*>(b.p + o_p1);
        t.a2_partial = reinterpret_cast<unsigned long long*>(b.p + o_p2);
        t.seed = r->seed_atomic;
        t.a1 = p.a1;
        t.a2 = p.a2;
        t.G = G;
        t.inj_leg = o.test_inject_mask && !march_inj ? o.test_inject_leg : -1;
        t.inj_counter = (unsigned long long)o.test_inject_word;
        t.inj_mask = o.test_inject_mask;

        CU_TRY(c, cudaEventRecord(ev[0], st));
        for (uint32_t it = 0; it < p.iterations; ++it)
            for (uint32_t el = 0; el < CRO_L2_ELEMENTS; ++el) {
                CU_TRY(c, launch_l2_march(a, el, it, dyn, st));
                c->launches++;
            }
        CU_TRY(c, cudaEventRecord(ev[1], st));
        CU_TRY(c, launch_l2_a1(t, st));
        CU_TRY(c, cudaEventRecord(ev[2], st));
        CU_TRY(c, launch_l2_a1_check(t, st));
        CU_TRY(c, cudaEventRecord(ev[3], st));
        CU_TRY(c, launch_l2_a2(t, st));
        CU_TRY(c, cudaEventRecord(ev[4], st));
        CU_TRY(c, launch_l2_a2_check(t, st));
        CU_TRY(c, cudaEventRecord(ev[5], st));
        CU_TRY(c, launch_l2_release(buf.p, p.bytes, (int)G, st));
        c->launches += 5;

        unsigned long long n_claims = 0;
        SweepOut hcf{};
        std::vector<cro_l2_fault> rec(CRO_L2_RECORDS);
        std::vector<L2Cta> hc((size_t)(launches * G));
        std::vector<unsigned char> bad1(p.a1), bad2(p.a2);
        std::vector<unsigned long long> p1(c1), p2(2ull * c2);
        CU_TRY(c, cudaMemcpyAsync(&n_claims, a.claims, sizeof n_claims, cudaMemcpyDeviceToHost, st));
        CU_TRY(c, cudaMemcpyAsync(&hcf, cf, sizeof hcf, cudaMemcpyDeviceToHost, st));
        CU_TRY(c, cudaMemcpyAsync(rec.data(), a.rec, rec.size() * sizeof(cro_l2_fault), cudaMemcpyDeviceToHost, st));
        CU_TRY(c, cudaMemcpyAsync(hc.data(), a.cta, hc.size() * sizeof(L2Cta), cudaMemcpyDeviceToHost, st));
        CU_TRY(c, cudaMemcpyAsync(bad1.data(), t.a1_bad, bad1.size(), cudaMemcpyDeviceToHost, st));
        CU_TRY(c, cudaMemcpyAsync(bad2.data(), t.a2_bad, bad2.size(), cudaMemcpyDeviceToHost, st));
        CU_TRY(c, cudaMemcpyAsync(p1.data(), t.a1_partial, 8 * p1.size(), cudaMemcpyDeviceToHost, st));
        CU_TRY(c, cudaMemcpyAsync(p2.data(), t.a2_partial, 8 * p2.size(), cudaMemcpyDeviceToHost, st));
        const int w = wait_stream(c, d);
        if (w) return w;
        float ms[5] = {};
        for (int i = 0; i < 5; ++i) CU_TRY(c, cudaEventElapsedTime(&ms[i], ev[i], ev[i + 1]));
        r->march_ns = ms_to_ns(ms[0]);
        r->a1_ns = ms_to_ns(ms[1]);
        r->a1_check_ns = ms_to_ns(ms[2]);
        r->a2_ns = ms_to_ns(ms[3]);
        r->a2_check_ns = ms_to_ns(ms[4]);
        r->march_bytes = 10ull * p.bytes * p.iterations;      // M0, M5 touch every word once, M1 .. M4 twice
        r->expect_xor = (p.iterations & 1) ? hcf.x : 0;
        r->expect_sum = hcf.s * p.iterations;
        r->expect_wsum = hcf.w * p.iterations;

        // the CTAs' records: per SM, per element, the fold; smid_of resolves a record's writer
        std::vector<uint32_t> smid_of(hc.size(), ~0u);
        std::set<uint32_t> seen;
        for (uint64_t l = 0; l < launches; ++l) {
            const uint32_t el = (uint32_t)(l % CRO_L2_ELEMENTS), it = (uint32_t)(l / CRO_L2_ELEMENTS);
            uint64_t t0 = ~0ull, t1 = 0;
            for (uint32_t j = 0; j < G; ++j) {
                const L2Cta& x = hc[l * G + j];
                if (x.stamp != k) {
                    r->unpublished++;
                    continue;
                }
                if (x.nsmid > CRO_L2_MAX_SMS) {
                    c->set_error("L2 probe: the device reports %nsmid = " + std::to_string(x.nsmid) + ", more SM ids than the " +
                                 std::to_string(CRO_L2_MAX_SMS) + " the result holds");
                    return CRO_ERR_UNSUPPORTED;
                }
                r->nsmid = x.nsmid;
                smid_of[l * G + j] = x.smid;
                if (el && blocks_of(j, el, r->blocks, G, delta)) seen.insert(x.smid);    // covered: it read words
                t0 = std::min<uint64_t>(t0, x.t0);
                t1 = std::max<uint64_t>(t1, x.t1);
                cro_l2_sm& S = per_sm[x.smid];
                S.smid = x.smid;
                S.launches++;
                S.mismatches[el] += x.count;
                if (it + 1 == p.iterations) S.last += x.count;
                if (el) S.words_read[el] += blocks_of(j, el, r->blocks, G, delta) * kL2BlockWords;
                S.ns += x.t1 > x.t0 ? x.t1 - x.t0 : 0;
                r->mismatches[el] += x.count;
                if (el == 5) {
                    r->fold_xor ^= x.fx;
                    r->fold_sum += x.fs;
                    r->fold_wsum += x.fw;
                }
            }
            if (t1 > t0) r->element_ns[el] += t1 - t0;
        }
        r->sms_covered = (uint32_t)seen.size();
        r->fold_ok = r->fold_xor == r->expect_xor && r->fold_sum == r->expect_sum && r->fold_wsum == r->expect_wsum ? 1u : 0u;
        uint64_t wrong = 0;
        for (uint64_t m : r->mismatches) wrong += m;
        const uint64_t kept = std::min<uint64_t>(n_claims, CRO_L2_RECORDS);
        r->overflow = wrong > kept ? 1u : 0u;
        for (uint64_t i = 0; i < kept; ++i) {
            cro_l2_fault f = rec[(size_t)i];
            const uint64_t wl = (uint64_t)f.iteration * CRO_L2_ELEMENTS + f.element - 1;    // the writer's launch
            f.writer_smid = f.element >= 1 && wl < launches && f.writer_cta < G ? smid_of[wl * G + f.writer_cta] : ~0u;
            faults->push_back(f);
        }
        for (unsigned long long x : p1) {
            if (x == ~0ull) r->unpublished++;
            else r->a1_bad += x;
        }
        for (unsigned i = 0; i < c2; ++i) {
            if (p2[2 * i] == ~0ull) {
                r->unpublished++;
                continue;
            }
            r->a2_holes += p2[2 * i];
            r->a2_bad += p2[2 * i + 1];
        }
        for (uint32_t i = 0, m = 0; i < p.a1 && m < CRO_L2_MAX_COUNTERS; ++i)
            if (bad1[i]) r->a1_bad_counter[m++] = i;
        for (uint32_t i = 0, m = 0; i < p.a2 && m < CRO_L2_MAX_COUNTERS; ++i)
            if (bad2[i]) r->a2_bad_counter[m++] = i;
        return CRO_OK;
    }();
    for (cudaEvent_t x : ev)
        if (x) cudaEventDestroy(x);
    if (rc == CRO_ERR_CUDA) r->cuda_error = (int32_t)cudaGetLastError();
    if (ran && nvml) identity::NvmlL2Health(uuid, true, &r->after);
    r->health = l2_health(r->before, r->after);
    if (rc) {
        blank_result(r, *r, sms, faults);
        r->wall_ns = now_ns() - t_call;
        return r->status = rc;
    }
    for (auto& kv : per_sm) sms->push_back(kv.second);
    std::sort(faults->begin(), faults->end(), [](const cro_l2_fault& x, const cro_l2_fault& y) {
        return std::make_tuple(x.word, x.iteration, x.element, x.smid) < std::make_tuple(y.word, y.iteration, y.element, y.smid);
    });
    l2_classify(r, sms->data(), sms->size(), faults->data(), faults->size());
    r->wall_ns = now_ns() - t_call;
    return r->status;
}

int ctx_probe_l2_uuid(cro_ctx* c, const char* uuid, const cro_l2_opts& o, cro_l2_result* r, std::vector<cro_l2_sm>* sms,
                      std::vector<cro_l2_fault>* faults, int cap) {
    blank_result(r, cro_l2_result{}, sms, faults);
    if (!uuid) return r->status = CRO_ERR_INVALID_ARG;
    L2Settings p;
    std::string why;
    if (!l2_check_args(o, 0, true, &p, &why)) {     // W's upper bound needs the device: the helper checks it
        set_call_error(c, why);
        return r->status = CRO_ERR_INVALID_ARG;
    }
    uint64_t helper_ns = 0;
    if (run_check_helper(c, cro_wire_l2, uuid, "L2 helper", "cro.probe_l2.helper", &o, cap, o.deadline_ms, &helper_ns, r, faults,
                         sms) == CRO_OK)
        r->helper_ns = helper_ns;
    return r->status;
}

}  // namespace cro
