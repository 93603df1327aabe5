// host_link.cu — the host link probe (cro_probe_host_link): the PCIe path between the host and a composed GPU, checked
// in both directions by the copy engines and the SMs, with a pointer chase through host memory for its latency.
#include <cstdio>

#include "pcilink.hpp"
#include "probe_internal.hpp"

namespace cro {

namespace {
constexpr uint64_t kLinkDefaultBytes = 256ull << 20;
constexpr uint32_t kLinkDefaultHops = 1024;
constexpr uint32_t kLinkMaxCtas = 4096;
// Result slots: [k] the fold of word check k, then the two write roles (SM_D2H, the duplex's), then the closed forms
// of P1, P2, P3
constexpr int kLSlotWrite = CRO_LINK_WORD_CHECKS, kLSlotExpect = kLSlotWrite + 2, kLSlots = kLSlotExpect + 3;
// Per word check: which pattern (0..2 = P1..P3) its buffer must hold, and which host buffer (0 = H0, 1 = H1) it involved.
constexpr int kCheckPattern[CRO_LINK_WORD_CHECKS] = {0, 0, 1, 2, 0};
constexpr int kCheckHost[CRO_LINK_WORD_CHECKS] = {0, 0, 1, 0, 1};

// The result of a call that checked nothing: zeroes, no failed check, unknown NUMA nodes, and the L it got to (0 before
// it knew it).
void blank_result(cro_link_result* r, std::vector<cro_link_fault>* faults, uint64_t bytes) {
    memset(r, 0, sizeof *r);
    r->bytes = bytes;
    r->first_fail = CRO_LINK_NO_FAIL;
    r->dev_numa = r->host_numa[0] = r->host_numa[1] = r->host_numa[2] = -1;
    r->path.numa_node = -1;
    faults->clear();
}

// Pinned, mapped host memory of `bytes` on `node` (pcilink::MapOnNode, then cudaHostRegister); nullptr on failure.
unsigned char* map_pinned(size_t bytes, int node) {
    void* p = pcilink::MapOnNode(bytes, node);
    if (!p) return nullptr;
    if (cudaHostRegister(p, bytes, cudaHostRegisterMapped | cudaHostRegisterPortable) != cudaSuccess) {
        cudaGetLastError();
        pcilink::Unmap(p, bytes);
        return nullptr;
    }
    return static_cast<unsigned char*>(p);
}
void unmap_pinned(unsigned char*& p, size_t bytes) {
    if (!p) return;
    cudaHostUnregister(p);
    pcilink::Unmap(p, bytes);
    p = nullptr;
}

// Why the options are refused for a sweep region of S bytes ("" when they pass): both forms' argument checks.
std::string link_opts_error(const cro_link_opts& o, uint64_t S) {
    const uint64_t L = o.bytes ? o.bytes : std::min(kLinkDefaultBytes, S);
    const uint32_t hops = o.hops ? o.hops : kLinkDefaultHops;
    if (L < 16 || L % 16 || L > S || hops > (1u << 24) || o.ctas > kLinkMaxCtas ||
        (o.test_inject_mask && (o.test_inject_check < 0 || o.test_inject_check >= CRO_LINK_WORD_CHECKS ||
                                o.test_inject_word >= L / 8)))
        return "host link probe: L = " + std::to_string(L) + " must be a multiple of 16 in [16, " + std::to_string(S) +
               "], hops at most 2^24, ctas at most " + std::to_string(kLinkMaxCtas) +
               ", and an injection must name a word check (0..4) and a word below L / 8";
    return "";
}

// Word check ck's counts and records once it ran (hv, the host mirror after the fetch), each record with word
// word_index of the host buffer the check involved (hb, n = L / 8 words, read now), appended to *faults by word index.
void take_link_check(const MismatchView& hv, int ck, const volatile uint64_t* hb, uint64_t n, cro_link_result* r,
                     std::vector<cro_link_fault>* faults) {
    cro_link_check& C = r->check[ck];
    C.mismatches = hv.ctr[ck].mismatches;
    C.recorded = std::min<uint64_t>(hv.ctr[ck].claims, kLocateRecords);
    std::vector<cro_link_fault> f;
    for (uint64_t j = 0; j < C.recorded; ++j) {
        const LocateRecord& R = hv.rec[(size_t)ck * kLocateRecords + j];
        f.push_back(cro_link_fault{(uint32_t)ck, 0, R.word, R.expected, R.actual, R.word < n ? hb[R.word] : 0});
    }
    std::sort(f.begin(), f.end(), [](const cro_link_fault& a, const cro_link_fault& b) { return a.word_index < b.word_index; });
    faults->insert(faults->end(), f.begin(), f.end());
}

// The verdict once every check was taken: each word check's fold against the closed form of its pattern (both over
// n = L / 8 words, the pattern seeds r->seed), then the chase's end (hco: the chase output words) against the host walk
// of hops steps through the (minor, minor) permutation.  first_fail is the lowest check that failed.
void classify_link(const MismatchView& hv, const unsigned long long* hco, int minor, uint32_t hops, cro_link_result* r) {
    const uint64_t n = r->bytes / 8;
    for (int ck = 0; ck < CRO_LINK_WORD_CHECKS; ++ck) {
        cro_link_check& C = r->check[ck];
        const SweepOut& s = hv.slots[ck];
        const SweepOut& cf = hv.slots[kLSlotExpect + kCheckPattern[ck]];
        C.words = n;
        C.seed = r->seed[kCheckPattern[ck]];
        C.fold_xor = s.x;
        C.fold_sum = s.s;
        C.fold_wsum = s.w;
        C.expect_xor = cf.x;
        C.expect_sum = cf.s;
        C.expect_wsum = cf.w;
        const bool bad = C.mismatches != 0 || s.n_words != n || cf.n_words != n || s.x != cf.x || s.s != cf.s || s.w != cf.w;
        if (bad && r->first_fail == CRO_LINK_NO_FAIL) r->first_fail = (uint32_t)ck;
    }
    std::vector<uint32_t> perm;
    chase_permutation(minor, minor, &perm);
    uint32_t at = 0;
    for (uint32_t h = 0; h < hops; ++h) at = perm[at];
    r->chase_expect = at;
    r->chase_end = (uint32_t)hco[0];
    r->chase_ns = hco[0] == kChaseArmed ? 0 : hco[1];
    if (hco[0] != at && r->first_fail == CRO_LINK_NO_FAIL) r->first_fail = CRO_LINK_CHECK_CHASE;
}

int link_status(const cro_link_result& r) { return r.first_fail == CRO_LINK_NO_FAIL ? CRO_OK : CRO_ERR_CHECKSUM; }
}  // namespace

int selftest_link_classify(uint64_t bytes, const uint64_t* seeds, uint32_t minor, uint32_t hops, const cro_locate_counters* ctr,
                           const cro_locate_record* records, const uint64_t* host, const cro_sweep_slot* slots,
                           const uint64_t* chase_out, cro_link_result* r, std::vector<cro_link_fault>* faults) {
    blank_result(r, faults, bytes);
    const uint64_t n = bytes / 8;
    for (int j = 0; j < 3; ++j) r->seed[j] = seeds[j];
    r->chase_hops = hops;
    r->chase_minor = minor;
    // the device's layout: kLocateRecords records per check, then the result slots
    std::vector<LocateCounters> c(CRO_LINK_WORD_CHECKS);
    std::vector<LocateRecord> rec((size_t)CRO_LINK_WORD_CHECKS * kLocateRecords);
    std::vector<SweepOut> s(kLSlots);
    memcpy(c.data(), ctr, sizeof(LocateCounters) * CRO_LINK_WORD_CHECKS);
    for (int ck = 0; ck < CRO_LINK_WORD_CHECKS; ++ck) {
        const uint64_t k = std::min<uint64_t>(ctr[ck].claims, kLocateRecords);
        if (k) memcpy(&rec[(size_t)ck * kLocateRecords], records, k * sizeof *records);
        records += k;
    }
    memcpy(s.data(), slots, kLSlots * sizeof *slots);
    const MismatchView hv{c.data(), nullptr, s.data(), rec.data(), nullptr, 0};
    for (int ck = 0; ck < CRO_LINK_WORD_CHECKS; ++ck) take_link_check(hv, ck, host + ck * n, n, r, faults);
    const unsigned long long co[2] = {chase_out[0], chase_out[1]};
    classify_link(hv, co, (int)minor, hops, r);
    return r->status = link_status(*r);
}

LinkState::~LinkState() {
    for (unsigned char*& h : host) unmap_pinned(h, cap);
    unmap_pinned(chase, (size_t)kChaseSlots * 128);
    for (cudaEvent_t e : ev)
        if (e) cudaEventDestroy(e);
}

int ctx_probe_host_link(cro_ctx* c, int idx, const cro_link_opts& o, cro_link_result* r, std::vector<cro_link_fault>* faults) {
    blank_result(r, faults, 0);
    Device* d = dev_at(c, idx);
    if (!d) return r->status = unknown_device(c, idx, "a GPU probed through the helper process has no resident region to probe its host link from");
    DeviceGuard g = enter_device(c, idx);
    if (g.rc) return r->status = g.rc;
    int rc = [&]() -> int {
        int e = ensure_region(c, d);
        if (e) return e;
        const uint64_t S = d->sweep_bytes;
        const uint64_t L = o.bytes ? o.bytes : std::min(kLinkDefaultBytes, S);
        const uint32_t hops = o.hops ? o.hops : kLinkDefaultHops;
        const std::string why = link_opts_error(o, S);
        if (!why.empty()) {
            c->set_error(why);
            return CRO_ERR_INVALID_ARG;
        }
        const int grid = o.ctas ? (int)o.ctas : d->plan.link_grid;
        const uint64_t n = L / 8;
        cro_pci_path before_path;
        // the PCI location as the CUDA driver reports it: the identity sources may not know it (NVML answers "[N/A]"
        // on some virtualised hosts)
        char bus_id[32] = {};
        if (cudaDeviceGetPCIBusId(bus_id, sizeof bus_id, d->ordinal) != cudaSuccess) {
            cudaGetLastError();
            snprintf(bus_id, sizeof bus_id, "%s", d->info.pci_bus_id);
        }
        const int node = pcilink::ReadPath(c->sys_root, bus_id, &before_path) == CRO_OK ? before_path.numa_node : -1;

        // first call (or a larger L): host buffers, chase table, device-side buffers, events
        if (!d->link) d->link.reset(new LinkState);
        LinkState& ls = *d->link;
        if (ls.cap < L) {
            for (unsigned char*& h : ls.host) unmap_pinned(h, ls.cap);
            ls.cap = 0;
            for (unsigned char*& h : ls.host)
                if (!(h = map_pinned(L, node))) {
                    for (unsigned char*& q : ls.host) unmap_pinned(q, L);
                    c->set_error("host link probe: could not allocate and pin " + std::to_string(L) + " bytes of host memory");
                    return CRO_ERR_OOM;
                }
            ls.cap = L;
        }
        if (!ls.chase) {
            if (!(ls.chase = map_pinned((size_t)kChaseSlots * 128, node))) {
                c->set_error("host link probe: could not allocate and pin the chase table");
                return CRO_ERR_OOM;
            }
            std::vector<uint32_t> perm;
            chase_permutation(d->info.device_minor, d->info.device_minor, &perm);
            unsigned long long* t = reinterpret_cast<unsigned long long*>(ls.chase);
            for (uint32_t i = 0; i < kChaseSlots; ++i) t[(size_t)i * 16] = perm[i];
        }
        MismatchBuffer& mb = ls.buf;
        const int max_grid = std::max({(int)kLinkMaxCtas, d->plan.locate.grid, d->plan.expect.grid, 1});
        if ((e = mb.ensure(c, CRO_LINK_WORD_CHECKS, S, kLSlots, kChaseOutWords * sizeof(unsigned long long), max_grid, 2))) return e;
        for (cudaEvent_t& x : ls.ev)
            if (!x) CU_TRY(c, cudaEventCreate(&x));
        void* dH[2];
        for (int b = 0; b < 2; ++b) CU_TRY(c, cudaHostGetDevicePointer(&dH[b], ls.host[b], 0));
        void* dchase = nullptr;
        CU_TRY(c, cudaHostGetDevicePointer(&dchase, ls.chase, 0));
        const MismatchView dv = mb.dev(), hv = mb.host();
        unsigned long long* chase_out = reinterpret_cast<unsigned long long*>(dv.tail);
        cudaStream_t st = d->stream;
        unsigned char* A = d->region;
        unsigned char* B = d->region + S;

        const uint64_t k = d->link_calls++;
        uint64_t P[3];
        for (int j = 0; j < 3; ++j) P[j] = space_seed(d, kSeedLink, k, (uint64_t)j);
        r->bytes = L;
        r->call = k;
        for (int j = 0; j < 3; ++j) r->seed[j] = P[j];
        r->chase_hops = hops;
        r->chase_minor = (uint32_t)d->info.device_minor;
        const std::string uuid = d->info.gpu_uuid;
        unsigned long long rp = 0;
        r->no_nvml = 1;
        if (!(c->opts.flags & CRO_F_NO_NVML) && identity::NvmlPcieReplays(uuid, &rp)) {
            r->no_nvml = 0;
            r->replays_before = rp;
        }

        const bool inj = o.test_inject_mask != 0;
        auto inject_host = [&](int check) -> int {      // the CPU flips the pinned word once the leg is done
            if (!inj || o.test_inject_check != check) return CRO_OK;
            const int rc2 = wait_stream(c, d);
            if (rc2) return rc2;
            reinterpret_cast<volatile uint64_t*>(ls.host[kCheckHost[check]])[o.test_inject_word] ^= o.test_inject_mask;
            return CRO_OK;
        };
        auto inject_b = [&](int check) -> int {
            if (!inj || o.test_inject_check != check) return CRO_OK;
            CU_TRY(c, launch_xor_words(B, o.test_inject_word, 1, o.test_inject_mask, st));
            c->launches++;
            return CRO_OK;
        };
        // Records of the given checks, with the host buffer's word read now: the callers run this once the checks are
        // done and before a later leg rewrites that buffer.
        auto harvest = [&](std::initializer_list<int> checks) -> int {
            int rc2 = mb.fetch(c, st);
            if (rc2 || (rc2 = wait_stream(c, d))) return rc2;
            for (int ck : checks)
                take_link_check(hv, ck, reinterpret_cast<const volatile uint64_t*>(ls.host[kCheckHost[ck]]), n, r, faults);
            return CRO_OK;
        };
        auto role = [&](void* buf, int pat, int scratch, SweepOut* out) {
            return LinkRole{buf, L, P[pat], mb.scratch[scratch], out, (unsigned)kLinkWarps};
        };
        const LinkRole off{nullptr, 0, 0, SweepScratch{}, nullptr, 0};
        const SweepScratch& sc0 = mb.scratch[0];

        if ((e = mb.zero(c, st))) return e;
        // A[0, L) <- P1, and the closed forms of P1..P3 over L
        CU_TRY(c, launch_fill(d->plan, A, L, Params{ProbeParams{P[0], k}, nullptr}, sc0, nullptr, st));
        d->half_known[0] = d->half_known[1] = false;      // both halves now hold the link probe's patterns
        d->filled = false;
        for (int j = 0; j < 3; ++j)
            CU_TRY(c, launch_expected(d->plan, L, Params{ProbeParams{P[j], k}, nullptr}, sc0, &dv.slots[kLSlotExpect + j], st));
        c->launches += 4;
        // CE d2h, then the SMs read H0 (check 0)
        CU_TRY(c, cudaEventRecord(ls.ev[0], st));
        CU_TRY(c, cudaMemcpyAsync(ls.host[0], A, L, cudaMemcpyDeviceToHost, st));
        CU_TRY(c, cudaEventRecord(ls.ev[1], st));
        if ((e = inject_host(CRO_LINK_CHECK_D2H_COPY))) return e;
        CU_TRY(c, cudaEventRecord(ls.ev[2], st));
        CU_TRY(c, launch_link_stream(role(dH[0], 0, 0, &dv.slots[0]), off, dv.check(0), grid, k, st));
        CU_TRY(c, cudaEventRecord(ls.ev[3], st));
        // CE h2d H0 -> B, checked in HBM (check 1)
        CU_TRY(c, cudaEventRecord(ls.ev[4], st));
        CU_TRY(c, cudaMemcpyAsync(B, ls.host[0], L, cudaMemcpyHostToDevice, st));
        CU_TRY(c, cudaEventRecord(ls.ev[5], st));
        if ((e = inject_b(CRO_LINK_CHECK_H2D_COPY))) return e;
        CU_TRY(c, launch_locate(d->plan, B, L, 0, P[0], 0, dv.check(1), sc0, &dv.slots[1], st));
        c->launches += 2;
        if ((e = harvest({0, 1}))) return e;              // before the duplex launch rewrites H0
        // SMs write P2 into H1
        CU_TRY(c, cudaEventRecord(ls.ev[6], st));
        CU_TRY(c, launch_link_stream(off, role(dH[1], 1, 1, &dv.slots[kLSlotWrite]), dv.check(2), grid, k, st));
        CU_TRY(c, cudaEventRecord(ls.ev[7], st));
        if ((e = inject_host(CRO_LINK_CHECK_SM_WRITE))) return e;
        // SM duplex: read H1 against P2 (check 2) and write P3 into H0, one launch
        CU_TRY(c, cudaEventRecord(ls.ev[8], st));
        CU_TRY(c, launch_link_stream(role(dH[1], 1, 0, &dv.slots[2]), role(dH[0], 2, 1, &dv.slots[kLSlotWrite + 1]), dv.check(2),
                                     grid, k, st));
        CU_TRY(c, cudaEventRecord(ls.ev[9], st));
        c->launches += 2;
        if ((e = harvest({2}))) return e;                 // before the CE duplex rewrites H1
        // CE duplex: H0 -> B on the device stream and A -> H1 on aux, at once
        CU_TRY(c, cudaEventRecord(ls.ev[10], st));
        CU_TRY(c, cudaStreamWaitEvent(d->aux, ls.ev[10], 0));
        CU_TRY(c, cudaMemcpyAsync(B, ls.host[0], L, cudaMemcpyHostToDevice, st));
        CU_TRY(c, cudaEventRecord(ls.ev[11], st));
        CU_TRY(c, cudaEventRecord(ls.ev[12], d->aux));
        CU_TRY(c, cudaMemcpyAsync(ls.host[1], A, L, cudaMemcpyDeviceToHost, d->aux));
        CU_TRY(c, cudaEventRecord(ls.ev[13], d->aux));
        CU_TRY(c, cudaStreamWaitEvent(st, ls.ev[13], 0));
        // an idle GPU trains its link down: sample the path while both copies are in flight
        if (pcilink::ReadPath(c->sys_root, bus_id, &r->path) == CRO_OK) {
            r->dev_numa = r->path.numa_node;
            r->degraded = pcilink::Degraded(r->path);
        }
        if ((e = wait_stream(c, d))) return e;
        if ((e = inject_b(CRO_LINK_CHECK_DUPLEX_WRITE))) return e;
        if ((e = inject_host(CRO_LINK_CHECK_DUPLEX_D2H_COPY))) return e;
        // check 3: B against P3; check 4: the SMs read H1 against P1 (verification only, untimed)
        CU_TRY(c, launch_locate(d->plan, B, L, 0, P[2], 0, dv.check(3), sc0, &dv.slots[3], st));
        CU_TRY(c, launch_link_stream(role(dH[1], 0, 0, &dv.slots[4]), off, dv.check(4), grid, k, st));
        // latency: one warp chases the self pair's permutation through host memory (check 5)
        ChaseArgs ca{};
        ca.n = 1;
        ca.hops = hops;
        ca.table[0] = static_cast<const unsigned long long*>(dchase);
        CU_TRY(c, arm_chase_out(chase_out, st));
        CU_TRY(c, launch_chase(ca, chase_out, st));
        c->launches += 3;
        if ((e = harvest({3, 4}))) return e;
        if (!r->no_nvml && identity::NvmlPcieReplays(uuid, &rp)) r->replays_after = rp;
        else if (!r->no_nvml) { r->no_nvml = 1; r->replays_before = 0; }

        auto span = [&](int a, int b) -> uint64_t {
            float ms = 0;
            return cudaEventElapsedTime(&ms, ls.ev[a], ls.ev[b]) == cudaSuccess ? ms_to_ns(ms) : 0;
        };
        auto window = [](const SweepOut& s) -> uint64_t { return s.t1 > s.t0 ? s.t1 - s.t0 : 0; };
        const int ev_of[CRO_LINK_LEGS][2] = {{0, 1}, {2, 3}, {4, 5}, {6, 7}, {8, 9}, {8, 9}, {10, 11}, {12, 13}};
        const int timer_of[CRO_LINK_LEGS] = {-1, 0, -1, kLSlotWrite, 2, kLSlotWrite + 1, -1, -1};   // result slot, -1: none
        for (int lg = 0; lg < CRO_LINK_LEGS; ++lg) {
            r->leg[lg].bytes = L;
            r->leg[lg].ns = span(ev_of[lg][0], ev_of[lg][1]);
            r->leg[lg].timer_ns = timer_of[lg] >= 0 ? window(hv.slots[timer_of[lg]]) : 0;
        }
        r->ce_duplex_span_ns = std::max(span(10, 11), span(10, 13));
        classify_link(hv, reinterpret_cast<const unsigned long long*>(hv.tail), d->info.device_minor, hops, r);
        for (int b = 0; b < 2; ++b) r->host_numa[b] = pcilink::NodeOf(ls.host[b]);
        r->host_numa[2] = pcilink::NodeOf(ls.chase);
        return CRO_OK;
    }();
    if (rc) {
        blank_result(r, faults, r->bytes);
        return r->status = rc;
    }
    return r->status = link_status(*r);
}

// The helper's sweep region is L, or the default L when none is given: refuse here what it would refuse there.
std::string link_helper_opts_error(const cro_link_opts& o) { return link_opts_error(o, o.bytes ? o.bytes : kLinkDefaultBytes); }

int ctx_probe_host_link_uuid(cro_ctx* c, const char* uuid, const cro_link_opts& o, int deadline_ms, cro_link_result* r,
                             std::vector<cro_link_fault>* faults, int cap, uint64_t* helper_ns) {
    blank_result(r, faults, 0);
    *helper_ns = 0;
    if (!uuid) return r->status = CRO_ERR_INVALID_ARG;
    const std::string why = link_helper_opts_error(o);
    if (!why.empty()) {
        set_call_error(c, why);
        return r->status = CRO_ERR_INVALID_ARG;
    }
    run_check_helper(c, cro_wire_link, uuid, "link helper", "cro.probe_host_link.helper", &o, cap, deadline_ms, helper_ns, r, faults);
    return r->status;
}

}  // namespace cro
