// health.cpp — the health check (cro_check_health / cro_check_health_uuid): a composed GPU's compute, precision, SRAM,
// L2, host link and whole-HBM checks in one call, in that order, each through its own in-process call.
#include <type_traits>

#include "c_api_util.hpp"
#include "probe_internal.hpp"

namespace cro {

static_assert(offsetof(cro_health_result, status) == 0 && std::is_same<decltype(cro_health_result::status), int32_t>::value,
              "run_probe_helper reads the health result's status from the first four bytes of its frame");

int health_step(uint32_t checks, const int32_t* status, int n, cro_health_result* r) {
    r->checks = checks;
    r->ran = r->failed = r->errored = r->not_run = 0;
    memset(r->check_status, 0, sizeof r->check_status);
    int used = 0, next = CRO_HEALTH_CHECKS;
    int32_t first_bad = CRO_OK;
    bool stopped = false;
    for (int c = 0; c < CRO_HEALTH_CHECKS; ++c) {
        const uint32_t bit = 1u << c;
        if (!(checks & bit)) continue;
        if (stopped) {          // a sticky CUDA error fails every later launch in the process: report, do not run
            r->not_run |= bit;
            continue;
        }
        if (used == n) {
            next = c;
            break;
        }
        const int32_t s = status[used++];
        r->ran |= bit;
        r->check_status[c] = s;
        if (s == CRO_ERR_CHECKSUM) r->failed |= bit;
        else if (s != CRO_OK) r->errored |= bit;
        if (s != CRO_OK && s != CRO_ERR_CHECKSUM && first_bad == CRO_OK) first_bad = s;
        stopped = s == CRO_ERR_CUDA;
    }
    r->status = r->failed ? CRO_ERR_CHECKSUM : first_bad;      // corruption found is never transient
    return used < n ? -1 : next;
}

std::string health_opts_error(const cro_health_opts& o) {
    const uint32_t checks = o.checks ? o.checks : CRO_HEALTH_ALL;
    if ((checks & ~CRO_HEALTH_ALL) || o.reserved0)
        return "health check: checks must be CRO_HEALTH_ALL bits and reserved0 zero";
    if (o.sram.deadline_ms || o.l2.deadline_ms || o.scan.deadline_ms)
        return "health check: the call has one deadline; sram, l2 and scan deadline_ms must be 0";
    std::string why;
    L2Settings l2;
    if ((checks & CRO_HEALTH_COMPUTE) && !(why = compute_opts_error(o.compute)).empty()) return why;
    if ((checks & CRO_HEALTH_PRECISION) && !(why = precision_opts_error(o.precision)).empty()) return why;
    if ((checks & CRO_HEALTH_SRAM) && !(why = sram_opts_error(o.sram)).empty()) return why;
    if ((checks & CRO_HEALTH_L2) && !l2_check_args(o.l2, 0, true, &l2, &why)) return why;
    if ((checks & CRO_HEALTH_LINK) && !(why = link_helper_opts_error(o.link)).empty()) return why;
    if ((checks & CRO_HEALTH_SCAN) && !(why = scan_opts_error(o.scan)).empty()) return why;
    return "";
}

int ctx_check_health(cro_ctx* c, int idx, const cro_health_opts& o, cro_health_result* r, HealthRecords* rec) {
    *r = cro_health_result{};
    *rec = HealthRecords{};
    const uint32_t checks = o.checks ? o.checks : CRO_HEALTH_ALL;
    r->seed_base = c->opts.seed_base;
    std::vector<int32_t> st;
    for (int next; (next = health_step(checks, st.data(), (int)st.size(), r)) < CRO_HEALTH_CHECKS;) {
        const uint64_t t0 = now_ns();
        int rc = CRO_ERR_INTERNAL;
        switch (next) {
            case 0: rc = ctx_probe_compute(c, idx, o.compute, &r->compute, &rec->compute_sms, &rec->compute_faults); break;
            case 1: rc = ctx_probe_precision(c, idx, o.precision, &r->precision, &rec->precision_sms, &rec->precision_faults); break;
            case 2: rc = ctx_probe_sram(c, idx, o.sram, &r->sram, &rec->sram_sms, &rec->sram_faults); break;
            case 3: rc = ctx_probe_l2(c, idx, o.l2, &r->l2, &rec->l2_sms, &rec->l2_faults); break;
            case 4: rc = ctx_probe_host_link(c, idx, o.link, &r->link, &rec->link_faults); break;
            case 5: rc = ctx_scan_hbm(c, idx, o.scan, &r->scan, &rec->scan_words); break;
        }
        r->check_ns[next] = now_ns() - t0;
        st.push_back(rc);
    }
    using capi::min_covered;
    const bool short_of[4] = {
        min_covered(r->compute.legs, r->compute.leg, CRO_COMPUTE_LEGS) < r->compute.sm_count,
        min_covered(r->precision.legs, r->precision.leg, CRO_PRECISION_LEGS) < r->precision.sm_count,
        min_covered(r->sram.legs, r->sram.leg, CRO_SRAM_LEGS) < r->sram.sm_count,
        r->l2.sms_covered < r->l2.sm_count};
    for (int k = 0; k < 4; ++k)
        if ((r->ran >> k & 1u) && short_of[k]) r->incomplete |= 1u << k;
    return r->status;
}

namespace {
// One check's part of the health-raw frame, laid out as its own -raw command writes it: the result, `counts` uint64_t
// counts, the per-SM block, then the records.  n_sms and n read a part's counts (n_sms 0 without a per-SM list).
struct Part {
    size_t result, counts, sms, rec, max_sms;
    void (*read)(const unsigned char* part, uint64_t* n_sms, uint64_t* n);
    size_t head() const { return result + counts * sizeof(uint64_t) + sms; }
};
template <class Result, class Sm, class Fault, size_t MAX_SMS>
Part sm_part() {
    using F = SmFrame<Result, Sm, Fault, MAX_SMS>;
    return {sizeof(Result), 2, MAX_SMS * sizeof(Sm), sizeof(Fault), MAX_SMS, [](const unsigned char* p, uint64_t* n_sms, uint64_t* n) {
                *n_sms = F::count(p, 0);
                *n = F::count(p, 1);
            }};
}
const Part kParts[CRO_HEALTH_CHECKS] = {
    sm_part<cro_compute_result, cro_compute_sm, cro_compute_fault, CRO_COMPUTE_MAX_SMS>(),
    sm_part<cro_precision_result, cro_precision_sm, cro_precision_fault, CRO_PRECISION_MAX_SMS>(),
    {sizeof(cro_sram_result), 0, CRO_SRAM_MAX_SMS * sizeof(cro_sram_sm), sizeof(cro_sram_fault), CRO_SRAM_MAX_SMS,
     [](const unsigned char* p, uint64_t* n_sms, uint64_t* n) {
         const cro_sram_result* r = reinterpret_cast<const cro_sram_result*>(p);
         *n_sms = r->sms_listed;
         *n = r->recorded;
     }},
    sm_part<cro_l2_result, cro_l2_sm, cro_l2_fault, CRO_L2_MAX_SMS>(),
    {sizeof(cro_link_result), 1, 0, sizeof(cro_link_fault), 0,
     [](const unsigned char* p, uint64_t* n_sms, uint64_t* n) {
         *n_sms = 0;
         memcpy(n, p + sizeof(cro_link_result), sizeof *n);
     }},
    {sizeof(cro_scan_report), 0, 0, sizeof(cro_fault_word), 0, [](const unsigned char* p, uint64_t* n_sms, uint64_t* n) {
         *n_sms = 0;
         *n = reinterpret_cast<const cro_scan_report*>(p)->recorded;
     }},
};

// The bytes after the health result in a frame of `size` bytes: each ran check's part in run order; ~0 when a part is
// cut short or lists more per-SM entries than its block holds.
uint64_t health_tail(const unsigned char* f, size_t size) {
    uint32_t ran;
    memcpy(&ran, f + offsetof(cro_health_result, ran), sizeof ran);
    size_t at = sizeof(cro_health_result);
    for (int c = 0; c < CRO_HEALTH_CHECKS; ++c) {
        if (!(ran >> c & 1u)) continue;
        const Part& p = kParts[c];
        if (size - at < p.head()) return ~0ull;
        uint64_t n_sms, n;
        p.read(f + at, &n_sms, &n);
        if (n_sms > p.max_sms || n > (size - at - p.head()) / p.rec) return ~0ull;
        at += p.head() + n * p.rec;
    }
    return at - sizeof(cro_health_result);
}

template <class T>
void take(const unsigned char* from, uint64_t n, std::vector<T>* to) {
    const T* t = reinterpret_cast<const T*>(from);
    to->assign(t, t + n);
}
}  // namespace

int ctx_check_health_uuid(cro_ctx* c, const char* uuid, const cro_health_opts& o, int deadline_ms, const HealthCaps& caps,
                          cro_health_result* r, HealthRecords* rec, uint64_t* helper_ns) {
    *r = cro_health_result{};
    *rec = HealthRecords{};
    *helper_ns = 0;
    const uint32_t checks = o.checks ? o.checks : CRO_HEALTH_ALL;
    r->checks = checks;
    if (!uuid) return r->status = CRO_ERR_INVALID_ARG;
    const std::string why = health_opts_error(o);
    if (!why.empty()) {
        set_call_error(c, why);
        return r->status = CRO_ERR_INVALID_ARG;
    }
    const std::string want = uuid;
    using std::to_string;
    auto u = [](uint64_t v) { return to_string(v); };
    auto i = [](int64_t v) { return to_string(v); };
    const cro_compute_opts& co = o.compute;
    const cro_precision_opts& po = o.precision;
    const cro_sram_opts& so = o.sram;
    const cro_l2_opts& lo = o.l2;
    const cro_link_opts& ko = o.link;
    const cro_scan_opts& xo = o.scan;
    // every option of every check, in run order, each check's as its own -raw command takes them, then its cap
    const std::vector<std::string> args = {
        "health-raw", want, u(helper_seed_base(c)), u(checks),
        u(co.iterations), u(co.alu_iterations), u(co.legs), u(co.max_rounds), i(co.test_inject_leg), i(co.test_inject_sm),
        u(co.test_inject_iteration), i(co.test_inject_row), i(co.test_inject_col), u(co.test_inject_mask), i(caps.faults[0]),
        u(po.iterations), u(po.alu_iterations), u(po.legs), u(po.max_rounds), i(po.test_inject_leg), i(po.test_inject_sm),
        u(po.test_inject_iteration), i(po.test_inject_row), i(po.test_inject_col), u(po.test_inject_mask), i(caps.faults[1]),
        u(so.legs), u(so.iterations), u(so.cluster), u(so.max_rounds), i(so.test_inject_leg), i(so.test_inject_sm),
        u(so.test_inject_element), u(so.test_inject_iteration), i(so.test_inject_word), u(so.test_inject_mask), i(caps.faults[2]),
        u(lo.bytes), u(lo.iterations), u(lo.a1_counters), u(lo.a2_counters), i(lo.test_inject_leg), i(lo.test_inject_sm),
        i(lo.test_inject_element), u(lo.test_inject_iteration), i(lo.test_inject_word), u(lo.test_inject_mask), i(caps.faults[3]),
        u(ko.bytes), u(ko.hops), u(ko.ctas), i(ko.test_inject_check), u(ko.test_inject_word), u(ko.test_inject_mask),
        i(caps.faults[4]),
        u(xo.max_bytes), u(xo.reserve_bytes), u(xo.seed), u(xo.test_chunk_bytes), u(xo.test_force_first), u(xo.test_force_count),
        u(xo.test_force_and), u(xo.test_force_or), i(caps.faults[5])};
    size_t max_tail = 0;
    for (int k = 0; k < CRO_HEALTH_CHECKS; ++k)
        if (checks >> k & 1u) max_tail += kParts[k].head() + (size_t)caps.faults[k] * kParts[k].rec;
    std::string got;
    const int rc = run_probe_helper(c, want, "health helper", "cro.check_health.helper", args, deadline_ms, sizeof *r, 1, max_tail,
                                    health_tail, &got, helper_ns);
    if (rc != CRO_OK) return r->status = rc;
    const unsigned char* f = reinterpret_cast<const unsigned char*>(got.data());
    memcpy(r, f, sizeof *r);
    // each part: its result equal to the one the health result holds, at most the asked-for records
    std::string bad;
    if (r->checks != checks || ((r->ran | r->not_run) & ~checks) || (r->ran & r->not_run)) bad = "checks outside the selection";
    size_t at = sizeof *r;
    void* held[CRO_HEALTH_CHECKS] = {&r->compute, &r->precision, &r->sram, &r->l2, &r->link, &r->scan};
    for (int k = 0; k < CRO_HEALTH_CHECKS && bad.empty(); ++k) {
        if (!(r->ran >> k & 1u)) {
            memset(held[k], 0, kParts[k].result);       // blank when it did not run
            continue;
        }
        const Part& p = kParts[k];
        const unsigned char* part = f + at;
        uint64_t n_sms, n;
        p.read(part, &n_sms, &n);
        if (memcmp(part, held[k], p.result) != 0) bad = "a check's result differs from the one the health result holds";
        else if (n > (uint64_t)caps.faults[k]) bad = "more records than asked for";
        const unsigned char* sms = part + p.head() - p.sms;
        const unsigned char* recs = part + p.head();
        switch (k) {
            case 0: take(sms, n_sms, &rec->compute_sms); take(recs, n, &rec->compute_faults); break;
            case 1: take(sms, n_sms, &rec->precision_sms); take(recs, n, &rec->precision_faults); break;
            case 2: take(sms, n_sms, &rec->sram_sms); take(recs, n, &rec->sram_faults); break;
            case 3: take(sms, n_sms, &rec->l2_sms); take(recs, n, &rec->l2_faults); break;
            case 4: take(recs, n, &rec->link_faults); break;
            case 5: take(recs, n, &rec->scan_words); break;
        }
        at += p.head() + n * p.rec;
    }
    if (!bad.empty()) {
        set_call_error(c, "health helper for " + want + " failed (" + bad + ")");
        *r = cro_health_result{};
        *rec = HealthRecords{};
        r->checks = checks;
        return r->status = CRO_ERR_EXEC;
    }
    r->helper_ns = *helper_ns;
    return r->status;
}

}  // namespace cro
