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
// The bytes after the health result in a frame of `size` bytes: each ran check's frame in run order; ~0 when one is
// malformed.
uint64_t health_tail(const unsigned char* f, size_t size) {
    uint32_t ran;
    memcpy(&ran, f + offsetof(cro_health_result, ran), sizeof ran);
    size_t at = sizeof(cro_health_result);
    for (int k = 0; k < CRO_HEALTH_CHECKS; ++k) {
        if (!(ran >> k & 1u)) continue;
        const cro_wire_frame& w = cro_wire_health[k].wire->frame;
        const uint64_t tail = read_frame(w, f + at, size - at);
        if (tail == ~0ull) return ~0ull;
        at += w.result + tail;
    }
    return at - sizeof(cro_health_result);
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
    // every option of every check, in run order, each check's as its own -raw command takes them, then its cap
    std::vector<std::string> args = {"health-raw", want, std::to_string(helper_seed_base(c)), std::to_string(checks)};
    size_t max_tail = 0;
    for (int k = 0; k < CRO_HEALTH_CHECKS; ++k) {
        const cro_wire& w = *cro_wire_health[k].wire;
        append_wire_args(w, reinterpret_cast<const char*>(&o) + cro_wire_health[k].opts_at, caps.faults[k], &args);
        if (checks >> k & 1u) max_tail += cro_wire_head(&w.frame) + (size_t)caps.faults[k] * w.frame.rec;
    }
    std::string got;
    const int rc = run_probe_helper(c, want, "health helper", "cro.check_health.helper", args, deadline_ms, sizeof *r, max_tail,
                                    health_tail, &got, helper_ns);
    if (rc != CRO_OK) return r->status = rc;
    const unsigned char* f = reinterpret_cast<const unsigned char*>(got.data());
    memcpy(r, f, sizeof *r);
    // each part: its result equal to the one the health result holds, at most the asked-for records
    std::string bad;
    if (r->checks != checks || ((r->ran | r->not_run) & ~checks) || (r->ran & r->not_run)) bad = "checks outside the selection";
    size_t at = sizeof *r;
    std::vector<unsigned char> no_sms;
    for (int k = 0; k < CRO_HEALTH_CHECKS && bad.empty(); ++k) {
        const cro_wire_frame& w = cro_wire_health[k].wire->frame;
        unsigned char* held = reinterpret_cast<unsigned char*>(r) + cro_wire_health[k].result_at;
        if (!(r->ran >> k & 1u)) {
            memset(held, 0, w.result);       // blank when it did not run
            continue;
        }
        const unsigned char* part = f + at;
        uint64_t tail = 0;
        size_t n = 0;
        auto take = [&](auto* recs, auto* sms) {
            tail = read_frame(w, part, got.size() - at, nullptr, recs, sms);
            n = recs->size();
        };
        switch (k) {
            case 0: take(&rec->compute_faults, &rec->compute_sms); break;
            case 1: take(&rec->precision_faults, &rec->precision_sms); break;
            case 2: take(&rec->sram_faults, &rec->sram_sms); break;
            case 3: take(&rec->l2_faults, &rec->l2_sms); break;
            case 4: take(&rec->link_faults, &no_sms); break;
            case 5: take(&rec->scan_words, &no_sms); break;
        }
        if (memcmp(part, held, w.result) != 0) bad = "a check's result differs from the one the health result holds";
        else if (n > (size_t)caps.faults[k]) bad = "more records than asked for";
        at += w.result + tail;
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
