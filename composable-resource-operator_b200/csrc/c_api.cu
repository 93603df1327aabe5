// c_api.cu — extern "C" surface of libcroprobe (include/croprobe.h).
#include <cstdio>
#include <cstring>
#include <map>
#include <set>
#include <string>

#include "../../include/croprobe.h"
#include "c_api_util.hpp"
#include "gojson.hpp"
#include "identity.hpp"
#include "probe.hpp"
#include "reconcile.hpp"
#include "cluster.hpp"
#include "detach.hpp"
#include "fabric.hpp"
#include "provider.hpp"
#include "nodes.hpp"
#include "gpus.hpp"
#include "env.hpp"
#include "inventory.hpp"
#include "gotypes.hpp"
#include "pcilink.hpp"
#include "compute.hpp"
#include <memory>
#include <new>
#include <stdexcept>

using namespace cro;

static_assert(sizeof(cro_probe_result) == 512, "cro_probe_result is the 512-byte all-gather payload");
static_assert(offsetof(cro_probe_result, gpu_uuid) == 16, "layout");
static_assert(offsetof(cro_probe_result, pci_bus_id) == 64, "layout");
static_assert(offsetof(cro_probe_result, checksum_xor) == 112, "layout");
static_assert(offsetof(cro_probe_result, p2p_read_ns) == 184, "layout");
static_assert(offsetof(cro_probe_result, p2p_access) == 344, "layout");
static_assert(offsetof(cro_probe_result, p2p_bytes) == 352, "layout");
static_assert(offsetof(cro_probe_result, p2p_write_ns) == 424, "layout");
static_assert(offsetof(cro_probe_result, nonce) == 488, "layout");
static_assert(offsetof(cro_probe_result, t_start_ns) == 504, "layout");
static_assert(sizeof(cro_fullbox_time) == 64 && offsetof(cro_fullbox_time, gather) == 56, "cro_fullbox_time layout");
static_assert(sizeof(cro_sweep_result) == 56, "layout");
static_assert(sizeof(cro_locate_opts) == 40 && sizeof(cro_fault_word) == 32, "locator layout");
static_assert(sizeof(cro_locate_pass) == 120 && offsetof(cro_locate_pass, fold_xor) == 72, "locator layout");
static_assert(sizeof(cro_fault_report) == 928 && offsetof(cro_fault_report, bit_flips) == 56 &&
                  offsetof(cro_fault_report, pass) == 568, "locator layout");
static_assert(sizeof(cro_pci_hop) == 32 && sizeof(cro_pci_path) == 272 && offsetof(cro_pci_path, hop) == 16, "link layout");
static_assert(sizeof(cro_link_opts) == 40 && sizeof(cro_link_fault) == 40 && sizeof(cro_link_leg) == 24 &&
                  sizeof(cro_link_check) == 80, "link layout");
static_assert(sizeof(cro_link_result) == 984 && offsetof(cro_link_result, leg) == 48 &&
                  offsetof(cro_link_result, ce_duplex_span_ns) == 240 && offsetof(cro_link_result, check) == 248 &&
                  offsetof(cro_link_result, chase_hops) == 648 && offsetof(cro_link_result, chase_ns) == 664 &&
                  offsetof(cro_link_result, dev_numa) == 672 && offsetof(cro_link_result, no_nvml) == 688 &&
                  offsetof(cro_link_result, replays_before) == 696 && offsetof(cro_link_result, path) == 712,
              "link layout");
static_assert(sizeof(cro_compute_opts) == 40 && sizeof(cro_compute_leg) == 104 && sizeof(cro_compute_sm_leg) == 40 &&
                  sizeof(cro_compute_sm) == 208 && sizeof(cro_compute_fault) == 24, "compute layout");
static_assert(sizeof(cro_compute_result) == 600 && offsetof(cro_compute_result, host_ref_ns) == 32 &&
                  offsetof(cro_compute_result, bad_sm) == 48 && offsetof(cro_compute_result, leg) == 80 &&
                  offsetof(cro_compute_leg, fold) == 88,
              "compute layout");
static_assert(sizeof(cro_precision_opts) == 48 && offsetof(cro_precision_opts, test_inject_mask) == 40 &&
                  sizeof(cro_precision_result) == 808 && offsetof(cro_precision_result, leg) == 80 &&
                  sizeof(cro_precision_sm) == 288 && sizeof(cro_precision_fault) == 32 &&
                  offsetof(cro_precision_fault, actual_bits) == 24,
              "precision layout");

static_assert(sizeof(cro_scan_opts) == 72 && sizeof(cro_hbm_health) == 56 && sizeof(cro_scan_pass) == 552 &&
                  sizeof(cro_scan_chunk) == 88, "scan layout");
static_assert(sizeof(cro_scan_report) == 12632 && offsetof(cro_scan_report, element_ns) == 88 &&
                  offsetof(cro_scan_report, before) == 152 && offsetof(cro_scan_report, pass) == 264 &&
                  offsetof(cro_scan_report, chunk) == 1368 && offsetof(cro_hbm_health, ecc_corrected) == 40,
              "scan layout");
static_assert(sizeof(cro_sram_opts) == 48 && sizeof(cro_sram_health) == 24 && sizeof(cro_sram_pair) == 8 &&
                  sizeof(cro_sram_leg) == 168 && offsetof(cro_sram_leg, fold_xor) == 120 && sizeof(cro_sram_sm_leg) == 80 &&
                  sizeof(cro_sram_sm) == 168 && sizeof(cro_sram_fault) == 48, "sram layout");
static_assert(sizeof(cro_sram_result) == 568 && offsetof(cro_sram_result, bad_sm) == 56 && offsetof(cro_sram_result, bad_pair) == 96 &&
                  offsetof(cro_sram_result, recorded) == 160 && offsetof(cro_sram_result, before) == 184 &&
                  offsetof(cro_sram_result, leg) == 232,
              "sram layout");
static_assert(sizeof(cro_l2_opts) == 56 && sizeof(cro_l2_health) == 48 && sizeof(cro_l2_sm) == 128 && sizeof(cro_l2_fault) == 56 &&
                  sizeof(cro_l2_result) == 616 && offsetof(cro_l2_result, mismatches) == 80 &&
                  offsetof(cro_l2_result, bad_line) == 184 && offsetof(cro_l2_result, a1_bad) == 312 &&
                  offsetof(cro_l2_result, element_ns) == 400 && offsetof(cro_l2_result, before) == 520,
              "l2 layout");
static_assert(sizeof(cro_selftest_sweep_opts) == 128 && offsetof(cro_selftest_sweep_opts, force_or) == 104 &&
                  sizeof(cro_selftest_sweep_out) == 168 && offsetof(cro_selftest_sweep_out, mismatches) == 128,
              "selftest sweep layout");

using namespace cro::capi;


namespace cro {
namespace capi {
int on_exception() noexcept {
    try {
        throw;
    } catch (const std::bad_alloc&) {
        set_thread_error("out of host memory");
        return CRO_ERR_OOM;
    } catch (const std::exception& e) {
        set_thread_error(std::string("internal error: ") + e.what());
        return CRO_ERR_INTERNAL;
    } catch (...) {
        set_thread_error("internal error: unknown exception");
        return CRO_ERR_INTERNAL;
    }
}

// Every record-returning entry point copies its records out the same way: the first min(v.size(), cap) of v to
// to[], their count to *n, and returns that count.
template <class T>
size_t copy_capped(const std::vector<T>& v, T* to, int cap, int* n) {
    const size_t k = std::min(v.size(), (size_t)cap);
    std::copy(v.begin(), v.begin() + k, to);
    *n = (int)k;
    return k;
}

// The four per-SM probes (compute, precision, SRAM, L2), in process and by UUID, share their C side: the argument
// check (target: the context, or the GPU's UUID), opts' defaults, *n_sms and *n zeroed, then run(o, &seen, &found)
// and sms[0 .. sms_cap) and faults[0 .. cap) copied out.  copied is false when the arguments were refused: nothing
// ran and nothing was written.
struct PerSmCopy {
    int rc;
    bool copied;
    size_t sms, faults;
};
template <class Opts, class Sm, class Fault, class Run>
PerSmCopy per_sm_call(const void* target, const void* out, const Opts* opts, Sm* sms, int sms_cap, int* n_sms,
                      Fault* faults, int cap, int* n, Run run) {
    if (!target || !out || !n || !n_sms || cap < 0 || sms_cap < 0 || (cap > 0 && !faults) || (sms_cap > 0 && !sms))
        return {CRO_ERR_INVALID_ARG, false, 0, 0};
    *n = *n_sms = 0;
    Opts o{};
    if (opts) o = *opts;
    std::vector<Sm> seen;
    std::vector<Fault> found;
    const int rc = run(o, &seen, &found);
    return {rc, true, copy_capped(seen, sms, sms_cap, n_sms), copy_capped(found, faults, cap, n)};
}
// The SRAM and L2 results also say how much the caller got: sms_listed and recorded.
template <class Result>
int listed(const PerSmCopy& k, Result* out) {
    if (k.copied) {
        out->sms_listed = (uint32_t)k.sms;
        out->recorded = k.faults;
    }
    return k.rc;
}
}  // namespace capi
}  // namespace cro

extern "C" {

const char* cro_version(void) { return "croprobe 0.2.0 (sm_90a, abi 2)"; }

const char* cro_strerror(int code) {
    switch (code) {
        case CRO_OK: return "ok";
        case CRO_ERR_INVALID_ARG: return "invalid argument";
        case CRO_ERR_ABI_MISMATCH: return "abi version mismatch";
        case CRO_ERR_NO_DEVICE: return "no CUDA device";
        case CRO_ERR_CUDA: return "cuda runtime error";
        case CRO_ERR_OOM: return "sweep buffer allocation failed";
        case CRO_ERR_CHECKSUM: return "hbm checksum mismatch";
        case CRO_ERR_BUFFER_SMALL: return "output buffer too small";
        case CRO_ERR_NCCL: return "nccl error";
        case CRO_ERR_DEADLINE: return "deadline exceeded";
        case CRO_ERR_UNSUPPORTED: return "unsupported field";
        case CRO_ERR_PARSE: return "parse error";
        case CRO_ERR_EXEC: return "enumerate command failed";
        case CRO_ERR_P2P: return "peer access error";
        case CRO_ERR_INTERNAL: return "internal error";
        default: return "unknown error";
    }
}

int cro_last_error(cro_ctx* ctx, char* buf, size_t cap) try {
    if (!ctx) return copy_out(last_init_error(), buf, cap, nullptr);
    std::lock_guard<std::mutex> g(ctx->err_mu);
    return copy_out(ctx->last_error, buf, cap, nullptr);
} CRO_API_CATCH

int cro_selftest_exception_barrier(int kind) try {
    if (kind == 0) throw std::runtime_error("exception barrier self-test");
    if (kind == 1) throw std::bad_alloc();
    if (kind == 2) throw 42;
    return CRO_OK;
} CRO_API_CATCH

int cro_selftest_probe_finalize(cro_ctx* ctx, int i, const cro_probe_result* tmpl, const cro_sweep_slot* slots, uint64_t seed,
                                uint64_t nonce, uint64_t sweep_bytes, uint32_t read_sweeps, uint32_t copy_sweeps,
                                uint32_t read_variant, uint32_t copy_variant, cro_probe_result* out) try {
    if (!ctx) return CRO_ERR_INVALID_ARG;
    ProbeParams pp{};
    pp.seed = seed;
    pp.nonce = nonce;
    return ctx_selftest_probe_finalize(ctx, i, tmpl, slots, pp, sweep_bytes, read_sweeps, copy_sweeps, read_variant, copy_variant, out);
} CRO_API_CATCH
int cro_selftest_p2p_finalize(cro_ctx* ctx, int i, cro_probe_result* result, const cro_sweep_slot* slots,
                              const cro_sweep_slot* const* peer_slots, const uint64_t* peer_stamp, const uint64_t* chase_out,
                              const uint32_t* chase_expect, uint32_t n, uint32_t self, uint32_t hops, uint32_t have_push,
                              uint32_t push_folded, uint64_t p2p_bytes, uint64_t stamp) try {
    if (!ctx) return CRO_ERR_INVALID_ARG;
    return ctx_selftest_p2p_finalize(ctx, i, result, slots, peer_slots, peer_stamp, chase_out, chase_expect, n, self, hops,
                                     have_push, push_folded, p2p_bytes, stamp);
} CRO_API_CATCH
int cro_selftest_chase(cro_ctx* ctx, int i, const int32_t* minor_src, const int32_t* minor_dst, uint32_t n, uint32_t hops,
                       uint64_t* out) try {
    return ctx ? ctx_selftest_chase(ctx, i, minor_src, minor_dst, n, hops, out) : CRO_ERR_INVALID_ARG;
} CRO_API_CATCH
int cro_selftest_sweep(cro_ctx* ctx, int i, const cro_selftest_sweep_opts* opts, cro_selftest_sweep_out* out, void* buf,
                       uint64_t cap_bytes, cro_fault_word* words, int cap, int* n) try {
    return ctx ? ctx_selftest_sweep(ctx, i, opts, out, buf, cap_bytes, words, cap, n) : CRO_ERR_INVALID_ARG;
} CRO_API_CATCH

int cro_probe_init(const cro_opts* opts, cro_ctx** out) try { return ctx_create(opts, out); } CRO_API_CATCH
void cro_probe_destroy(cro_ctx* ctx) { ctx_destroy(ctx); }

int cro_device_count(cro_ctx* ctx, int* n) try {
    if (!ctx || !n) return CRO_ERR_INVALID_ARG;
    *n = (int)ctx->devs.size();
    return CRO_OK;
} CRO_API_CATCH

int cro_enumerate(cro_ctx* ctx, cro_dev_info* out, int cap, int* n) try {
    if (!ctx || !n) return CRO_ERR_INVALID_ARG;
    std::vector<cro_dev_info> inv;
    int rc = ctx_inventory(ctx, &inv);      // fresh every call: the reference re-execs nvidia-smi per reconcile
    if (rc) return rc;
    *n = (int)inv.size();
    if (*n == 0) return CRO_OK;
    if (!out || cap < *n) return CRO_ERR_BUFFER_SMALL;
    for (int i = 0; i < *n; ++i) out[i] = inv[(size_t)i];
    return CRO_OK;
} CRO_API_CATCH

int cro_node_inventory(const char* proc_root, const cro_dev_info* in_process, int n_in, cro_dev_info* out, int cap, int* n) try {
    if (!n || n_in < 0 || (n_in > 0 && !in_process)) return CRO_ERR_INVALID_ARG;
    const std::string root = proc_root && *proc_root ? proc_root : "/proc";
    std::vector<cro_dev_info> mine(in_process, in_process + n_in);
    const bool have = inventory::ProcRegistryExists(root);
    const std::vector<cro_dev_info> inv =
        inventory::Merge(mine, have, have ? inventory::FromProc(identity::ScanProc(root)) : std::vector<inventory::Seen>());
    *n = (int)inv.size();
    if (*n == 0) return CRO_OK;
    if (!out || cap < *n) return CRO_ERR_BUFFER_SMALL;
    for (int i = 0; i < *n; ++i) out[i] = inv[(size_t)i];
    return CRO_OK;
} CRO_API_CATCH

int cro_probe_uuid(cro_ctx* ctx, const char* gpu_uuid, cro_probe_result* out) try {
    return ctx_probe_uuid(ctx, gpu_uuid, out);
} CRO_API_CATCH

int cro_emit_csv(const cro_dev_info* devs, int n, const char* query, char* buf, size_t cap, size_t* len) try {
    if (!query || (n > 0 && !devs)) return CRO_ERR_INVALID_ARG;
    std::string out, err;
    int rc = identity::EmitCsv(devs, n, query, &out, &err);
    if (rc != CRO_OK) {
        copy_out(err, buf, cap, len);
        return rc;
    }
    return copy_out(out, buf, cap, len);
} CRO_API_CATCH

static int finish_parse(const identity::GpuInfoResult& r, char* buf, size_t cap, size_t* len) {
    if (r.code != CRO_OK) {
        int rc = copy_out(r.error, buf, cap, len);
        return rc == CRO_OK ? r.code : rc;
    }
    return copy_out(identity::GpuInfosToJson(r), buf, cap, len);
}

int cro_parse_gpu_csv(const char* std_out, const char* std_err, const char* exec_err, const char* query,
                      char* buf, size_t cap, size_t* len) try {
    if (!query) return CRO_ERR_INVALID_ARG;
    return finish_parse(identity::getGPUInfoFromNvidiaSmiOutput(S(std_out), S(std_err), exec_err, query),
                        buf, cap, len);
} CRO_API_CATCH

int cro_parse_proc_csv(const char* std_out, const char* std_err, const char* exec_err, const char* query,
                       char* buf, size_t cap, size_t* len) try {
    if (!query) return CRO_ERR_INVALID_ARG;
    return finish_parse(identity::getGPUInfoFromProcOutput(S(std_out), S(std_err), exec_err, query), buf,
                        cap, len);
} CRO_API_CATCH

int cro_proc_information_to_line(const char* text, char* buf, size_t cap, size_t* len) try {
    if (!text) return CRO_ERR_INVALID_ARG;
    return copy_out(identity::ProcInformationToLine(text), buf, cap, len);
} CRO_API_CATCH

int cro_check_gpu_visible(const cro_dev_info* devs, int n, const char* device_id, int* visible) try {
    if (!visible || !device_id || (n > 0 && !devs)) return CRO_ERR_INVALID_ARG;
    *visible = identity::CheckGPUVisible(devs, n, device_id) ? 1 : 0;
    return CRO_OK;
} CRO_API_CATCH

int cro_normalize(int kind, const char* in, char* buf, size_t cap, size_t* len) try {
    if (!in) return CRO_ERR_INVALID_ARG;
    std::string out;
    int rc = identity::Normalize(kind, in, &out);
    if (rc) return rc;
    return copy_out(out, buf, cap, len);
} CRO_API_CATCH

int cro_probe_device(cro_ctx* ctx, int dev_index, cro_probe_result* out) try {
    if (!ctx) return CRO_ERR_INVALID_ARG;
    return ctx_probe_device(ctx, dev_index, out);
} CRO_API_CATCH

int cro_probe_begin(cro_ctx* ctx, int dev_index) try { return ctx ? ctx_probe_begin(ctx, dev_index) : CRO_ERR_INVALID_ARG; } CRO_API_CATCH
int cro_probe_end(cro_ctx* ctx, int dev_index, cro_probe_result* out) try {
    return ctx ? ctx_probe_end(ctx, dev_index, out) : CRO_ERR_INVALID_ARG;
} CRO_API_CATCH

int cro_probe_all(cro_ctx* ctx, cro_probe_result* out, int cap, int* n) try {
    return ctx_probe_all(ctx, out, cap, n);
} CRO_API_CATCH

int cro_result_device_ptr(cro_ctx* ctx, int dev_index, uint64_t* dptr) try {
    if (!ctx || !dptr || dev_index < 0 || dev_index >= (int)ctx->devs.size()) return CRO_ERR_INVALID_ARG;
    *dptr = (uint64_t)(uintptr_t)ctx->devs[(size_t)dev_index]->d_result;
    return CRO_OK;
} CRO_API_CATCH

int cro_hbm_fill(cro_ctx* ctx, int i, cro_sweep_result* out) try { return ctx ? ctx_fill(ctx, i, 1, out) : CRO_ERR_INVALID_ARG; } CRO_API_CATCH
int cro_hbm_fill_loop(cro_ctx* ctx, int i, uint32_t iters, cro_sweep_result* out) try {
    return ctx ? ctx_fill(ctx, i, iters, out) : CRO_ERR_INVALID_ARG;
} CRO_API_CATCH
int cro_hbm_read_checksum(cro_ctx* ctx, int i, uint32_t variant, cro_sweep_result* out) try {
    return ctx ? ctx_read(ctx, i, variant, 1, false, out) : CRO_ERR_INVALID_ARG;
} CRO_API_CATCH
int cro_hbm_read_checksum_dst(cro_ctx* ctx, int i, uint32_t variant, cro_sweep_result* out) try {
    return ctx ? ctx_read(ctx, i, variant, 1, true, out) : CRO_ERR_INVALID_ARG;
} CRO_API_CATCH
int cro_hbm_read_loop(cro_ctx* ctx, int i, uint32_t variant, uint32_t iters, cro_sweep_result* out) try {
    return ctx ? ctx_read(ctx, i, variant, iters, false, out) : CRO_ERR_INVALID_ARG;
} CRO_API_CATCH
int cro_hbm_copy(cro_ctx* ctx, int i, uint32_t variant, cro_sweep_result* out) try {
    return ctx ? ctx_copy(ctx, i, variant, 1, out) : CRO_ERR_INVALID_ARG;
} CRO_API_CATCH
int cro_hbm_copy_loop(cro_ctx* ctx, int i, uint32_t variant, uint32_t iters, cro_sweep_result* out) try {
    return ctx ? ctx_copy(ctx, i, variant, iters, out) : CRO_ERR_INVALID_ARG;
} CRO_API_CATCH
int cro_hbm_expected_checksum(cro_ctx* ctx, int i, cro_sweep_result* out) try {
    return ctx ? ctx_expected(ctx, i, out) : CRO_ERR_INVALID_ARG;
} CRO_API_CATCH
int cro_inject_fault(cro_ctx* ctx, int i, uint64_t word, uint64_t mask) try {
    return ctx ? ctx_inject(ctx, i, word, mask) : CRO_ERR_INVALID_ARG;
} CRO_API_CATCH
int cro_read_words(cro_ctx* ctx, int i, uint64_t first, uint64_t n, uint64_t* out) try {
    return ctx ? ctx_read_words(ctx, i, first, n, out) : CRO_ERR_INVALID_ARG;
} CRO_API_CATCH
int cro_locate_faults(cro_ctx* ctx, int i, const cro_locate_opts* opts, cro_fault_report* out, cro_fault_word* words, int cap,
                      int* n) try {
    if (!ctx || !out || !n || cap < 0 || (cap > 0 && !words)) return CRO_ERR_INVALID_ARG;
    *n = 0;
    cro_locate_opts o{};
    if (opts) o = *opts;
    std::vector<cro_fault_word> found;
    const int rc = ctx_locate(ctx, i, o, out, &found);
    out->recorded = copy_capped(found, words, cap, n);
    if (out->recorded < found.size()) out->complete = 0;        // the caller's list misses some located words
    return rc;
} CRO_API_CATCH
int cro_probe_host_link(cro_ctx* ctx, int i, const cro_link_opts* opts, cro_link_result* out, cro_link_fault* faults, int cap,
                        int* n) try {
    if (!ctx || !out || !n || cap < 0 || (cap > 0 && !faults)) return CRO_ERR_INVALID_ARG;
    *n = 0;
    cro_link_opts o{};
    if (opts) o = *opts;
    std::vector<cro_link_fault> found;
    const int rc = ctx_probe_host_link(ctx, i, o, out, &found);
    copy_capped(found, faults, cap, n);
    return rc;
} CRO_API_CATCH
int cro_probe_host_link_uuid(cro_ctx* ctx, const char* gpu_uuid, const cro_link_opts* opts, int deadline_ms, cro_link_result* out,
                             cro_link_fault* faults, int cap, int* n, uint64_t* helper_ns) try {
    if (!gpu_uuid || !out || !n || cap < 0 || (cap > 0 && !faults)) return CRO_ERR_INVALID_ARG;
    *n = 0;
    if (helper_ns) *helper_ns = 0;
    cro_link_opts o{};
    if (opts) o = *opts;
    std::vector<cro_link_fault> found;
    uint64_t ns = 0;
    const int rc = ctx_probe_host_link_uuid(ctx, gpu_uuid, o, deadline_ms, out, &found, cap, &ns);
    copy_capped(found, faults, cap, n);
    if (helper_ns) *helper_ns = ns;
    return rc;
} CRO_API_CATCH
int cro_probe_compute(cro_ctx* ctx, int i, const cro_compute_opts* opts, cro_compute_result* out, cro_compute_sm* sms,
                      int sms_cap, int* n_sms, cro_compute_fault* faults, int cap, int* n) try {
    return per_sm_call(ctx, out, opts, sms, sms_cap, n_sms, faults, cap, n, [&](const cro_compute_opts& o, auto* seen, auto* found) {
        return ctx_probe_compute(ctx, i, o, out, seen, found);
    }).rc;
} CRO_API_CATCH
int cro_probe_compute_uuid(cro_ctx* ctx, const char* gpu_uuid, const cro_compute_opts* opts, int deadline_ms,
                           cro_compute_result* out, cro_compute_sm* sms, int sms_cap, int* n_sms, cro_compute_fault* faults,
                           int cap, int* n, uint64_t* helper_ns) try {
    return per_sm_call(gpu_uuid, out, opts, sms, sms_cap, n_sms, faults, cap, n, [&](const cro_compute_opts& o, auto* seen, auto* found) {
        uint64_t ns = 0;
        if (helper_ns) *helper_ns = 0;
        const int rc = ctx_probe_compute_uuid(ctx, gpu_uuid, o, deadline_ms, out, seen, found, cap, &ns);
        if (helper_ns) *helper_ns = ns;
        return rc;
    }).rc;
} CRO_API_CATCH
int cro_probe_precision(cro_ctx* ctx, int i, const cro_precision_opts* opts, cro_precision_result* out, cro_precision_sm* sms,
                        int sms_cap, int* n_sms, cro_precision_fault* faults, int cap, int* n) try {
    return per_sm_call(ctx, out, opts, sms, sms_cap, n_sms, faults, cap, n, [&](const cro_precision_opts& o, auto* seen, auto* found) {
        return ctx_probe_precision(ctx, i, o, out, seen, found);
    }).rc;
} CRO_API_CATCH
int cro_probe_precision_uuid(cro_ctx* ctx, const char* gpu_uuid, const cro_precision_opts* opts, int deadline_ms,
                             cro_precision_result* out, cro_precision_sm* sms, int sms_cap, int* n_sms,
                             cro_precision_fault* faults, int cap, int* n, uint64_t* helper_ns) try {
    return per_sm_call(gpu_uuid, out, opts, sms, sms_cap, n_sms, faults, cap, n, [&](const cro_precision_opts& o, auto* seen, auto* found) {
        uint64_t ns = 0;
        if (helper_ns) *helper_ns = 0;
        const int rc = ctx_probe_precision_uuid(ctx, gpu_uuid, o, deadline_ms, out, seen, found, cap, &ns);
        if (helper_ns) *helper_ns = ns;
        return rc;
    }).rc;
} CRO_API_CATCH
int cro_scan_hbm(cro_ctx* ctx, int i, const cro_scan_opts* opts, cro_scan_report* out, cro_fault_word* words, int cap, int* n) try {
    if (!ctx || !out || !n || cap < 0 || (cap > 0 && !words)) return CRO_ERR_INVALID_ARG;
    *n = 0;
    cro_scan_opts o{};
    if (opts) o = *opts;
    std::vector<cro_fault_word> found;
    const int rc = ctx_scan_hbm(ctx, i, o, out, &found);
    out->recorded = copy_capped(found, words, cap, n);
    if (out->recorded < found.size()) out->complete = 0;        // the caller's list misses some words
    return rc;
} CRO_API_CATCH
int cro_scan_hbm_uuid(cro_ctx* ctx, const char* gpu_uuid, const cro_scan_opts* opts, cro_scan_report* out, cro_fault_word* words,
                      int cap, int* n) try {
    if (!gpu_uuid || !out || !n || cap < 0 || (cap > 0 && !words)) return CRO_ERR_INVALID_ARG;
    *n = 0;
    cro_scan_opts o{};
    if (opts) o = *opts;
    std::vector<cro_fault_word> found;
    const int rc = ctx_scan_hbm_uuid(ctx, gpu_uuid, o, out, &found, cap);
    out->recorded = copy_capped(found, words, cap, n);
    out->complete = out->complete && found.size() <= (size_t)cap;
    return rc;
} CRO_API_CATCH
int cro_read_hbm_health(const char* gpu_uuid, cro_hbm_health* out) try {
    if (!gpu_uuid || !out) return CRO_ERR_INVALID_ARG;
    identity::NvmlHbmHealth(gpu_uuid, true, out);
    return CRO_OK;
} CRO_API_CATCH
int cro_probe_sram(cro_ctx* ctx, int i, const cro_sram_opts* opts, cro_sram_result* out, cro_sram_sm* sms, int sms_cap,
                   int* n_sms, cro_sram_fault* faults, int cap, int* n) try {
    return listed(per_sm_call(ctx, out, opts, sms, sms_cap, n_sms, faults, cap, n, [&](const cro_sram_opts& o, auto* seen, auto* found) {
        return ctx_probe_sram(ctx, i, o, out, seen, found);
    }), out);
} CRO_API_CATCH
int cro_probe_sram_uuid(cro_ctx* ctx, const char* gpu_uuid, const cro_sram_opts* opts, cro_sram_result* out, cro_sram_sm* sms,
                        int sms_cap, int* n_sms, cro_sram_fault* faults, int cap, int* n) try {
    return listed(per_sm_call(gpu_uuid, out, opts, sms, sms_cap, n_sms, faults, cap, n, [&](const cro_sram_opts& o, auto* seen, auto* found) {
        return ctx_probe_sram_uuid(ctx, gpu_uuid, o, out, seen, found, cap);
    }), out);
} CRO_API_CATCH
int cro_read_sram_health(const char* gpu_uuid, cro_sram_health* out) try {
    if (!gpu_uuid || !out) return CRO_ERR_INVALID_ARG;
    identity::NvmlSramHealth(gpu_uuid, true, out);
    return CRO_OK;
} CRO_API_CATCH
int cro_probe_l2(cro_ctx* ctx, int i, const cro_l2_opts* opts, cro_l2_result* out, cro_l2_sm* sms, int sms_cap, int* n_sms,
                 cro_l2_fault* faults, int cap, int* n) try {
    return listed(per_sm_call(ctx, out, opts, sms, sms_cap, n_sms, faults, cap, n, [&](const cro_l2_opts& o, auto* seen, auto* found) {
        return ctx_probe_l2(ctx, i, o, out, seen, found);
    }), out);
} CRO_API_CATCH
int cro_probe_l2_uuid(cro_ctx* ctx, const char* gpu_uuid, const cro_l2_opts* opts, cro_l2_result* out, cro_l2_sm* sms,
                      int sms_cap, int* n_sms, cro_l2_fault* faults, int cap, int* n) try {
    return listed(per_sm_call(gpu_uuid, out, opts, sms, sms_cap, n_sms, faults, cap, n, [&](const cro_l2_opts& o, auto* seen, auto* found) {
        return ctx_probe_l2_uuid(ctx, gpu_uuid, o, out, seen, found, cap);
    }), out);
} CRO_API_CATCH
int cro_read_l2_health(const char* gpu_uuid, cro_l2_health* out) try {
    if (!gpu_uuid || !out) return CRO_ERR_INVALID_ARG;
    identity::NvmlL2Health(gpu_uuid, true, out);
    return CRO_OK;
} CRO_API_CATCH
int cro_selftest_l2_classify(cro_l2_result* r, cro_l2_sm* sms, int n_sms, cro_l2_fault* faults, int n) try {
    if (!r || n_sms < 0 || n < 0 || (n_sms > 0 && !sms) || (n > 0 && !faults)) return CRO_ERR_INVALID_ARG;
    l2_classify(r, sms, (size_t)n_sms, faults, (size_t)n);
    return CRO_OK;
} CRO_API_CATCH
int cro_selftest_sm_legs_classify(int probe, uint32_t legs, const uint32_t* iterations, uint32_t grid, uint64_t call,
                                  const uint32_t* rounds, const cro_sm_cta* ctas, const uint64_t* sm_bits, const uint64_t* claims,
                                  const void* records, void* out, void* sms, int sms_cap, int* n_sms, void* faults, int cap,
                                  int* n) try {
    const uint32_t n_legs = probe == CRO_SM_LEGS_COMPUTE ? CRO_COMPUTE_LEGS : CRO_PRECISION_LEGS;
    const uint32_t max_records = probe == CRO_SM_LEGS_COMPUTE ? CRO_COMPUTE_RECORDS : CRO_PRECISION_RECORDS;
    const uint32_t all = (1u << n_legs) - 1;
    if (legs == 0) legs = all;
    if ((probe != CRO_SM_LEGS_COMPUTE && probe != CRO_SM_LEGS_PRECISION) || (legs & ~all) || !iterations || !rounds || !claims ||
        grid == 0 || !out || !n_sms || !n || sms_cap < 0 || cap < 0 || (sms_cap > 0 && !sms) || (cap > 0 && !faults))
        return CRO_ERR_INVALID_ARG;
    uint64_t n_rounds = 0, n_records = 0;
    for (uint32_t l = 0; l < n_legs; ++l) {
        if (!(legs >> l & 1u)) continue;
        if (!iterations[l]) return CRO_ERR_INVALID_ARG;
        n_rounds += rounds[l];
        n_records += std::min<uint64_t>(claims[l], max_records);
    }
    if ((n_rounds && (!ctas || !sm_bits)) || (n_records && !records)) return CRO_ERR_INVALID_ARG;
    *n = *n_sms = 0;
    if (probe == CRO_SM_LEGS_COMPUTE) {
        std::vector<cro_compute_sm> seen;
        std::vector<cro_compute_fault> found;
        const int rc = classify_compute(legs, iterations, grid, call, rounds, ctas, sm_bits, claims,
                                        static_cast<const cro_compute_fault*>(records), static_cast<cro_compute_result*>(out),
                                        &seen, &found);
        copy_capped(seen, static_cast<cro_compute_sm*>(sms), sms_cap, n_sms);
        copy_capped(found, static_cast<cro_compute_fault*>(faults), cap, n);
        return rc;
    }
    std::vector<cro_precision_sm> seen;
    std::vector<cro_precision_fault> found;
    const int rc = classify_precision(legs, iterations, grid, call, rounds, ctas, sm_bits, claims,
                                      static_cast<const cro_precision_fault*>(records), static_cast<cro_precision_result*>(out),
                                      &seen, &found);
    copy_capped(seen, static_cast<cro_precision_sm*>(sms), sms_cap, n_sms);
    copy_capped(found, static_cast<cro_precision_fault*>(faults), cap, n);
    return rc;
} CRO_API_CATCH
int cro_selftest_sram_classify(uint32_t legs, uint32_t iterations, uint32_t n_words, uint64_t seed, uint32_t cluster,
                               uint32_t sm_count, uint32_t net_grid, uint64_t call, const uint32_t* rounds, const cro_sram_cta* ctas,
                               const uint64_t* claims, const cro_sram_record* records, cro_sram_result* out, cro_sram_sm* sms,
                               int sms_cap, int* n_sms, cro_sram_fault* faults, int cap, int* n) try {
    if (legs == 0) legs = CRO_SRAM_ALL_LEGS;
    const bool net = legs & CRO_SRAM_LEG_DSMEM;
    if ((legs & ~CRO_SRAM_ALL_LEGS) || iterations == 0 || iterations > CRO_SRAM_MAX_ITERATIONS ||
        (cluster != 2 && cluster != 4 && cluster != 8) || sm_count == 0 || (net && (net_grid == 0 || net_grid % cluster)) ||
        !rounds || !claims || !out || !n_sms || !n || sms_cap < 0 || cap < 0 || (sms_cap > 0 && !sms) || (cap > 0 && !faults))
        return CRO_ERR_INVALID_ARG;
    uint64_t n_ctas = 0, n_records = 0;
    for (uint32_t l = 0; l < CRO_SRAM_LEGS; ++l) {
        if (!(legs >> l & 1u)) continue;
        n_ctas += (uint64_t)rounds[l] * (l == CRO_SRAM_DSMEM ? net_grid : sm_count);
        n_records += std::min<uint64_t>(claims[l], CRO_SRAM_RECORDS);
    }
    if ((n_ctas && !ctas) || (n_records && !records)) return CRO_ERR_INVALID_ARG;
    *n = *n_sms = 0;
    std::vector<cro_sram_sm> seen;
    std::vector<cro_sram_fault> found;
    const int rc = classify_sram(legs, iterations, n_words, seed, cluster, sm_count, net_grid, call, rounds, ctas, claims, records,
                                 out, &seen, &found);
    return listed({rc, true, copy_capped(seen, sms, sms_cap, n_sms), copy_capped(found, faults, cap, n)}, out);
} CRO_API_CATCH
int cro_compute_expected(int answer, uint64_t seed, int32_t* out) try {
    return compute::Expected(answer, seed, out);
} CRO_API_CATCH
int cro_precision_expected(int answer, uint64_t seed, int64_t* out) try {
    return precision::Expected(answer, seed, out);
} CRO_API_CATCH
int cro_pci_link_path(const char* sys_root, const char* pci_bus_id, cro_pci_path* out) try {
    if (!pci_bus_id || !out) return CRO_ERR_INVALID_ARG;
    return pcilink::ReadPath(sys_root && *sys_root ? sys_root : "/sys", pci_bus_id, out);
} CRO_API_CATCH
int cro_device_seed(cro_ctx* ctx, int i, uint64_t* seed) try {
    if (!ctx || !seed || i < 0 || i >= (int)ctx->devs.size()) return CRO_ERR_INVALID_ARG;
    std::lock_guard<std::mutex> g(ctx->devs[(size_t)i]->mu);
    *seed = ctx->devs[(size_t)i]->seed_cur;
    return CRO_OK;
} CRO_API_CATCH

int cro_probe_sweep_times(cro_ctx* ctx, int i, cro_sweep_time* out, int cap, int* n) try {
    return ctx ? ctx_sweep_times(ctx, i, out, cap, n) : CRO_ERR_INVALID_ARG;
} CRO_API_CATCH

int cro_p2p_detail_get(cro_ctx* ctx, int i, int peer, cro_p2p_detail* out) try {
    return ctx ? ctx_p2p_detail(ctx, i, peer, out) : CRO_ERR_INVALID_ARG;
} CRO_API_CATCH

int cro_fullbox_times(cro_ctx* ctx, cro_fullbox_time* out) try {
    if (!ctx || !out) return CRO_ERR_INVALID_ARG;
    std::lock_guard<std::mutex> g(ctx->all_mu);
    const FullBoxTimes& f = ctx->fullbox;
    out->enqueue_ns = f.enqueue_ns;
    out->wall_ns = f.wall_ns;
    out->hbm_ns = f.hbm_ns;
    out->p2p_ns = f.p2p_ns;
    out->chase_ns = f.chase_ns;
    out->gather_ns = f.gather_ns;
    out->rounds = f.rounds;
    out->host_syncs = f.host_syncs;
    out->gather = f.gather;
    out->reserved = 0;
    return CRO_OK;
} CRO_API_CATCH

int cro_set_latency_hops(cro_ctx* ctx, uint32_t hops) try {
    if (!ctx || hops == 0 || hops > (1u << 24)) return CRO_ERR_INVALID_ARG;
    std::lock_guard<std::mutex> g(ctx->all_mu);
    ctx->opts.latency_hops = hops;      // the next cro_probe_all recomputes where each chase must end
    return CRO_OK;
} CRO_API_CATCH

int cro_metrics_text(cro_ctx* ctx, char* buf, size_t cap, size_t* len) try {
    if (!ctx) return CRO_ERR_INVALID_ARG;
    return copy_out(ctx_metrics_text(ctx), buf, cap, len);
} CRO_API_CATCH

static void describe_type(const gojson::GoType& t, gojson::Writer* w) {
    w->begin_object();
    w->field("type", t.name);
    if (t.kind == gojson::GoType::Struct) {
        w->field("struct", t.structName);
        w->key("fields").begin_array();
        for (const auto& f : t.fields) {
            w->begin_object();
            w->field("json", f.first);
            w->key("of");
            describe_type(*f.second, w);
            w->end_object();
        }
        w->end_array();
    } else if (t.kind == gojson::GoType::Slice && t.elem) {
        w->key("elem");
        describe_type(*t.elem, w);
    }
    w->end_object();
}

int cro_describe_wire_type(const char* name, char* buf, size_t cap, size_t* len) try {
    const std::string n = S(name);
    const gojson::GoType* t = n == "FMScaleUpResponse" ? &gotypes::FMScaleUpResponse()
                              : n == "FMGetMachineResponse" ? &gotypes::FMGetMachineResponse()
                              : n == "CMMachineData" ? &gotypes::CMMachineData() : nullptr;
    if (!t) return CRO_ERR_INVALID_ARG;
    gojson::Writer w;
    describe_type(*t, &w);
    return copy_out(w.take(), buf, cap, len);
} CRO_API_CATCH

int cro_chase_end(int minor_src, int minor_dst, uint32_t hops, uint32_t* end) try {
    if (!end) return CRO_ERR_INVALID_ARG;
    std::vector<uint32_t> perm;
    chase_permutation(minor_src, minor_dst, &perm);
    uint32_t at = 0;
    for (uint32_t h = 0; h < hops; ++h) at = perm[at];
    *end = at;
    return CRO_OK;
} CRO_API_CATCH

int cro_validate_env(const char* name, const char* value, char* err_buf, size_t err_cap) try {
    int n = 0;
    const env::Knob* t = env::table(&n);
    std::string why;
    if (name) {
        for (int i = 0; i < n; ++i) {
            if (S(name) != t[i].name) continue;
            unsigned v = 0;
            if (env::parse(t[i], value, &v, &why)) return CRO_OK;
            copy_out(why, err_buf, err_cap, nullptr);
            return CRO_ERR_INVALID_ARG;
        }
        copy_out("unknown knob " + S(name), err_buf, err_cap, nullptr);
        return CRO_ERR_UNSUPPORTED;
    }
    env::Values checked;                      // a check only: no context's knobs change
    if (env::read(&checked, &why)) return CRO_OK;
    copy_out(why, err_buf, err_cap, nullptr);
    return CRO_ERR_INVALID_ARG;
} CRO_API_CATCH
uint64_t cro_launch_count(cro_ctx* ctx) { return ctx ? ctx->launches.load() : 0; }

// ---- emitters --------------------------------------------------------------

int cro_emit_status_json(const char* state, const char* error, const char* device_id,
                         const char* cdi_device_id, char* buf, size_t cap, size_t* len) try {
    controller::ComposableResourceStatus st;
    st.State = S(state);
    st.Error = S(error);
    st.DeviceID = S(device_id);
    st.CDIDeviceID = S(cdi_device_id);
    return copy_out(st.MarshalJSON(), buf, cap, len);
} CRO_API_CATCH

int cro_emit_scalar_status_json(const char* state, const char* device_id, const char* cdi_device_id,
                                const char* node_name, const char* error, char* buf, size_t cap,
                                size_t* len) try {
    // api/v1alpha1/composabilityrequest_types.go:74-80 (declaration order)
    gojson::Writer w;
    w.begin_object();
    w.field("state", S(state));
    w.field_omitempty("device_id", S(device_id));
    w.field_omitempty("cdi_device_id", S(cdi_device_id));
    w.field_omitempty("node_name", S(node_name));
    w.field_omitempty("error", S(error));
    w.end_object();
    return copy_out(w.str(), buf, cap, len);
} CRO_API_CATCH

int cro_emit_fm_scale_up(const char* tenant_uuid, const char* mach_uuid, const char* res_type,
                         const char* model, char* buf, size_t cap, size_t* len) try {
    return copy_out(fabric::FMScaleUpBody(S(tenant_uuid), S(mach_uuid), S(res_type), S(model)), buf, cap, len);
} CRO_API_CATCH

int cro_emit_fm_scale_down(const char* tenant_uuid, const char* mach_uuid, const char* res_type,
                           const char* res_uuid, char* buf, size_t cap, size_t* len) try {
    return copy_out(fabric::FMScaleDownBody(S(tenant_uuid), S(mach_uuid), S(res_type), S(res_uuid)), buf, cap, len);
} CRO_API_CATCH

int cro_emit_cm_scale_up(const char* spec_uuid, int device_count, char* buf, size_t cap, size_t* len) try {
    return copy_out(fabric::CMScaleUpBody(S(spec_uuid), device_count), buf, cap, len);
} CRO_API_CATCH

int cro_emit_cm_scale_down(const char* spec_uuid, int device_count, const char* device_id, char* buf,
                           size_t cap, size_t* len) try {
    return copy_out(fabric::CMScaleDownBody(S(spec_uuid), device_count, S(device_id)), buf, cap, len);
} CRO_API_CATCH

int cro_emit_sunfish_request(const char* name, long long count, const char* proc_type, const char* model,
                             char* buf, size_t cap, size_t* len) try {
    return copy_out(fabric::SunfishBody(S(name), count, S(proc_type), S(model)), buf, cap, len);
} CRO_API_CATCH

}  // extern "C" (reopened below)

// ---- annotation helpers: each emitter names its own keys and builds their values from these ----

using Annotations = std::map<std::string, std::string>;

static int emit(const Annotations& m, char* buf, size_t cap, size_t* len) {
    gojson::Writer w;
    w.string_map(m);
    return copy_out(w.str(), buf, cap, len);
}
// "f(0),f(1),...,f(n-1)"
template <class F>
static std::string join(uint64_t n, F f) {
    std::string s;
    for (uint64_t j = 0; j < n; ++j) s += (j ? "," : "") + f(j);
    return s;
}
// The first n values of v, in decimal.
template <class T>
static std::string join(const T* v, uint64_t n) {
    return join(n, [&](uint64_t j) { return std::to_string(v[j]); });
}
// The bit numbers b < 64 for which flipped(b) holds, comma-joined.
template <class F>
static std::string bit_numbers(F flipped) {
    std::string s;
    for (int b = 0; b < 64; ++b)
        if (flipped(b)) s += (s.empty() ? "" : ",") + std::to_string(b);
    return s;
}
// names[b] for each bit b < n set in mask, comma-joined.
static std::string bit_names(uint32_t mask, const char* const* names, int n) {
    std::string s;
    for (int b = 0; b < n; ++b)
        if (mask >> b & 1u) s += (s.empty() ? "" : ",") + std::string(names[b]);
    return s;
}
// A list-valued key is written only when its list has an entry.
static void put_list(Annotations& m, const std::string& key, const std::string& list) {
    if (!list.empty()) m[key] = list;
}
// The least sms_covered over the legs run: the "sms" key's numerator, 0 when no leg ran.
template <class Leg>
static uint32_t min_covered(uint32_t legs, const Leg* leg, int n_legs) {
    uint32_t covered = 0xFFFFFFFFu;
    for (int l = 0; l < n_legs; ++l)
        if (legs >> l & 1u) covered = std::min(covered, leg[l].sms_covered);
    return covered == 0xFFFFFFFFu ? 0u : covered;
}
// How much each ECC count grew over the call, for a count NVML gave both before and after it.
template <class Health>
static void ecc_delta(Annotations& m, const std::string& p, const Health& B, const Health& A, uint32_t corrected_bit,
                      uint32_t uncorrected_bit) {
    if (B.nvml & A.nvml & corrected_bit) m[p + "ecc-corrected"] = std::to_string(A.ecc_corrected - B.ecc_corrected);
    if (B.nvml & A.nvml & uncorrected_bit) m[p + "ecc-uncorrected"] = std::to_string(A.ecc_uncorrected - B.ecc_uncorrected);
}
static std::string cuda_error(int32_t e) { return "cuda-error:" + std::to_string(e); }

// The compute and precision results both hold a cro_compute_leg per leg.  Their annotations differ only in the key
// prefix p, the leg names and which legs report a rate under which key.
struct LegRate {
    int leg;
    const char* key;
};
template <class Result>
static int emit_sm_legs(const Result& r, const std::string& p, const char* const* leg_name, int n_legs,
                        std::initializer_list<LegRate> rates, char* buf, size_t cap, size_t* len) {
    Annotations m;
    m[p + "verdict"] = r.status == CRO_OK                                               ? "ok"
                       : r.status == CRO_ERR_CHECKSUM && r.verdict == CRO_COMPUTE_SM  ? "sm"
                       : r.status == CRO_ERR_CHECKSUM && r.verdict == CRO_COMPUTE_ALL ? "all"
                                                                                      : "error";
    m[p + "sms"] = std::to_string(min_covered(r.legs, r.leg, n_legs)) + "/" + std::to_string(r.sm_count);
    if (r.bad_sms) m[p + "bad-sms"] = join(r.bad_sm, std::min<uint32_t>(r.bad_sms, 16));
    uint32_t failed = 0;
    int worst = n_legs;     // the first leg with the largest slow_permille
    for (int l = 0; l < n_legs; ++l) {
        if (!(r.legs >> l & 1u)) continue;
        const cro_compute_leg& L = r.leg[l];
        if (L.mismatches || L.fold_mismatches || L.unpublished) failed |= 1u << l;
        if (worst == n_legs || L.slow_permille > r.leg[worst].slow_permille) worst = l;
    }
    put_list(m, p + "failed-legs", bit_names(failed, leg_name, n_legs));
    for (const LegRate& q : rates) {
        const cro_compute_leg& L = r.leg[q.leg];
        m[p + q.key] = std::to_string(L.ns ? L.ops / L.ns : 0ull);
    }
    if (worst < n_legs)
        m[p + "slowest-sm"] = std::to_string(r.leg[worst].slowest_sm) + " " + std::to_string(r.leg[worst].slow_permille);
    return emit(m, buf, cap, len);
}

std::map<std::string, std::string> cro::capi::probe_annotations(const cro_probe_result& r) {
    std::map<std::string, std::string> m;
    m["cohdi.io/probe-status"] = cro_strerror(r.status);
    m["cohdi.io/probe-device-id"] = fixed_str(r.gpu_uuid, sizeof r.gpu_uuid);
    m["cohdi.io/probe-pci-bus-id"] = fixed_str(r.pci_bus_id, sizeof r.pci_bus_id);
    m["cohdi.io/probe-device-minor"] = std::to_string(r.device_minor);
    m["cohdi.io/probe-sweep-bytes"] = std::to_string(r.sweep_bytes);
    m["cohdi.io/probe-checksum"] = hex16(r.checksum_xor) + ":" + hex16(r.checksum_sum) + ":" + hex16(r.checksum_wsum);
    m["cohdi.io/probe-nonce"] = std::to_string(r.nonce);
    if (r.copy_sweeps) m["cohdi.io/probe-copies-verified"] = std::to_string((unsigned)r.copy_verified) + "/" + std::to_string((unsigned)r.copy_sweeps);
    m["cohdi.io/probe-ecc-uncorrected"] = std::to_string(r.ecc_errors);
    m["cohdi.io/probe-hbm-fill-gbs"] = gbs_x10(r.sweep_bytes, r.fill_ns);
    m["cohdi.io/probe-hbm-read-gbs"] = gbs_x10(r.sweep_bytes, r.read_best_ns);
    if (r.copy_sweeps) m["cohdi.io/probe-hbm-copy-gbs"] = gbs_x10(2 * r.sweep_bytes, r.copy_best_ns);
    std::string bw, lat;
    for (int j = 0; j < 8; ++j) {
        if (!r.p2p_read_ns[j]) continue;
        if (!bw.empty()) { bw += ","; lat += ","; }
        bw += std::to_string(j) + ":" + gbs_x10(r.p2p_bytes, r.p2p_read_ns[j]);
        lat += std::to_string(j) + ":" + std::to_string(r.p2p_latency_ns_x16[j] / 16);
    }
    if (!bw.empty()) {
        m["cohdi.io/probe-nvlink-read-gbs"] = bw;
        m["cohdi.io/probe-nvlink-latency-ns"] = lat;
    }
    std::string wr;
    for (int j = 0; j < 8; ++j) {
        if (!r.p2p_write_ns[j]) continue;
        if (!wr.empty()) wr += ",";
        wr += std::to_string(j) + ":" + gbs_x10(r.p2p_bytes, r.p2p_write_ns[j]);
    }
    if (!wr.empty()) m["cohdi.io/probe-nvlink-write-gbs"] = wr;
    return m;
}

extern "C" {

int cro_emit_probe_annotations_json(const cro_probe_result* r, char* buf, size_t cap, size_t* len) try {
    if (!r) return CRO_ERR_INVALID_ARG;
    return emit(probe_annotations(*r), buf, cap, len);
} CRO_API_CATCH

int cro_emit_fault_annotations_json(const cro_fault_report* r, const cro_fault_word* words, int n, char* buf, size_t cap,
                                    size_t* len) try {
    if (!r || n < 0 || (n > 0 && !words)) return CRO_ERR_INVALID_ARG;
    static const char* const kVerdict[] = {"none", "unclassified", "not-reproduced", "persistent"};
    Annotations m;
    m["cohdi.io/probe-fault-verdict"] = kVerdict[fault_verdict(*r)];
    const uint32_t np = std::min<uint32_t>(r->n_passes, CRO_LOCATE_PASSES);
    m["cohdi.io/probe-fault-mismatches"] =
        join(np, [&](uint64_t p) { return std::to_string(p) + ":" + std::to_string(r->pass[p].mismatches); });
    m["cohdi.io/probe-fault-granules"] =
        join(np, [&](uint64_t p) { return std::to_string(p) + ":" + std::to_string(r->pass[p].granules); });
    put_list(m, "cohdi.io/probe-fault-bits", bit_numbers([&](int b) { return r->bit_flips[b] != 0; }));
    put_list(m, "cohdi.io/probe-fault-words", join(std::min(n, 8), [&](uint64_t k) {
                 char idx[24];
                 snprintf(idx, sizeof idx, "%llx", (unsigned long long)words[k].word_index);
                 return std::string(idx) + ":" + hex16(words[k].expected ^ words[k].actual);
             }));
    return emit(m, buf, cap, len);
} CRO_API_CATCH

static std::string link_speed(uint32_t tenths) {
    if (!tenths) return "unknown";
    return std::to_string(tenths / 10) + "." + std::to_string(tenths % 10) + "GT/s";
}
static std::string mbps(uint64_t bytes, uint64_t ns) {
    // bytes * 1000 / ns without overflow: 128-bit intermediate
    return std::to_string(ns ? (uint64_t)((unsigned __int128)bytes * 1000u / ns) : 0ull);
}

int cro_emit_link_annotations_json(const cro_link_result* r, char* buf, size_t cap, size_t* len) try {
    if (!r) return CRO_ERR_INVALID_ARG;
    static const char* const kCheck[CRO_LINK_CHECKS] = {"d2h-copy", "h2d-copy", "sm-write", "duplex-write", "duplex-d2h-copy",
                                                         "chase"};
    static const char* const kDegraded[4] = {"speed", "width", "path", "bottleneck"};
    Annotations m;
    const std::string p = "cohdi.io/probe-link-";
    m[p + "verdict"] = r->first_fail < CRO_LINK_CHECKS ? std::string("corrupt:") + kCheck[r->first_fail]
                       : r->status == CRO_OK       ? "ok"
                                                   : "error";
    const cro_link_leg* L = r->leg;
    m[p + "h2d-mbps"] = mbps(L[CRO_LINK_LEG_CE_H2D].bytes, L[CRO_LINK_LEG_CE_H2D].ns);
    m[p + "d2h-mbps"] = mbps(L[CRO_LINK_LEG_CE_D2H].bytes, L[CRO_LINK_LEG_CE_D2H].ns);
    m[p + "duplex-mbps"] = mbps(L[CRO_LINK_LEG_CE_DUPLEX_H2D].bytes + L[CRO_LINK_LEG_CE_DUPLEX_D2H].bytes, r->ce_duplex_span_ns);
    m[p + "sm-h2d-mbps"] = mbps(L[CRO_LINK_LEG_SM_H2D].bytes, L[CRO_LINK_LEG_SM_H2D].ns);
    m[p + "sm-d2h-mbps"] = mbps(L[CRO_LINK_LEG_SM_D2H].bytes, L[CRO_LINK_LEG_SM_D2H].ns);
    m[p + "latency-ns"] = std::to_string(r->chase_hops ? r->chase_ns / r->chase_hops : 0ull);
    const cro_pci_hop& g = r->path.hop[0];
    m[p + "link"] = link_speed(g.cur_speed) + " x" + std::to_string(g.cur_width) + " / " + link_speed(g.max_speed) + " x" +
                    std::to_string(g.max_width);
    if ((r->degraded & CRO_LINK_DEGRADED_BOTTLENECK) && r->path.bottleneck < CRO_PCI_MAX_HOPS) {
        const cro_pci_hop& b = r->path.hop[r->path.bottleneck];
        m[p + "bottleneck"] = std::string(b.bdf, strnlen(b.bdf, sizeof b.bdf)) + " " + link_speed(b.cur_speed) + " x" +
                              std::to_string(b.cur_width);
    }
    put_list(m, p + "degraded", bit_names(r->degraded, kDegraded, 4));
    if (!r->no_nvml) m[p + "replays"] = std::to_string(r->replays_after - r->replays_before);
    return emit(m, buf, cap, len);
} CRO_API_CATCH

int cro_emit_compute_annotations_json(const cro_compute_result* r, char* buf, size_t cap, size_t* len) try {
    static const char* const kLeg[CRO_COMPUTE_LEGS] = {"s8", "bf16", "e4m3", "ffma", "imad"};
    if (!r) return CRO_ERR_INVALID_ARG;
    return emit_sm_legs(*r, "cohdi.io/probe-compute-", kLeg, CRO_COMPUTE_LEGS,
                        {{CRO_COMPUTE_LEG_S8, "s8-gops"}, {CRO_COMPUTE_LEG_BF16, "bf16-gflops"}, {CRO_COMPUTE_LEG_E4M3, "e4m3-gflops"}},
                        buf, cap, len);
} CRO_API_CATCH

int cro_emit_precision_annotations_json(const cro_precision_result* r, char* buf, size_t cap, size_t* len) try {
    static const char* const kLeg[CRO_PRECISION_LEGS] = {"f64", "dfma", "tf32", "f16", "f16acc", "e5m2", "hfma2"};
    if (!r) return CRO_ERR_INVALID_ARG;
    return emit_sm_legs(*r, "cohdi.io/probe-precision-", kLeg, CRO_PRECISION_LEGS,
                        {{CRO_PRECISION_LEG_F64, "f64-gflops"}, {CRO_PRECISION_LEG_TF32, "tf32-gflops"},
                         {CRO_PRECISION_LEG_F16, "f16-gflops"}, {CRO_PRECISION_LEG_F16ACC, "f16acc-gflops"},
                         {CRO_PRECISION_LEG_E5M2, "e5m2-gflops"}},
                        buf, cap, len);
} CRO_API_CATCH

int cro_emit_scan_annotations_json(const cro_scan_report* r, char* buf, size_t cap, size_t* len) try {
    if (!r) return CRO_ERR_INVALID_ARG;
    static const char* const kHealth[4] = {"ecc-corrected", "ecc-uncorrected", "remap-pending", "remap-failure"};
    Annotations m;
    const std::string p = "cohdi.io/hbm-scan-";
    m[p + "verdict"] = r->status == CRO_OK            ? "ok"
                       : r->status == CRO_ERR_CHECKSUM ? "corrupt"
                       : r->status == CRO_ERR_CUDA     ? cuda_error(r->cuda_error)
                                                       : "error";
    m[p + "covered-bytes"] = std::to_string(r->covered_bytes);
    m[p + "free-bytes"] = std::to_string(r->free_bytes);
    m[p + "seed"] = hex16(r->seed);
    m[p + "mismatches"] = std::to_string(r->pass[0].mismatches) + "," + std::to_string(r->pass[1].mismatches);
    m[p + "granules"] = std::to_string(r->pass[0].granules) + "," + std::to_string(r->pass[1].granules);
    uint64_t ns = 0;
    for (uint64_t e : r->element_ns) ns += e;
    m[p + "gbs"] = std::to_string(ns ? (uint64_t)((unsigned __int128)r->covered_bytes * 4u / ns) : 0ull);
    put_list(m, p + "bits", bit_numbers([&](int b) { return r->pass[0].bit_flips[b] || r->pass[1].bit_flips[b]; }));
    put_list(m, p + "health", bit_names(r->health, kHealth, 4));
    const cro_hbm_health& A = r->after;
    ecc_delta(m, p, r->before, A, CRO_HBM_NVML_ECC_CORRECTED, CRO_HBM_NVML_ECC_UNCORRECTED);
    if (A.nvml & CRO_HBM_NVML_REMAP) m[p + "remapped"] = std::to_string(A.remap_corrected) + "," + std::to_string(A.remap_uncorrected);
    if (A.nvml & CRO_HBM_NVML_HISTOGRAM) m[p + "remap-histogram"] = join(A.histogram, 5);
    return emit(m, buf, cap, len);
} CRO_API_CATCH

int cro_emit_sram_annotations_json(const cro_sram_result* r, char* buf, size_t cap, size_t* len) try {
    if (!r) return CRO_ERR_INVALID_ARG;
    static const char* const kHealth[3] = {"corrected", "uncorrected", "threshold-exceeded"};
    Annotations m;
    const std::string p = "cohdi.io/probe-sram-";
    m[p + "verdict"] = r->status == CRO_OK                                                ? "ok"
                       : r->status == CRO_ERR_CHECKSUM && r->verdict == CRO_SRAM_SM   ? "sm"
                       : r->status == CRO_ERR_CHECKSUM && r->verdict == CRO_SRAM_LINK ? "link"
                       : r->status == CRO_ERR_CHECKSUM && r->verdict == CRO_SRAM_ALL  ? "all"
                       : r->status == CRO_ERR_CUDA ? cuda_error(r->cuda_error)
                                                   : "error";
    m[p + "sms"] = std::to_string(min_covered(r->legs, r->leg, CRO_SRAM_LEGS)) + "/" + std::to_string(r->sm_count);
    if (r->bad_sms) m[p + "bad-sms"] = join(r->bad_sm, std::min<uint32_t>(r->bad_sms, 16));
    if (r->bad_pairs)
        m[p + "bad-pairs"] = join(std::min<uint32_t>(r->bad_pairs, CRO_SRAM_MAX_PAIRS), [&](uint64_t j) {
            const cro_sram_pair& q = r->bad_pair[j];
            return std::to_string(q.from) + "-" + std::to_string(q.owner) + (q.direction == CRO_SRAM_DIR_READ ? ":r" : ":w");
        });
    m[p + "bytes-per-sm"] = std::to_string(r->bytes_per_sm);
    put_list(m, p + "health", bit_names(r->health, kHealth, 3));
    ecc_delta(m, p, r->before, r->after, CRO_SRAM_NVML_ECC_CORRECTED, CRO_SRAM_NVML_ECC_UNCORRECTED);
    return emit(m, buf, cap, len);
} CRO_API_CATCH

int cro_emit_l2_annotations_json(const cro_l2_result* r, char* buf, size_t cap, size_t* len) try {
    if (!r) return CRO_ERR_INVALID_ARG;
    static const char* const kHealth[6] = {"sram-corrected", "sram-uncorrected", "l2-corrected", "l2-uncorrected",
                                           "threshold-exceeded", "l2-bucket"};
    static const char* const kVerdict[5] = {"", "sm", "line", "atomic", "all"};
    Annotations m;
    const std::string p = "cohdi.io/probe-l2-";
    m[p + "verdict"] = r->status == CRO_OK                                                           ? "ok"
                       : r->status == CRO_ERR_CHECKSUM && r->verdict >= 1 && r->verdict <= CRO_L2_ALL ? kVerdict[r->verdict]
                       : r->status == CRO_ERR_CUDA ? cuda_error(r->cuda_error)
                                                   : "error";
    m[p + "sms"] = std::to_string(r->sms_covered) + "/" + std::to_string(r->sm_count);
    m[p + "bytes"] = std::to_string(r->bytes);
    m[p + "iterations"] = std::to_string(r->iterations);
    m[p + "march-gbs"] = std::to_string(r->march_ns ? r->march_bytes / r->march_ns : 0ull);
    if (r->bad_sms) m[p + "bad-sms"] = join(r->bad_sm, std::min<uint64_t>(r->bad_sms, 16));
    if (r->bad_lines) m[p + "bad-lines"] = join(r->bad_line, std::min<uint64_t>(r->bad_lines, CRO_L2_MAX_LINES));
    if (r->a1_bad) m[p + "a1-bad-counters"] = join(r->a1_bad_counter, std::min<uint64_t>(r->a1_bad, CRO_L2_MAX_COUNTERS));
    if (r->a2_bad) m[p + "a2-bad-counters"] = join(r->a2_bad_counter, std::min<uint64_t>(r->a2_bad, CRO_L2_MAX_COUNTERS));
    if (r->a2_holes) m[p + "a2-holes"] = std::to_string(r->a2_holes);
    if (r->overflow) m[p + "overflow"] = "1";
    put_list(m, p + "health", bit_names(r->health, kHealth, 6));
    return emit(m, buf, cap, len);
} CRO_API_CATCH

int cro_fm_parse_scale_up_response(const char* body, const char* resource_name, const char* res_type,
                                   const char* model, char* device_id, size_t device_id_cap,
                                   char* cdi_device_id, size_t cdi_cap, char* err_buf, size_t err_cap) try {
    if (!body) return CRO_ERR_INVALID_ARG;
    std::string dev, cdi;
    controller::Error e = controller::FMScaleUpResponseToIDs(body, S(resource_name), S(res_type), S(model), &dev, &cdi);
    if (!e.ok()) {
        copy_out(e.msg, err_buf, err_cap, nullptr);
        return CRO_ERR_PARSE;
    }
    int rc = copy_out(dev, device_id, device_id_cap, nullptr);
    if (rc) return rc;
    return copy_out(cdi, cdi_device_id, cdi_cap, nullptr);
} CRO_API_CATCH

int cro_cm_check_adding_resources(const char* machine_body, const char* existing_device_ids,
                                  const char* res_type, const char* model, char* spec_uuid, size_t spec_cap,
                                  int* device_count, char* device_id, size_t device_id_cap,
                                  char* cdi_device_id, size_t cdi_cap, char* err_buf, size_t err_cap) try {
    if (!machine_body) return CRO_ERR_INVALID_ARG;
    std::vector<std::string> existing;
    if (existing_device_ids) existing = identity::Split(existing_device_ids, "\n");
    controller::CMAddingResult r = controller::CMCheckAddingResources(machine_body, existing, S(res_type), S(model));
    if (device_count) *device_count = (int)r.deviceCount;
    int rc = copy_out(r.specUUID, spec_uuid, spec_cap, nullptr);
    if (rc) return rc;
    if ((rc = copy_out(r.deviceID, device_id, device_id_cap, nullptr))) return rc;
    if ((rc = copy_out(r.CDIDeviceID, cdi_device_id, cdi_cap, nullptr))) return rc;
    copy_out(r.err.ok() ? std::string() : r.err.msg, err_buf, err_cap, nullptr);
    return r.err.ok() ? CRO_OK : CRO_ERR_PARSE;
} CRO_API_CATCH

// ---- fabric wire codec ---------------------------------------------------------------

int cro_fabric_check_resource(const char* kind, const char* machine_body, const char* res_type, const char* model,
                              const char* device_id, char* err_buf, size_t err_cap) try {
    if (!kind || !machine_body) return CRO_ERR_INVALID_ARG;
    controller::Error e;
    if (S(kind) == "fm") e = fabric::FMCheckResource(machine_body, S(res_type), S(model), S(device_id));
    else if (S(kind) == "cm") e = fabric::CMCheckResource(machine_body, S(res_type), S(model), S(device_id));
    else return CRO_ERR_INVALID_ARG;
    copy_out(e.ok() ? std::string() : e.msg, err_buf, err_cap, nullptr);
    return e.ok() ? CRO_OK : CRO_ERR_EXEC;
} CRO_API_CATCH

int cro_fabric_get_resources(const char* kind, const char* machine_body, const char* node_name, const char* machine_uuid,
                             char* buf, size_t cap, size_t* len) try {
    if (!kind || !machine_body) return CRO_ERR_INVALID_ARG;
    std::vector<fabric::DeviceInfo> v;
    controller::Error e;
    if (S(kind) == "fm") e = fabric::FMGetResources(machine_body, S(node_name), S(machine_uuid), &v);
    else if (S(kind) == "cm") e = fabric::CMGetResources(machine_body, S(node_name), S(machine_uuid), &v);
    else return CRO_ERR_INVALID_ARG;
    if (!e.ok()) {
        copy_out(e.msg, buf, cap, len);
        return CRO_ERR_PARSE;
    }
    return copy_out(fabric::DeviceInfosToJson(v), buf, cap, len);
} CRO_API_CATCH

// ---- detach-side pre-flight -------------------------------------------------------

static int finish_err(const controller::Error& e, char* err_buf, size_t err_cap) {
    copy_out(e.ok() ? std::string() : e.msg, err_buf, err_cap, nullptr);
    return e.ok() ? CRO_OK : CRO_ERR_EXEC;
}

int cro_check_no_gpu_loads(const char* std_out, const char* std_err, const char* exec_err, const char* pod_name,
                           const char* node_name, const char* target_uuid, int driver_enabled, char* err_buf,
                           size_t err_cap) try {
    std::string uuid = S(target_uuid);
    return finish_err(detach::CheckNoGPULoadsFromOutput(S(std_out), S(std_err), exec_err, S(pod_name), S(node_name),
                                                        target_uuid ? &uuid : nullptr, driver_enabled != 0),
                      err_buf, err_cap);
} CRO_API_CATCH

int cro_check_gpu_drain_status(const char* std_out, const char* std_err, const char* exec_err, const char* node_name,
                               const char* bus_id, int* draining, char* err_buf, size_t err_cap) try {
    bool d = false;
    controller::Error e = detach::checkGPUDrainStatusFromOutput(S(std_out), S(std_err), exec_err, S(node_name), S(bus_id), &d);
    if (draining) *draining = d ? 1 : 0;
    return finish_err(e, err_buf, err_cap);
} CRO_API_CATCH

int cro_check_device_file_scan(const char* std_out, const char* std_err, const char* exec_err, int rke2, char* err_buf,
                               size_t err_cap) try {
    return finish_err(detach::CheckDeviceFileScanResult(S(std_out), S(std_err), exec_err, rke2 != 0), err_buf, err_cap);
} CRO_API_CATCH

int cro_scan_device_file_holders(const char* proc_root, const char* target, int rke2, char* buf, size_t cap, size_t* len) try {
    if (!target) return CRO_ERR_INVALID_ARG;
    return copy_out(detach::ScanDeviceFileHolders(S(proc_root), target, rke2 != 0), buf, cap, len);
} CRO_API_CATCH

// ---- in-memory cluster -----------------------------------------------------------

struct cro_sim {
    std::unique_ptr<sim::Cluster> cluster;
    std::mutex mu;
};

int cro_sim_create(cro_ctx* ctx, const char* config_json, cro_sim** out) try {
    if (!out) return CRO_ERR_INVALID_ARG;
    std::string perr;
    gojson::ValuePtr cfg = gojson::parse(config_json ? config_json : "{}", &perr);
    if (!cfg || cfg->kind != gojson::Value::Object) return CRO_ERR_PARSE;
    cro_sim* s = new cro_sim;
    s->cluster.reset(new sim::Cluster(ctx, *cfg));
    *out = s;
    return CRO_OK;
} CRO_API_CATCH
void cro_sim_destroy(cro_sim* s) { delete s; }

static int sim_json_call(cro_sim* s, const char* json, char* err_buf, size_t err_cap,
                         controller::Error (sim::Cluster::*fn)(const gojson::Value&)) {
    if (!s || !json) return CRO_ERR_INVALID_ARG;
    std::string perr;
    gojson::ValuePtr v = gojson::parse(json, &perr);
    if (!v || v->kind != gojson::Value::Object) {
        copy_out(perr, err_buf, err_cap, nullptr);
        return CRO_ERR_PARSE;
    }
    std::lock_guard<std::mutex> g(s->mu);
    controller::Error e = (s->cluster.get()->*fn)(*v);
    copy_out(e.ok() ? std::string() : e.msg, err_buf, err_cap, nullptr);
    return e.ok() ? CRO_OK : CRO_ERR_INVALID_ARG;
}
int cro_sim_apply(cro_sim* s, const char* json, char* err_buf, size_t err_cap) try {
    return sim_json_call(s, json, err_buf, err_cap, &sim::Cluster::Apply);
} CRO_API_CATCH
int cro_sim_plant(cro_sim* s, const char* json, char* err_buf, size_t err_cap) try {
    return sim_json_call(s, json, err_buf, err_cap, &sim::Cluster::Plant);
} CRO_API_CATCH
int cro_sim_delete(cro_sim* s, const char* name) try {
    if (!s || !name) return CRO_ERR_INVALID_ARG;
    std::lock_guard<std::mutex> g(s->mu);
    return s->cluster->Delete(name).ok() ? CRO_OK : CRO_ERR_INVALID_ARG;
} CRO_API_CATCH
int cro_sim_run(cro_sim* s, long long max_reconciles, char* buf, size_t cap, size_t* len) try {
    if (!s) return CRO_ERR_INVALID_ARG;
    std::lock_guard<std::mutex> g(s->mu);
    s->cluster->Run(max_reconciles > 0 ? max_reconciles : (1ll << 40));
    return copy_out(s->cluster->StatsJSON(), buf, cap, len);
} CRO_API_CATCH
int cro_sim_reconcile_request(cro_sim* s, const char* name, char* err_buf, size_t err_cap) try {
    if (!s || !name) return CRO_ERR_INVALID_ARG;
    std::lock_guard<std::mutex> g(s->mu);
    controller::Error e = s->cluster->ReconcileRequestOnce(name);
    copy_out(e.ok() ? std::string() : e.msg, err_buf, err_cap, nullptr);
    return e.ok() ? CRO_OK : CRO_ERR_EXEC;
} CRO_API_CATCH
int cro_sim_reconcile_resource(cro_sim* s, const char* name, char* err_buf, size_t err_cap) try {
    if (!s || !name) return CRO_ERR_INVALID_ARG;
    std::lock_guard<std::mutex> g(s->mu);
    controller::Error e = s->cluster->ReconcileResourceOnce(name);
    copy_out(e.ok() ? std::string() : e.msg, err_buf, err_cap, nullptr);
    return e.ok() ? CRO_OK : CRO_ERR_EXEC;
} CRO_API_CATCH
int cro_sim_sync_upstream(cro_sim* s, const char* devices_json, long long now_s, char* err_buf, size_t err_cap) try {
    if (!s || !devices_json) return CRO_ERR_INVALID_ARG;
    std::string perr;
    gojson::ValuePtr v = gojson::parse(devices_json, &perr);
    if (!v) {
        copy_out("failed to fetch data from upstream server: " + perr, err_buf, err_cap, nullptr);
        return CRO_ERR_PARSE;
    }
    std::lock_guard<std::mutex> g(s->mu);
    controller::Error e = s->cluster->SyncUpstream(*v, now_s);
    copy_out(e.ok() ? std::string() : e.msg, err_buf, err_cap, nullptr);
    return e.ok() ? CRO_OK : CRO_ERR_EXEC;
} CRO_API_CATCH
int cro_sim_dump(cro_sim* s, char* buf, size_t cap, size_t* len) try {
    if (!s) return CRO_ERR_INVALID_ARG;
    std::lock_guard<std::mutex> g(s->mu);
    return copy_out(s->cluster->DumpJSON(), buf, cap, len);
} CRO_API_CATCH

}  // extern "C"
