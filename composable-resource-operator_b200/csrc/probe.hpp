// probe.hpp — the long-lived probe context behind the C ABI.
//
// Takes the slot of utils.RunNvidiaSmi + utils.CheckGPUVisible in
// handleAttachingState (internal/controller/composableresource_controller.go:259,275;
// internal/utils/gpus.go:666-689, 54-86).  One Device per managed GPU holds the
// resident sweep buffers (2*S bytes: halves A and B), two streams, the timing
// events, the reduction scratch and the device-written result struct, so a warm
// probe is one cudaGraphLaunch and one 512-byte copy-back.
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <chrono>
#include <cstring>
#include <deque>
#include <functional>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "../../include/croprobe.h"
#include "helper_wire.h"
#include "kernels.cuh"

namespace cro {

// Everything ONE probe in flight owns.  A device has two lanes, so a second probe can be enqueued behind a running
// one (cro_probe_begin twice): its kernels start the moment the first probe's finalize kernel retires, with no host
// round trip in between — what keeps a GPU busy when one reconcile worker feeds eight of them.
struct Lane {
    ProbeParams* d_params = nullptr;   // what the graph's kernels read
    ProbeParams* h_params = nullptr;   // pinned; refreshed by the host before each launch
    SweepOut* d_out = nullptr;         // device sweep-result slots (lane 0: kSlotCount, lane 1: the first 64)
    SweepOut* h_out = nullptr;         // pinned host mirror
    cro_probe_result* d_result = nullptr;  // written by the finalize kernels; lane 0's is the all-gather send buffer
    cro_probe_result* h_result = nullptr;  // pinned copy-back target
    std::vector<cudaEvent_t> evpool;   // per-sweep timing events of the full probe (bench / tests read them)
    cudaEvent_t ev_done = nullptr;     // recorded behind the probe's last copy-back
    // the whole probe captured as one CUDA graph (timing events are external event-record nodes)
    cudaGraphExec_t graph_exec = nullptr;
    uint64_t graph_key = 0;
    size_t graph_events = 0;
    bool graph_failed = false;
    size_t events = 0;                 // timing events the in-flight / last probe recorded
    uint32_t reads = 0, copies = 0;
    bool timed = false;                // the events of the last probe on this lane are valid
    bool in_flight = false;
    std::chrono::steady_clock::time_point since{};
};

class MismatchBuffer;   // probe_internal.hpp
struct LinkState;

struct Device {
    int ordinal = -1;              // CUDA ordinal
    int index = -1;                // rank: position in the minor-sorted list
    cro_dev_info info{};
    std::mutex mu;
    cudaStream_t stream = nullptr; // every sweep
    cudaStream_t aux = nullptr;    // the closed-form generator (ALU only) runs beside the copy sweeps
    cudaEvent_t ev0 = nullptr, ev1 = nullptr, ev_fork = nullptr, ev_join = nullptr;
    Lane lanes[2];
    int lane_head = 0;                 // oldest probe in flight
    int lane_count = 0;                // probes in flight (0..2)
    int last_lane = 0;                 // lane of the most recently COLLECTED probe (cro_probe_sweep_times)
    unsigned char* region = nullptr;   // [0,S) half A, [S,2S) half B
    uint64_t sweep_bytes = 0;
    uint64_t seed_dev = 0;             // seed_base | minor
    uint64_t seed_cur = 0;             // seed of the pattern half A holds (or will hold after the next fill)
    uint64_t nonce_cur = 0;            // ... and its nonce
    uint64_t nonce_next = 0;           // nonce the next probe takes
    bool filled = false;
    // What each half (0 = A, 1 = B) holds, for the fault locator's post-mortem pass: a pattern of seed half_seed[h]
    // when half_known[h], else nothing it can compare against (never written, a peer's push, a locator retest).
    bool half_known[2] = {false, false};
    uint64_t half_seed[2] = {0, 0};
    std::unique_ptr<MismatchBuffer> locate;   // fault locator (ctx_locate), made at its first call
    std::unique_ptr<LinkState> link;       // host link probe (ctx_probe_host_link), made at its first call
    uint64_t link_calls = 0;               // k of the next host link probe call: its seeds
    uint64_t compute_calls = 0;            // k of the next compute probe call (ctx_probe_compute): its operand seed
    uint64_t sram_calls = 0;               // k of the next SRAM probe call (ctx_probe_sram): its seeds
    uint64_t l2_calls = 0;                 // k of the next L2 probe call (ctx_probe_l2): its seeds
    uint64_t precision_calls = 0;          // k of the next precision probe call (ctx_probe_precision): its operand seed
    uint64_t sparse_calls = 0;             // k of the next sparse probe call (ctx_probe_sparse): its operand seed
    uint64_t regfile_calls = 0;            // k of the next register-file probe call (ctx_probe_regfile): its seeds
    uint64_t warpmma_calls = 0;            // k of the next warp-MMA probe call (ctx_probe_warpmma): its operand seed
    uint64_t xlane_calls = 0;              // k of the next cross-lane probe call (ctx_probe_xlane): its seeds
    uint64_t alu_calls = 0;                // k of the next ALU probe call (ctx_probe_alu): its table's seed
    uint64_t barrier_calls = 0;            // k of the next barrier probe call (ctx_probe_barrier): its table's seed
    KernelPlan plan{};
    SweepScratch scratch{}, scratch_aux{}, scratch_pfx{};   // main stream / closed form / p2p prefix closed form
    // lane 0's buffers under their old names: the synchronous probe, the single sweeps and cro_probe_all use lane 0
    SweepOut*& d_out = lanes[0].d_out;
    SweepOut*& h_out = lanes[0].h_out;
    cro_probe_result*& d_result = lanes[0].d_result;
    cro_probe_result*& h_result = lanes[0].h_result;
    cro_probe_result* d_tmpl = nullptr;    // identity + options, staged by the host
    cro_probe_result* d_gather = nullptr;  // all-gather receive buffer (world entries)
    cro_probe_result* h_gather = nullptr;  // pinned, CRO_MAX_DEVICES entries
    cro_probe_result tmpl{};               // host copy of d_tmpl
    // NVLink latency: tables[j] is the permutation device j chases THROUGH this device's memory
    std::vector<unsigned long long*> d_chase_tables;
    std::vector<unsigned> chase_expect;    // where this device's chase into peer j must end (hops of the last build)
    unsigned chase_hops_built = 0;
    unsigned long long* d_chase_out = nullptr;
    unsigned long long* h_chase_out = nullptr;   // pinned, 2 * CRO_MAX_DEVICES
    std::vector<cudaEvent_t> ev_push_done, ev_reread_done;   // one per NVLink round
    cudaEvent_t ev_hbm_done = nullptr, ev_aux_done = nullptr, ev_chase_ready = nullptr;
    // asynchronous probes (ctx_probe_begin / ctx_probe_end): results drained off the stream but not yet collected
    struct Collected { cro_probe_result r; int rc; std::chrono::steady_clock::time_point at; };
    std::deque<Collected> done;
    unsigned sm_clock_mhz = 0, mem_clock_mhz = 0;
    uint32_t ecc_uncorrected = 0;      // NVML count cached at init / full-box probe / failed probe
    std::chrono::steady_clock::time_point ecc_at{};   // last NVML read by cro_probe_all
    cro_probe_result last{};           // the most recent collected result (cro_metrics_text)
    bool have_last = false;

    Device() = default;
    Device(const Device&) = delete;
    Device& operator=(const Device&) = delete;
    // Releases every CUDA object this device owns (probe.cu; the probes' own state goes with its owners, after the
    // streams are synchronised).  Runs for half-built devices too, so a cro_probe_init that fails midway (OOM on the
    // sweep region) leaks nothing.
    ~Device();
};

// Phases of the most recent cro_probe_all, host wall clock + device windows (bench "fullbox").
struct FullBoxTimes {
    uint64_t enqueue_ns = 0;       // host time to enqueue everything
    uint64_t wall_ns = 0;          // host wall clock of the whole call
    uint64_t hbm_ns = 0;           // max over devices of the HBM probe (device timers)
    uint64_t p2p_ns = 0;           // first NVLink kernel start .. last NVLink kernel end (device timers, max over devices)
    uint64_t chase_ns = 0;         // max chase duration
    uint64_t gather_ns = 0;        // all-gather, CUDA events on rank 0's stream
    uint32_t rounds = 0;
    uint32_t host_syncs = 0;       // stream synchronisations the call performed
    uint32_t gather = 0;           // CRO_GATHER_*
};

}  // namespace cro

struct cro_ctx {
    cro_opts opts{};
    std::vector<std::unique_ptr<cro::Device>> devs;   // minor-sorted
    std::atomic<uint64_t> launches{0};
    // gauges / counters behind cro_metrics_text (the operator's Prometheus registry, cmd/main.go:66,119-125)
    std::atomic<uint64_t> m_probes{0}, m_probe_failures{0}, m_fullbox{0}, m_helper_probes{0}, m_helper_failures{0};
    // helper calls that took a seed base so far: the seed base of each (helper_seed_base)
    std::atomic<uint64_t> helper_seeds{0};
    std::mutex err_mu;
    std::string last_error;
    std::mutex all_mu;                 // serialises cro_probe_all
    void* nccl_lib = nullptr;
    std::vector<void*> nccl_comms;     // ncclComm_t per device
    bool nccl_ready = false;
    bool peers_enabled = false;
    bool nvtx = true;
    // the CRO_* knobs as validated by cro_probe_init: everything the context plans and probes with reads these
    cro::env::Values knobs;
    std::string proc_root = "/proc";   // where the node's /proc is mounted (tests point it at a fake tree)
    std::string sys_root = "/sys";     // where the node's sysfs is mounted (CRO_SYS_ROOT): the host link probe's path
    // the node's inventory as of the last enumeration (inventory.hpp)
    std::mutex inv_mu;
    std::string inv_key;               // uuid/minor set the cached list was built from
    std::vector<cro_dev_info> inv;
    bool inv_valid = false;
    bool inv_refreshing = false;       // a background full re-read is under way
    std::thread inv_thread;
    std::chrono::steady_clock::time_point inv_full_at{};   // last time the `information` files were read
    std::chrono::steady_clock::time_point inv_nvml_at{};   // last NVML re-initialisation (rate limit when /proc is absent)
    std::atomic<uint64_t> inv_rescans{0};                  // times the inventory had to be rebuilt
    cro::FullBoxTimes fullbox{};
    // NCCL entry points, resolved once
    int (*ncclCommInitAll)(void**, int, const int*) = nullptr;
    int (*ncclGroupStart)() = nullptr;
    int (*ncclGroupEnd)() = nullptr;
    int (*ncclAllGather)(const void*, void*, size_t, int, void*, cudaStream_t) = nullptr;
    const char* (*ncclGetErrorString)(int) = nullptr;

    void set_error(const std::string& m) {
        std::lock_guard<std::mutex> g(err_mu);
        last_error = m;
    }
    // a context that dies during cro_probe_init hands its error text to the calling thread
    // (cro_last_error(NULL, ...)); defined in probe.cu
    ~cro_ctx();
};

namespace cro {

const std::string& last_init_error();   // calling thread's last failed ctx_create (or exception stopped at the C ABI)
void set_thread_error(const std::string& m) noexcept;
int ctx_create(const cro_opts* o, cro_ctx** out);
void ctx_destroy(cro_ctx* c);
int ctx_probe_device(cro_ctx* c, int idx, cro_probe_result* out);
int ctx_probe_all(cro_ctx* c, cro_probe_result* out, int cap, int* n);
// cro_selftest_p2p_plan: the plan ctx_probe_all walks, from caller-given sizes, access rows and options (fullbox.cu).
int selftest_p2p_plan(uint32_t n, const uint64_t* sweep_bytes, uint64_t p2p_bytes, const uint8_t* access, uint32_t flags,
                      uint32_t unidir, uint32_t write_variant, cro_p2p_plan* out);
int ctx_probe_begin(cro_ctx* c, int idx);
int ctx_probe_end(cro_ctx* c, int idx, cro_probe_result* out);
int ctx_probe_poll(cro_ctx* c, int idx);
int ctx_probe_wait(cro_ctx* c, int idx);
int ctx_probe_depth(cro_ctx* c, int idx);
std::string ctx_metrics_text(cro_ctx* c);
int ctx_sweep_times(cro_ctx* c, int idx, cro_sweep_time* out, int cap, int* n);
// Fresh inventory of the node merged with the context's own devices (inventory.hpp).
// force: re-read every `information` file even if the registry's listing looks unchanged (done by itself once a
// second, and by the callers whenever a UUID they were told about is NOT in the list they got).
int ctx_inventory(cro_ctx* c, std::vector<cro_dev_info>* out, bool force = false);
// Probe by UUID: in-process device, helper process for one attached after init, CRO_ERR_NO_DEVICE when not on the node.
int ctx_probe_uuid(cro_ctx* c, const char* uuid, cro_probe_result* out);
// The node's inventory entry of a UUID (looked up twice, the second time with a forced re-read); CRO_ERR_NO_DEVICE with
// the error text set when the node does not list it.
int find_on_node(cro_ctx* c, const std::string& uuid, cro_dev_info* hit);
int ctx_p2p_detail(cro_ctx* c, int idx, int peer, cro_p2p_detail* out);

// single sweeps (each takes the device mutex)
int ctx_fill(cro_ctx* c, int idx, uint32_t iters, cro_sweep_result* out);
int ctx_read(cro_ctx* c, int idx, uint32_t variant, uint32_t iters, bool dst_half, cro_sweep_result* out);
int ctx_copy(cro_ctx* c, int idx, uint32_t variant, uint32_t iters, cro_sweep_result* out);
int ctx_expected(cro_ctx* c, int idx, cro_sweep_result* out);
int ctx_inject(cro_ctx* c, int idx, uint64_t word, uint64_t mask);
int ctx_read_words(cro_ctx* c, int idx, uint64_t first, uint64_t n, uint64_t* out);

// Fault locator (include/croprobe.h, cro_locate_faults): *words gets every located word, sorted by region index.
int ctx_locate(cro_ctx* c, int idx, const cro_locate_opts& o, cro_fault_report* rep, std::vector<cro_fault_word>* words);
// CRO_FAULTS_* of a report, from its per-pass mismatch counts.
uint32_t fault_verdict(const cro_fault_report& r);
// cro_selftest_locate_collect: the locator's report from the caller's counters, records, bitmaps and slots, as
// ctx_locate makes it from its kernels' (CRO_ERR_INVALID_ARG when the compared halves have more than
// CRO_LOCATE_PASSES distinct seeds).
int selftest_locate_collect(uint64_t sweep_bytes, const cro_locate_pass* passes, uint32_t n_passes, const cro_locate_counters* ctr,
                            const cro_locate_record* records, const uint64_t* granules, uint64_t granule_words,
                            const cro_sweep_slot* slots, cro_fault_report* rep, std::vector<cro_fault_word>* words);

// Host link probe (include/croprobe.h, cro_probe_host_link / cro_probe_host_link_uuid): *faults gets every recorded
// mismatch, by check, then index.  The uuid form runs `croprobe-cli link-raw` and asks it for at most cap faults;
// *helper_ns is the helper's spawn to exit.
int ctx_probe_host_link(cro_ctx* c, int idx, const cro_link_opts& o, cro_link_result* r, std::vector<cro_link_fault>* faults);
int ctx_probe_host_link_uuid(cro_ctx* c, const char* uuid, const cro_link_opts& o, int deadline_ms, cro_link_result* r,
                             std::vector<cro_link_fault>* faults, int cap, uint64_t* helper_ns);
// cro_selftest_link_classify: the probe's takes and classification of the caller's counters, records, host words,
// slots and chase output, as ctx_probe_host_link makes them from its kernels'.
int selftest_link_classify(uint64_t bytes, const uint64_t* seeds, uint32_t minor, uint32_t hops, const cro_locate_counters* ctr,
                           const cro_locate_record* records, const uint64_t* host, const cro_sweep_slot* slots,
                           const uint64_t* chase_out, cro_link_result* r, std::vector<cro_link_fault>* faults);

// SM compute probe (include/croprobe.h, cro_probe_compute / cro_probe_compute_uuid): *sms gets one entry per SM seen, by
// SM id; *faults every recorded element, by (leg, smid, row, col).  The uuid form runs `croprobe-cli compute-raw` and
// asks it for at most cap faults; *helper_ns is the helper's spawn to exit.
int ctx_probe_compute(cro_ctx* c, int idx, const cro_compute_opts& o, cro_compute_result* r, std::vector<cro_compute_sm>* sms,
                      std::vector<cro_compute_fault>* faults);
int ctx_probe_compute_uuid(cro_ctx* c, const char* uuid, const cro_compute_opts& o, int deadline_ms, cro_compute_result* r,
                           std::vector<cro_compute_sm>* sms, std::vector<cro_compute_fault>* faults, int cap, uint64_t* helper_ns);

// SM precision probe (include/croprobe.h, cro_probe_precision / cro_probe_precision_uuid, precision_probe.cu): as the
// compute probe's two forms; the uuid form runs `croprobe-cli precision-raw`.
int ctx_probe_precision(cro_ctx* c, int idx, const cro_precision_opts& o, cro_precision_result* r,
                        std::vector<cro_precision_sm>* sms, std::vector<cro_precision_fault>* faults);
int ctx_probe_precision_uuid(cro_ctx* c, const char* uuid, const cro_precision_opts& o, int deadline_ms, cro_precision_result* r,
                             std::vector<cro_precision_sm>* sms, std::vector<cro_precision_fault>* faults, int cap,
                             uint64_t* helper_ns);
// cro_selftest_sm_legs_classify: each probe's classification of the caller's rounds and records (sm_legs.hpp).
int classify_compute(uint32_t legs, const uint32_t* iterations, uint32_t grid, uint64_t k, const uint32_t* rounds,
                     const cro_sm_cta* ctas, const uint64_t* sm_bits, const uint64_t* claims, const cro_compute_fault* records,
                     cro_compute_result* r, std::vector<cro_compute_sm>* sms, std::vector<cro_compute_fault>* faults);
int classify_precision(uint32_t legs, const uint32_t* iterations, uint32_t grid, uint64_t k, const uint32_t* rounds,
                       const cro_sm_cta* ctas, const uint64_t* sm_bits, const uint64_t* claims, const cro_precision_fault* records,
                       cro_precision_result* r, std::vector<cro_precision_sm>* sms, std::vector<cro_precision_fault>* faults);
// SM sparse probe (include/croprobe.h, cro_probe_sparse / cro_probe_sparse_uuid, sparse_probe.cu): as the compute
// probe's two forms; the uuid form runs `croprobe-cli sparse-raw`.
int ctx_probe_sparse(cro_ctx* c, int idx, const cro_sparse_opts& o, cro_sparse_result* r, std::vector<cro_sparse_sm>* sms,
                     std::vector<cro_sparse_fault>* faults);
int ctx_probe_sparse_uuid(cro_ctx* c, const char* uuid, const cro_sparse_opts& o, int deadline_ms, cro_sparse_result* r,
                          std::vector<cro_sparse_sm>* sms, std::vector<cro_sparse_fault>* faults, int cap, uint64_t* helper_ns);
int classify_sparse(uint32_t legs, const uint32_t* iterations, uint32_t grid, uint64_t k, const uint32_t* rounds,
                    const cro_sm_cta* ctas, const uint64_t* sm_bits, const uint64_t* claims, const cro_sparse_fault* records,
                    cro_sparse_result* r, std::vector<cro_sparse_sm>* sms, std::vector<cro_sparse_fault>* faults);
namespace sparse {
// The answer tile of the operands of `seed` (include/croprobe.h): answer CRO_SPARSE_ANSWER_*, M x N int32 values,
// row-major.  CRO_ERR_INVALID_ARG for another answer.
int Expected(int answer, uint64_t seed, int32_t* out);
}  // namespace sparse
namespace precision {
// The answer tile of the operands of `seed` (include/croprobe.h): answer CRO_PRECISION_ANSWER_*, M x N int64 values,
// row-major.  CRO_ERR_INVALID_ARG for another answer.
int Expected(int answer, uint64_t seed, int64_t* out);
// The sum over every element e of an answer's tile of canon(value in its legs' type) * (2e + 1) (mod 2^64).
uint64_t TileFold(int answer, const int64_t* tile);
}  // namespace precision
// SM warp-MMA probe (include/croprobe.h, cro_probe_warpmma / cro_probe_warpmma_uuid, warpmma_probe.cu): as the compute
// probe's two forms; the uuid form runs `croprobe-cli warpmma-raw`.
int ctx_probe_warpmma(cro_ctx* c, int idx, const cro_warpmma_opts& o, cro_warpmma_result* r, std::vector<cro_warpmma_sm>* sms,
                      std::vector<cro_warpmma_fault>* faults);
int ctx_probe_warpmma_uuid(cro_ctx* c, const char* uuid, const cro_warpmma_opts& o, int deadline_ms, cro_warpmma_result* r,
                           std::vector<cro_warpmma_sm>* sms, std::vector<cro_warpmma_fault>* faults, int cap, uint64_t* helper_ns);
int classify_warpmma(uint32_t legs, const uint32_t* iterations, uint32_t grid, uint64_t k, const uint32_t* rounds,
                     const cro_sm_cta* ctas, const uint64_t* sm_bits, const uint64_t* claims, const cro_warpmma_fault* records,
                     cro_warpmma_result* r, std::vector<cro_warpmma_sm>* sms, std::vector<cro_warpmma_fault>* faults);
namespace warpmma {
// The answer tile of the operands of `seed` (include/croprobe.h): answer CRO_WARPMMA_ANSWER_*, M x N int32 values,
// row-major.  CRO_ERR_INVALID_ARG for another answer.
int Expected(int answer, uint64_t seed, int32_t* out);
}  // namespace warpmma

// The helper run behind the uuid forms of the host link, compute, precision, sparse, warp-MMA, scan, SRAM and L2 probes and the
// health check.  Bad options are refused by the caller first.  With a context, the node must list the GPU
// (CRO_ERR_NO_DEVICE otherwise) and a GPU that is also an in-process device is held under its device guard while the
// helper runs.  Then `croprobe-cli args...` runs as inventory::RunHelperRaw runs it ("<what> for <uuid> ..." in its
// errors): its stdout, head bytes and then tail(out, size) more, at most max_tail, lands in *got.  *helper_ns: spawn to
// exit.  CRO_OK means *got is a whole frame; the result's status, its first field, is the call's status then, and one
// other than CRO_OK or CRO_ERR_CHECKSUM is an error too.  An error goes to the context, or to the calling thread
// without one.
int run_probe_helper(cro_ctx* c, const std::string& uuid, const std::string& what, const char* range,
                     const std::vector<std::string>& args, int deadline_ms, size_t head, size_t max_tail,
                     const std::function<uint64_t(const unsigned char* out, size_t size)>& tail, std::string* got,
                     uint64_t* helper_ns);
// One check's frame (helper_wire.h) at f, size bytes from there on: the bytes it takes after its result, or ~0 when it
// is cut short, lists more per-SM entries than its block holds or more records than follow.  Its result, records and
// per-SM entries go to whichever of r, recs and sms are given.
template <class Rec = unsigned char, class Sm = unsigned char>
uint64_t read_frame(const cro_wire_frame& w, const unsigned char* f, size_t size, void* r = nullptr,
                    std::vector<Rec>* recs = nullptr, std::vector<Sm>* sms = nullptr) {
    const size_t head = cro_wire_head(&w);
    if (size < head) return ~0ull;
    uint64_t n_sms = 0, n = 0;
    memcpy(&n_sms, f + w.n_sms_at, w.n_sms_width);
    memcpy(&n, f + w.n_at, w.n_width);
    if (n_sms > w.max_sms || n > (size - head) / w.rec) return ~0ull;
    if (r) memcpy(r, f, w.result);
    if (sms) {
        const Sm* s = reinterpret_cast<const Sm*>(f + head - (size_t)w.max_sms * w.sm);
        sms->assign(s, s + n_sms);
    }
    if (recs) {
        const Rec* x = reinterpret_cast<const Rec*>(f + head);
        recs->assign(x, x + n);
    }
    return head - w.result + n * w.rec;
}
// The cro_opts.seed_base a helper of the link, compute, precision and L2 forms gets: with a context, its seed_base +
// (h << 8) for the context's h-th such call (h from 1, so no helper repeats the context's own seeds); without one, a
// clock-derived base.  The low byte is clear either way: the helper ORs the minor into it.
uint64_t helper_seed_base(cro_ctx* c);
// Sets an error text on the context, or on the calling thread without one.
void set_call_error(cro_ctx* c, const std::string& m);
// w's option fields of the options at o as argv, then the record cap.
void append_wire_args(const cro_wire& w, const void* o, int cap, std::vector<std::string>* args);
// The helper form of one check: `croprobe-cli <w.cmd> <uuid> [<seed base>] <options> <cap>` (a fresh seed base,
// helper_seed_base, when w is seeded) through run_probe_helper, its frame unpacked into *r, *recs and *sms.  Returns
// run_probe_helper's code; *r is blank but for its status when that is not CRO_OK.
template <class Result, class Rec, class Sm = unsigned char>
int run_check_helper(cro_ctx* c, const cro_wire& w, const std::string& uuid, const std::string& what, const char* range,
                     const void* opts, int cap, int deadline_ms, uint64_t* helper_ns, Result* r, std::vector<Rec>* recs,
                     std::vector<Sm>* sms = nullptr) {
    std::vector<std::string> args = {w.cmd, uuid};
    if (w.seeded) args.push_back(std::to_string(helper_seed_base(c)));
    append_wire_args(w, opts, cap, &args);
    std::string got;
    const int rc = run_probe_helper(c, uuid, what, range, args, deadline_ms, w.frame.result,
                                    cro_wire_head(&w.frame) - w.frame.result + (size_t)cap * w.frame.rec,
                                    [&w](const unsigned char* f, size_t size) { return read_frame(w.frame, f, size); }, &got,
                                    helper_ns);
    if (rc != CRO_OK) {
        r->status = rc;
        return rc;
    }
    read_frame(w.frame, reinterpret_cast<const unsigned char*>(got.data()), got.size(), r, recs, sms);
    return CRO_OK;
}

// Whole-HBM scan (include/croprobe.h, cro_scan_hbm / cro_scan_hbm_uuid, hbm_scan.cu): *words gets every recorded word,
// merged by scan index.  The uuid form runs `croprobe-cli scan-raw` and asks it for at most cap words.
int ctx_scan_hbm(cro_ctx* c, int idx, const cro_scan_opts& o, cro_scan_report* rep, std::vector<cro_fault_word>* words);
int ctx_scan_hbm_uuid(cro_ctx* c, const char* uuid, const cro_scan_opts& o, cro_scan_report* rep, std::vector<cro_fault_word>* words,
                      int cap);
// CRO_SCAN_HEALTH_* of the NVML reads before E0 and after E3.
uint32_t scan_health(const cro_hbm_health& before, const cro_hbm_health& after);
// cro_selftest_scan_collect: the scan's passes, words and status from the caller's counters, records, bitmaps and
// slots, as ctx_scan_hbm makes them from its kernels'.  *rep gives n_chunks, elements_done and the chunks' word0 and
// bytes.
int selftest_scan_collect(int32_t cuda_error, const cro_locate_counters* ctr, const cro_locate_record* records,
                          const uint64_t* granules, uint64_t granule_words, const cro_sweep_slot* slots, cro_scan_report* rep,
                          std::vector<cro_fault_word>* words);

// Each check's argument check, as its calls make it: why the options are refused ("" when they pass).  The link
// check's is its helper form's (L against a region of L); the L2 check's is l2_check_args.
std::string compute_opts_error(const cro_compute_opts& o);
std::string precision_opts_error(const cro_precision_opts& o);
std::string sram_opts_error(const cro_sram_opts& o);
std::string link_helper_opts_error(const cro_link_opts& o);
std::string scan_opts_error(const cro_scan_opts& o);

// SRAM probe (include/croprobe.h, cro_probe_sram / cro_probe_sram_uuid, sram_probe.cu): *sms gets one entry per SM
// seen, by SM id; *faults every recorded word, by (leg, element, smid, iteration, word).  The uuid form runs
// `croprobe-cli sram-raw` and asks it for at most cap words.
int ctx_probe_sram(cro_ctx* c, int idx, const cro_sram_opts& o, cro_sram_result* r, std::vector<cro_sram_sm>* sms,
                   std::vector<cro_sram_fault>* faults);
int ctx_probe_sram_uuid(cro_ctx* c, const char* uuid, const cro_sram_opts& o, cro_sram_result* r, std::vector<cro_sram_sm>* sms,
                        std::vector<cro_sram_fault>* faults, int cap);
// CRO_SRAM_HEALTH_* of the NVML reads before the first leg and after the last.
uint32_t sram_health(const cro_sram_health& before, const cro_sram_health& after);
// cro_selftest_sram_classify: the probe's classification of the caller's rounds and records, as ctx_probe_sram makes it.
int classify_sram(uint32_t legs, uint32_t iterations, uint32_t n_words, uint64_t seed, uint32_t cluster, uint32_t sm_count,
                  uint32_t net_grid, uint64_t k, const uint32_t* rounds, const cro_sram_cta* ctas, const uint64_t* claims,
                  const cro_sram_record* records, cro_sram_result* r, std::vector<cro_sram_sm>* sms,
                  std::vector<cro_sram_fault>* faults);

// Register-file probe (include/croprobe.h, cro_probe_regfile / cro_probe_regfile_uuid, regfile_probe.cu): *sms gets one
// entry per SM seen, by SM id; *faults every recorded slot, by (smid, iteration, element, warp, lane, slot).  The uuid
// form runs `croprobe-cli regfile-raw` with a fresh seed base and asks it for at most cap slots.
std::string regfile_opts_error(const cro_regfile_opts& o);
int ctx_probe_regfile(cro_ctx* c, int idx, const cro_regfile_opts& o, cro_regfile_result* r, std::vector<cro_regfile_sm>* sms,
                      std::vector<cro_regfile_fault>* faults);
int ctx_probe_regfile_uuid(cro_ctx* c, const char* uuid, const cro_regfile_opts& o, cro_regfile_result* r,
                           std::vector<cro_regfile_sm>* sms, std::vector<cro_regfile_fault>* faults, int cap);
// cro_selftest_regfile_classify: the probe's classification of the caller's rounds and records, as ctx_probe_regfile
// makes it.
int classify_regfile(uint32_t iterations, uint64_t seed, uint32_t sm_count, uint64_t k, uint32_t rounds,
                     const cro_regfile_cta* ctas, uint64_t claims, const cro_regfile_fault* records, cro_regfile_result* r,
                     std::vector<cro_regfile_sm>* sms, std::vector<cro_regfile_fault>* faults);

// Cross-lane probe (include/croprobe.h, cro_probe_xlane / cro_probe_xlane_uuid, xlane_probe.cu): *sms gets one entry
// per SM seen, by SM id; *faults the records, by (leg, smid, iteration, op, warp, lane), at most CRO_XLANE_RECORDS.  The
// uuid form runs `croprobe-cli xlane-raw` with a fresh seed base and asks it for at most cap records.
std::string xlane_opts_error(const cro_xlane_opts& o);
int ctx_probe_xlane(cro_ctx* c, int idx, const cro_xlane_opts& o, cro_xlane_result* r, std::vector<cro_xlane_sm>* sms,
                    std::vector<cro_xlane_fault>* faults);
int ctx_probe_xlane_uuid(cro_ctx* c, const char* uuid, const cro_xlane_opts& o, cro_xlane_result* r,
                         std::vector<cro_xlane_sm>* sms, std::vector<cro_xlane_fault>* faults, int cap);
// cro_xlane_expected and cro_selftest_xlane_classify.
void xlane_expected(unsigned leg, uint64_t seed, uint32_t iteration, unsigned warp, uint64_t* out);
int classify_xlane(uint32_t legs, uint32_t iterations, uint64_t seed, uint32_t sm_count, uint64_t k, uint32_t rounds,
                   const cro_xlane_cta* ctas, const cro_xlane_thread* threads, const cro_xlane_fault* records,
                   cro_xlane_result* r, std::vector<cro_xlane_sm>* sms, std::vector<cro_xlane_fault>* faults);

// ALU probe (include/croprobe.h, cro_probe_alu / cro_probe_alu_uuid, alu_probe.cu): *sms gets one entry per SM seen,
// by SM id; *faults the records, by (leg, smid, iteration, op, warp, lane), at most CRO_ALU_RECORDS.  The uuid form
// runs `croprobe-cli alu-raw` with a fresh seed base and asks it for at most cap records.
std::string alu_opts_error(const cro_alu_opts& o);
int ctx_probe_alu(cro_ctx* c, int idx, const cro_alu_opts& o, cro_alu_result* r, std::vector<cro_alu_sm>* sms,
                  std::vector<cro_alu_fault>* faults);
int ctx_probe_alu_uuid(cro_ctx* c, const char* uuid, const cro_alu_opts& o, cro_alu_result* r, std::vector<cro_alu_sm>* sms,
                       std::vector<cro_alu_fault>* faults, int cap);
// cro_alu_expected and cro_selftest_alu_classify.
void alu_expected(unsigned leg, uint64_t seed, unsigned warp, cro_alu_record* out);
int classify_alu(uint32_t legs, uint32_t iterations, uint64_t seed, uint32_t sm_count, uint64_t k, uint32_t rounds,
                 const cro_alu_cta* ctas, const cro_alu_thread* threads, const cro_alu_fault* records, cro_alu_result* r,
                 std::vector<cro_alu_sm>* sms, std::vector<cro_alu_fault>* faults);

// Barrier probe (include/croprobe.h, cro_probe_barrier / cro_probe_barrier_uuid, barrier_probe.cu): *sms gets one entry
// per SM seen, by SM id; *faults the records, by (leg, smid, iteration, op, warp, lane), at most CRO_BARRIER_RECORDS.
// The uuid form runs `croprobe-cli barrier-raw` with a fresh seed base and asks it for at most cap records.
std::string barrier_opts_error(const cro_barrier_opts& o);
int ctx_probe_barrier(cro_ctx* c, int idx, const cro_barrier_opts& o, cro_barrier_result* r, std::vector<cro_barrier_sm>* sms,
                      std::vector<cro_barrier_fault>* faults);
int ctx_probe_barrier_uuid(cro_ctx* c, const char* uuid, const cro_barrier_opts& o, cro_barrier_result* r,
                           std::vector<cro_barrier_sm>* sms, std::vector<cro_barrier_fault>* faults, int cap);
// cro_barrier_expected and cro_selftest_barrier_classify.
void barrier_expected(unsigned leg, uint64_t seed, uint32_t cluster, cro_barrier_row* rows, uint64_t* words);
int classify_barrier(uint32_t legs, uint32_t iterations, uint64_t seed, uint32_t cluster, uint32_t sm_count, uint64_t k, uint32_t rounds,
                     const cro_barrier_cta* ctas, const cro_barrier_thread* threads, const cro_barrier_fault* records,
                     cro_barrier_result* r, std::vector<cro_barrier_sm>* sms, std::vector<cro_barrier_fault>* faults);

// L2 probe (include/croprobe.h, cro_probe_l2, l2_probe.cu): *sms gets one entry per SM seen, by SM id; *faults every
// recorded word, by (word, iteration, element, smid).
int ctx_probe_l2(cro_ctx* c, int idx, const cro_l2_opts& o, cro_l2_result* r, std::vector<cro_l2_sm>* sms,
                 std::vector<cro_l2_fault>* faults);
// The uuid form runs `croprobe-cli l2-raw` with a fresh seed base (helper_seed_base) and asks it for at most cap words.
int ctx_probe_l2_uuid(cro_ctx* c, const char* uuid, const cro_l2_opts& o, cro_l2_result* r, std::vector<cro_l2_sm>* sms,
                      std::vector<cro_l2_fault>* faults, int cap);
// The options with their defaults filled in.
struct L2Settings {
    uint64_t bytes;
    uint32_t iterations, a1, a2;
};
// Checks a call's options against a device whose L2 holds l2_size bytes (0: not known here, W's upper bound is left to
// the helper), filling *p; false with *why set when they are refused.  Both forms call it before anything is launched
// or spawned; `helper` says which (only the helper form takes a deadline).
bool l2_check_args(const cro_l2_opts& o, uint64_t l2_size, bool helper, L2Settings* p, std::string* why);
// The rotation step of G CTAs (0: G < 5, no step puts M1 .. M5 of a word on five CTAs).
uint32_t l2_delta(uint32_t G);
// CRO_L2_HEALTH_* of the NVML reads before and after the call.
uint32_t l2_health(const cro_l2_health& before, const cro_l2_health& after);
// The verdict, bad SMs and lines, marks and line flags of a call's counts and records (cro_selftest_l2_classify).
void l2_classify(cro_l2_result* r, cro_l2_sm* sms, size_t n_sms, cro_l2_fault* faults, size_t n);

// Health check (include/croprobe.h, cro_check_health / cro_check_health_uuid, health.cpp): every record each check
// found, as its own call lists them.
struct HealthRecords {
    std::vector<cro_compute_sm> compute_sms;
    std::vector<cro_compute_fault> compute_faults;
    std::vector<cro_precision_sm> precision_sms;
    std::vector<cro_precision_fault> precision_faults;
    std::vector<cro_sram_sm> sram_sms;
    std::vector<cro_sram_fault> sram_faults;
    std::vector<cro_l2_sm> l2_sms;
    std::vector<cro_l2_fault> l2_faults;
    std::vector<cro_link_fault> link_faults;
    std::vector<cro_fault_word> scan_words;
};
// The record caps the helper is asked for, in run order: compute, precision, SRAM, L2 faults, link faults, scan words.
struct HealthCaps {
    int faults[CRO_HEALTH_CHECKS];
};
// The stop and status rules (cro_selftest_health_classify): checks is the selection, status[0 .. n) what the first n
// checks to run returned.  Writes r's status, checks, ran, failed, errored, not_run and check_status; returns the index
// of the check to run next, CRO_HEALTH_CHECKS when none is left, or -1 when the rules let fewer than n checks run.
int health_step(uint32_t checks, const int32_t* status, int n, cro_health_result* r);
// Why a health call's options are refused before anything runs ("" when they pass): check bits, sub-option deadlines
// and each selected check's own argument check.
std::string health_opts_error(const cro_health_opts& o);
int ctx_check_health(cro_ctx* c, int idx, const cro_health_opts& o, cro_health_result* r, HealthRecords* rec);
// The uuid form runs `croprobe-cli health-raw` with a fresh seed base and asks it for at most caps records per list.
int ctx_check_health_uuid(cro_ctx* c, const char* uuid, const cro_health_opts& o, int deadline_ms, const HealthCaps& caps,
                          cro_health_result* r, HealthRecords* rec, uint64_t* helper_ns);

// test hooks (include/croprobe.h, cro_selftest_*): the verdict kernels and the chase on caller-given inputs
int ctx_selftest_probe_finalize(cro_ctx* c, int idx, const cro_probe_result* tmpl, const cro_sweep_slot* slots,
                                const ProbeParams& pp, uint64_t sweep_bytes, uint32_t R, uint32_t C, uint32_t rv,
                                uint32_t cv, cro_probe_result* out);
int ctx_selftest_p2p_finalize(cro_ctx* c, int idx, cro_probe_result* result, const cro_sweep_slot* slots,
                              const cro_sweep_slot* const* peer_slots, const uint64_t* peer_stamp, const uint64_t* chase_out,
                              const uint32_t* chase_expect, uint32_t n, uint32_t self, uint32_t hops, uint32_t have_push,
                              uint32_t push_folded, uint64_t p2p_bytes, uint64_t stamp);
int ctx_selftest_chase(cro_ctx* c, int idx, const int32_t* minor_src, const int32_t* minor_dst, uint32_t n, uint32_t hops,
                       uint64_t* out);
// One sweep kernel on a guarded buffer of the hook's own (cro_selftest_sweep).
int ctx_selftest_sweep(cro_ctx* c, int idx, const cro_selftest_sweep_opts* o, cro_selftest_sweep_out* out, void* buf,
                       uint64_t cap_bytes, cro_fault_word* words, int cap, int* n_words);

// CRO_READ_AUTO / CRO_COPY_AUTO resolved with a context's knobs (CRO_READ_VARIANT, CRO_COPY_VARIANT).
uint32_t resolve_read_variant(uint32_t v, uint64_t bytes, const env::Values& knobs);
uint32_t resolve_copy_variant(uint32_t v, const env::Values& knobs);

// Host restatement of the latency permutation of one directed pair (Sattolo cycle over kChaseSlots slots,
// mt19937_64 seeded with minor_src * 8 + minor_dst; SURVEY.md §8d config 3): perm[i] = successor of slot i.
constexpr uint32_t kChaseSlots = 65536;
void chase_permutation(int minor_src, int minor_dst, std::vector<uint32_t>* perm);

}  // namespace cro
