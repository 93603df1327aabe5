// probe.cu — probe context: enumeration, resident sweep buffers, the probe as
// one CUDA graph with a device-written verdict, its lanes and collection,
// metrics and the node's inventory.  The single sweeps, the fault locator, the
// host link and compute probes and the full-box probe have their own files.
//
// Reference slot: utils.RunNvidiaSmi (internal/utils/gpus.go:666-689) and
// utils.CheckGPUVisible (internal/utils/gpus.go:54-86) as called from
// handleAttachingState (internal/controller/composableresource_controller.go:259,275).
#include <dlfcn.h>
#include <unistd.h>

#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <random>
#include <type_traits>

#include "env.hpp"
#include "inventory.hpp"
#include "probe_internal.hpp"

namespace cro {

namespace {

constexpr uint64_t kDefaultSweep = 4ull << 30;
constexpr uint64_t kDefaultP2P = 1ull << 30;
constexpr uint64_t kDefaultSeedBase = 0x00C0FFEE00000000ull;
// 1024 hops: a dependent chase of that length already averages over the hop-to-hop jitter, while 64 Ki hops of a
// microsecond-scale peer load would cost more than the rest of the full-box probe.  SURVEY.md §8d's 64 Ki is one
// cro_set_latency_hops / latency_hops away, and bench.py runs 1 Ki, 4 Ki, 16 Ki and 64 Ki every time on several GPUs.
constexpr uint32_t kDefaultHops = 1024;

Params graph_params(const Lane& L) { return Params{ProbeParams{0, 0}, L.d_params}; }

void copy_cstr(char* dst, size_t cap, const std::string& s) {
    memset(dst, 0, cap);
    memcpy(dst, s.data(), std::min(cap - 1, s.size()));
}

}  // namespace

uint32_t resolve_read_variant(uint32_t v, uint64_t bytes, const env::Values& knobs) {
    // AUTO: the TMA ring has the higher asymptote but a larger constant cost per launch (ring ramp and drain), so small
    // sweeps go to plain 128-bit LDG.  Whole probes on an H100 SXM (700 W), median of 21: 64 MiB 438 us with LDG vs 457
    // with TMA, 128 MiB 791 vs 803, 256 MiB 1502 vs 1494, 1 GiB 5702 vs 5627 — the crossover sits between 128 and
    // 256 MiB (profiles/h100_700w_read_variants.jsonl; a 400 W card agrees, h100_400w_read_variants.jsonl).  The 32-byte
    // LDG flavour lost to one or the other at every size from 64 MiB to 4 GiB.
    if (v == CRO_READ_AUTO) {
        v = knobs.get("CRO_READ_VARIANT");
        if (v == CRO_READ_AUTO) v = bytes <= (128ull << 20) ? CRO_READ_LDG : CRO_READ_TMA;
    }
    return (v == READ_LDG || v == READ_TMA || v == READ_LDG256) ? v : (uint32_t)READ_TMA;
}
uint32_t resolve_copy_variant(uint32_t v, const env::Values& knobs) {
    if (v == CRO_COPY_AUTO) {
        v = knobs.get("CRO_COPY_VARIANT");
        if (v == CRO_COPY_AUTO) v = CRO_COPY_TMA_FUSED;
    }
    return (v == COPY_LDG || v == COPY_TMA || v == COPY_TMA_FUSED) ? v : (uint32_t)COPY_TMA_FUSED;
}

void chase_permutation(int minor_src, int minor_dst, std::vector<uint32_t>* perm) {
    perm->resize(kChaseSlots);
    for (uint32_t i = 0; i < kChaseSlots; ++i) (*perm)[i] = i;
    std::mt19937_64 rng((uint64_t)((long long)minor_src * 8 + (long long)minor_dst));
    for (uint32_t i = kChaseSlots - 1; i > 0; --i) {        // Sattolo: one cycle through every slot
        const uint32_t j = (uint32_t)(rng() % i);
        std::swap((*perm)[i], (*perm)[j]);
    }
}

// ---------------------------------------------------------------------------
// context
// ---------------------------------------------------------------------------

int ctx_create(const cro_opts* o, cro_ctx** out) {
    if (!out) return CRO_ERR_INVALID_ARG;
    *out = nullptr;
    cro_opts opts;
    memset(&opts, 0, sizeof opts);
    if (o) opts = *o;
    else opts.abi_version = CRO_ABI_VERSION;
    if (opts.abi_version != CRO_ABI_VERSION) return CRO_ERR_ABI_MISMATCH;
    if (opts.sweep_bytes == 0) opts.sweep_bytes = kDefaultSweep;
    if (opts.sweep_bytes % 16 != 0 || opts.sweep_bytes < 16) return CRO_ERR_INVALID_ARG;
    if (opts.p2p_bytes == 0) opts.p2p_bytes = std::min(kDefaultP2P, opts.sweep_bytes);
    if (opts.p2p_bytes > opts.sweep_bytes || opts.p2p_bytes % 16 != 0) return CRO_ERR_INVALID_ARG;
    if (opts.seed_base == 0) opts.seed_base = kDefaultSeedBase;
    if (opts.read_sweeps == 0) opts.read_sweeps = 5;
    if (opts.copy_sweeps == 0) opts.copy_sweeps = 5;
    if (opts.read_sweeps > kMaxSweepsEach || opts.copy_sweeps > kMaxSweepsEach) return CRO_ERR_INVALID_ARG;
    if (opts.latency_hops == 0) opts.latency_hops = kDefaultHops;
    if (opts.n_devices < 0 || opts.n_devices > CRO_MAX_DEVICES) return CRO_ERR_INVALID_ARG;

    std::unique_ptr<cro_ctx> c(new cro_ctx);
    c->opts = opts;
    // CRO_TRACE_INIT=1: where the cold start goes, phase by phase, on stderr (the hot-plug helper pays all of it)
    const bool trace_init = getenv("CRO_TRACE_INIT") && getenv("CRO_TRACE_INIT")[0] == '1';
    uint64_t t_phase = now_ns();
    auto phase = [&](const char* name) {
        if (!trace_init) return;
        const uint64_t t = now_ns();
        fprintf(stderr, "cro_probe_init: %-28s %8.3f ms\n", name, (double)(t - t_phase) / 1e6);
        t_phase = t;
    };
    {
        // the CRO_* knobs, validated the way the reference validates its own environment
        // (internal/controller/composableresource_adapter.go:42-45), and kept: the context never reads them again
        std::string why;
        if (!env::read(&c->knobs, &why)) {
            c->set_error(why);
            return CRO_ERR_INVALID_ARG;
        }
        c->nvtx = c->knobs.get("CRO_NVTX") != 0;
        if (const char* pr = getenv("CRO_PROC_ROOT"))
            if (*pr) c->proc_root = pr;
        if (const char* sr = getenv("CRO_SYS_ROOT"))
            if (*sr) c->sys_root = sr;
    }

    phase("options + environment");
    int n_cuda = 0;
    cudaError_t e = cudaGetDeviceCount(&n_cuda);
    phase("cuInit (cudaGetDeviceCount)");
    if (e == cudaErrorNoDevice || e == cudaErrorInsufficientDriver) {
        // No usable GPU.  A probe library without a GPU must say so loudly:
        // there is no CPU fallback on this path.
        cudaGetLastError();
        return CRO_ERR_NO_DEVICE;
    }
    if (e != cudaSuccess) {
        cudaGetLastError();
        return CRO_ERR_CUDA;
    }
    std::vector<int> ordinals;
    if (opts.n_devices > 0) {
        for (int i = 0; i < opts.n_devices; ++i) {
            if (opts.devices[i] < 0 || opts.devices[i] >= n_cuda) return CRO_ERR_INVALID_ARG;
            ordinals.push_back(opts.devices[i]);
        }
    } else {
        for (int i = 0; i < n_cuda && i < CRO_MAX_DEVICES; ++i) ordinals.push_back(i);
    }

    // Identity: /proc first (a directory walk), NVML only when asked to (its first call is slow and serialises
    // across processes) — CRO_F_NO_NVML keeps it off the hot-plug path entirely.
    const std::vector<identity::ProcGpu> proc = identity::ScanProc(c->proc_root);
    std::vector<identity::NvmlGpu> nvml;
    bool have_nvml = false;
    if (!(opts.flags & CRO_F_NO_NVML)) have_nvml = identity::ScanNvml(&nvml, nullptr);

    phase("identity scan (/proc, NVML)");
    struct Keyed { std::unique_ptr<Device> d; long long key; };
    std::vector<Keyed> keyed;
    for (int ord : ordinals) {
        std::unique_ptr<Device> d(new Device);
        d->ordinal = ord;
        cudaDeviceProp prop;
        CU_TRY(c.get(), cudaGetDeviceProperties(&prop, ord));
        cro_dev_info& info = d->info;
        memset(&info, 0, sizeof info);
        info.cuda_ordinal = ord;
        info.device_minor = -1;
        const std::string uuid = identity::FormatGpuUuid(reinterpret_cast<const unsigned char*>(prop.uuid.bytes));
        copy_cstr(info.gpu_uuid, sizeof info.gpu_uuid, uuid);
        copy_cstr(info.pci_bus_id, sizeof info.pci_bus_id,
                  identity::FormatBusIdSmi((unsigned)prop.pciDomainID, (unsigned)prop.pciBusID,
                                           (unsigned)prop.pciDeviceID, 0));
        copy_cstr(info.name, sizeof info.name, prop.name);
        info.hbm_bytes_total = prop.totalGlobalMem;
        info.sm_count = (uint32_t)prop.multiProcessorCount;
        info.cc_major = (uint32_t)prop.major;
        info.cc_minor = (uint32_t)prop.minor;
        info.identity_source = 3;
        long long key = ((long long)prop.pciDomainID << 16) | ((long long)prop.pciBusID << 8) |
                        (long long)prop.pciDeviceID;
        bool matched = false;
        if (have_nvml) {
            for (size_t k = 0; k < nvml.size(); ++k) {
                if (nvml[k].uuid != uuid) continue;
                info.device_minor = nvml[k].minor;
                if (!nvml[k].bus_id.empty()) copy_cstr(info.pci_bus_id, sizeof info.pci_bus_id, nvml[k].bus_id);
                info.identity_source = 1;
                d->sm_clock_mhz = nvml[k].sm_clock_mhz;
                d->mem_clock_mhz = nvml[k].mem_clock_mhz;
                key = (long long)k;   // nvidia-smi lists in NVML index order
                matched = true;
                break;
            }
        }
        if (!matched) {
            for (const identity::ProcGpu& g : proc) {
                if (g.uuid != uuid) continue;
                info.device_minor = atoi(g.minor.c_str());
                info.identity_source = 2;
                break;
            }
        }
        keyed.push_back({std::move(d), key});
    }
    std::stable_sort(keyed.begin(), keyed.end(), [](const Keyed& a, const Keyed& b) { return a.key < b.key; });

    for (size_t i = 0; i < keyed.size(); ++i) {
        Device* d = keyed[i].d.get();
        d->index = (int)i;
        d->sweep_bytes = opts.sweep_bytes;
        d->seed_dev = opts.seed_base | (uint64_t)(d->info.device_minor >= 0 ? d->info.device_minor : d->ordinal);
        d->seed_cur = d->seed_dev;
        phase("device properties");
        CU_TRY(c.get(), cudaSetDevice(d->ordinal));
        CU_TRY(c.get(), cudaStreamCreateWithFlags(&d->stream, cudaStreamNonBlocking));
        phase("primary context + stream");
        CU_TRY(c.get(), cudaStreamCreateWithFlags(&d->aux, cudaStreamNonBlocking));
        CU_TRY(c.get(), cudaEventCreate(&d->ev0));
        CU_TRY(c.get(), cudaEventCreate(&d->ev1));
        for (cudaEvent_t* ev : {&d->ev_fork, &d->ev_join, &d->ev_hbm_done, &d->ev_aux_done, &d->ev_chase_ready})
            CU_TRY(c.get(), cudaEventCreateWithFlags(ev, cudaEventDisableTiming));
        {
            std::string why;
            const cudaError_t pe = plan_kernels(d->ordinal, c->knobs, &d->plan, &why);
            if (pe != cudaSuccess) {     // a ring the device cannot hold is the knob's fault, not CUDA's
                c->set_error(why.empty() ? std::string("plan_kernels: ") + cudaGetErrorString(pe) : why);
                return why.empty() ? CRO_ERR_CUDA : CRO_ERR_INVALID_ARG;
            }
        }
        phase("kernel plan (module load)");
        const int max_grid = std::max({d->plan.fill.grid, d->plan.read_ldg.grid, d->plan.read_ldg256.grid,
                                       d->plan.read_tma.grid, d->plan.copy_fused.grid, d->plan.expect.grid, 1});
        int rc = alloc_scratch(c.get(), &d->scratch, max_grid);
        if (rc) return rc;
        if ((rc = alloc_scratch(c.get(), &d->scratch_aux, max_grid))) return rc;
        if ((rc = alloc_scratch(c.get(), &d->scratch_pfx, max_grid))) return rc;
        for (int k = 0; k < 2; ++k) {
            Lane& L = d->lanes[k];
            const size_t slots = k == 0 ? (size_t)kSlotCount : 64;
            CU_TRY(c.get(), cudaMalloc(&L.d_out, sizeof(SweepOut) * slots));
            CU_TRY(c.get(), cudaMemset(L.d_out, 0xFF, sizeof(SweepOut) * slots));   // no slot starts with a plausible stamp
            CU_TRY(c.get(), cudaMallocHost(&L.h_out, sizeof(SweepOut) * slots));
            CU_TRY(c.get(), cudaMalloc(&L.d_params, sizeof(ProbeParams)));
            CU_TRY(c.get(), cudaMallocHost(&L.h_params, sizeof(ProbeParams)));
            CU_TRY(c.get(), cudaMalloc(&L.d_result, sizeof(cro_probe_result)));
            CU_TRY(c.get(), cudaMallocHost(&L.h_result, sizeof(cro_probe_result)));
            CU_TRY(c.get(), cudaMemset(L.d_result, 0, sizeof(cro_probe_result)));
            CU_TRY(c.get(), cudaEventCreateWithFlags(&L.ev_done, cudaEventDisableTiming));
        }
        CU_TRY(c.get(), cudaMalloc(&d->d_tmpl, sizeof(cro_probe_result)));
        CU_TRY(c.get(), cudaMalloc(&d->d_gather, sizeof(cro_probe_result) * CRO_MAX_DEVICES));
        CU_TRY(c.get(), cudaMallocHost(&d->h_gather, sizeof(cro_probe_result) * CRO_MAX_DEVICES));
        CU_TRY(c.get(), cudaMalloc(&d->d_chase_out, 2 * CRO_MAX_DEVICES * sizeof(unsigned long long)));
        CU_TRY(c.get(), cudaMallocHost(&d->h_chase_out, 2 * CRO_MAX_DEVICES * sizeof(unsigned long long)));
        phase("buffers (device + pinned)");
        if (!(opts.flags & CRO_F_LAZY_ALLOC)) {
            if ((rc = ensure_region(c.get(), d))) return rc;
            phase("sweep region");
        }
        refresh_ecc(c.get(), d);
        c->devs.push_back(std::move(keyed[i].d));
    }
    for (auto& d : c->devs) {
        CU_TRY(c.get(), cudaSetDevice(d->ordinal));
        int rc = stage_template(c.get(), d.get());
        if (rc) return rc;
    }
    phase("identity template");
    *out = c.release();
    return CRO_OK;
}

thread_local std::string g_init_error;
const std::string& last_init_error() { return g_init_error; }
void set_thread_error(const std::string& m) noexcept {
    try { g_init_error = m; } catch (...) {}
}

}  // namespace cro
cro_ctx::~cro_ctx() {
    if (inv_thread.joinable()) inv_thread.join();     // a background inventory refresh still reads this context
    if (!last_error.empty()) cro::g_init_error = last_error;
}
namespace cro {

Device::~Device() {
    if (ordinal < 0) return;                      // never bound to a CUDA device: owns nothing
    // the members (the locator's and the link probe's state) are released after this body: with the device current
    // and both streams idle
    cudaSetDevice(ordinal);
    if (stream) cudaStreamSynchronize(stream);
    if (aux) cudaStreamSynchronize(aux);
    cudaFree(region);                             // cudaFree(nullptr) is a no-op
    free_scratch(&scratch);
    free_scratch(&scratch_aux);
    free_scratch(&scratch_pfx);
    for (Lane& L : lanes) {
        cudaFree(L.d_out);
        if (L.h_out) cudaFreeHost(L.h_out);
        cudaFree(L.d_params);
        if (L.h_params) cudaFreeHost(L.h_params);
        cudaFree(L.d_result);
        if (L.h_result) cudaFreeHost(L.h_result);
        if (L.graph_exec) cudaGraphExecDestroy(L.graph_exec);
        for (cudaEvent_t e : L.evpool) cudaEventDestroy(e);
        if (L.ev_done) cudaEventDestroy(L.ev_done);
    }
    cudaFree(d_tmpl);
    cudaFree(d_gather);
    if (h_gather) cudaFreeHost(h_gather);
    for (unsigned long long* t : d_chase_tables) cudaFree(t);
    cudaFree(d_chase_out);
    if (h_chase_out) cudaFreeHost(h_chase_out);
    for (cudaEvent_t e : ev_push_done) cudaEventDestroy(e);
    for (cudaEvent_t e : ev_reread_done) cudaEventDestroy(e);
    for (cudaEvent_t e : {ev0, ev1, ev_fork, ev_join, ev_hbm_done, ev_aux_done, ev_chase_ready})
        if (e) cudaEventDestroy(e);
    if (aux) cudaStreamDestroy(aux);
    if (stream) cudaStreamDestroy(stream);
    cudaGetLastError();                           // a failed release must not poison the caller's next CUDA call
}

void ctx_destroy(cro_ctx* c) {
    if (!c) return;
    if (c->nccl_ready && c->nccl_lib) {
        auto destroy = (int (*)(void*))dlsym(c->nccl_lib, "ncclCommDestroy");
        if (destroy)
            for (void* comm : c->nccl_comms)
                if (comm) destroy(comm);
    }
    delete c;                                     // ~Device releases the per-device CUDA objects
}

DeviceGuard enter_device(cro_ctx* c, int idx, bool args_ok) {
    DeviceGuard g;
    Device* d = g.d = dev_at(c, idx);
    if (!d || !args_ok) {
        g.rc = CRO_ERR_INVALID_ARG;
        return g;
    }
    g.lock = std::unique_lock<std::mutex>(d->mu);
    drain_pending(c, d);
    g.rc = [&]() -> int {
        CU_TRY(c, cudaSetDevice(d->ordinal));
        return CRO_OK;
    }();
    return g;
}

// ---------------------------------------------------------------------------
// full per-device probe
// ---------------------------------------------------------------------------
// Which half (0 = A, 1 = B) a sweep touches.  Copies run ping-pong — A->B, B->A, ... — so the checksum
// copy k+1 folds out of its source is the verification of what copy k wrote; the first read sweep reads the
// last copy's destination and the reads alternate from there.
static int copy_src_half(uint32_t k) { return (int)(k & 1u); }
static int read_half(uint32_t copies, uint32_t k) {
    if (copies == 0) return 0;
    const int last_dst = (int)(copies & 1u);           // C odd: B, C even: A
    return (k & 1u) ? 1 - last_dst : last_dst;
}

// Caller holds d->mu.  Enqueues one whole probe on the device's stream, using lane L's buffers, and returns without
// waiting: params refresh, fill, copy sweeps, read sweeps, the closed-form generator on the side stream, the finalize
// kernel that writes the result struct, and the copy-back of that struct.
int probe_enqueue(cro_ctx* c, Device* d, Lane& L) {
    const cro_opts& o = c->opts;
    Range nv(c, "cro.probe.enqueue");
    CU_TRY(c, cudaSetDevice(d->ordinal));
    int rc = ensure_region(c, d);
    if (rc) return rc;
    const uint32_t rv = resolve_read_variant(o.read_variant, d->sweep_bytes, c->knobs);
    const uint32_t cv = resolve_copy_variant(o.copy_variant, c->knobs);
    const uint32_t R = o.read_sweeps;
    const uint32_t C = (o.flags & CRO_F_SKIP_COPY) ? 0 : o.copy_sweeps;
    if (d->tmpl.sweep_bytes != d->sweep_bytes) {      // ensure_region degraded S
        if ((rc = stage_template(c, d))) return rc;
    }

    // events: one before the fill, one after every sweep (pool lives with the lane)
    const size_t need = 2 + R + C;
    while (L.evpool.size() < need) {
        cudaEvent_t e;
        CU_TRY(c, cudaEventCreate(&e));
        L.evpool.push_back(e);
    }
    std::vector<cudaEvent_t>& ev = L.evpool;
    const bool overlap = c->knobs.get("CRO_EXPECT_OVERLAP") != 0;
    unsigned char* half[2] = {d->region, d->region + d->sweep_bytes};
    const Params gp = graph_params(L);

    size_t k = 0;
    // The whole probe as one sequence; `external` records the timing events as external event-record
    // nodes so that the same sequence can be stream-captured into a CUDA graph once and replayed.
    auto issue = [&](bool external) -> int {
        const unsigned flag = external ? cudaEventRecordExternal : cudaEventRecordDefault;
        k = 0;
        CU_TRY(c, cudaMemcpyAsync(L.d_params, L.h_params, sizeof(ProbeParams), cudaMemcpyHostToDevice, d->stream));
        CU_TRY(c, cudaEventRecordWithFlags(ev[k++], d->stream, flag));
        uint32_t sweep_no = 0;
        auto maybe_inject = [&]() -> int {      // CRO_F_TEST_INJECT: corrupt one word behind a chosen sweep
            if ((o.flags & CRO_F_TEST_INJECT) && o.test_inject_after == sweep_no && o.test_inject_word < 2 * (d->sweep_bytes / 8))
                CU_TRY(c, launch_xor_word(d->region, o.test_inject_word, o.test_inject_mask, d->stream));
            ++sweep_no;
            return CRO_OK;
        };
        CU_TRY(c, launch_fill(d->plan, half[0], d->sweep_bytes, gp, d->scratch, &L.d_out[kSlotFill], d->stream));
        CU_TRY(c, cudaEventRecordWithFlags(ev[k++], d->stream, flag));
        if (maybe_inject()) return CRO_ERR_CUDA;
        // the closed form: ALU only, so it runs beside the copy sweeps (which leave the ALUs idle)
        cudaStream_t es = overlap ? d->aux : d->stream;
        if (overlap) {
            CU_TRY(c, cudaEventRecord(d->ev_fork, d->stream));
            CU_TRY(c, cudaStreamWaitEvent(d->aux, d->ev_fork, 0));
        }
        CU_TRY(c, launch_expected(d->plan, d->sweep_bytes, gp, d->scratch_aux, &L.d_out[kSlotExpect], es));
        if (overlap) CU_TRY(c, cudaEventRecord(d->ev_join, d->aux));
        for (uint32_t i = 0; i < C; ++i) {
            const int s = copy_src_half(i);
            CU_TRY(c, launch_copy(d->plan, cv, half[1 - s], half[s], d->sweep_bytes, gp, d->scratch,
                                  &L.d_out[kSlotSweep0 + i], d->stream));
            CU_TRY(c, cudaEventRecordWithFlags(ev[k++], d->stream, flag));
            if (maybe_inject()) return CRO_ERR_CUDA;
        }
        for (uint32_t i = 0; i < R; ++i) {
            CU_TRY(c, launch_read(d->plan, rv, half[read_half(C, i)], d->sweep_bytes, gp, d->scratch,
                                  &L.d_out[kSlotSweep0 + C + i], d->stream));
            CU_TRY(c, cudaEventRecordWithFlags(ev[k++], d->stream, flag));
            if (maybe_inject()) return CRO_ERR_CUDA;
        }
        if (overlap) CU_TRY(c, cudaStreamWaitEvent(d->stream, d->ev_join, 0));
        CU_TRY(c, launch_finalize(finalize_args(d->d_tmpl, L.d_result, L.d_out, L.d_params, d->sweep_bytes, R, C, rv, cv), d->stream));
        CU_TRY(c, cudaMemcpyAsync(L.h_result, L.d_result, sizeof(cro_probe_result), cudaMemcpyDeviceToHost, d->stream));
        CU_TRY(c, cudaMemcpyAsync(L.h_out, L.d_out, sizeof(SweepOut) * 64, cudaMemcpyDeviceToHost, d->stream));
        return CRO_OK;
    };

    // this probe's seed: the host refreshes the 16 bytes the graph's first node copies to the device
    const uint64_t nonce = d->nonce_next++;
    L.h_params->seed = space_seed(d, kSeedNonce, nonce);
    L.h_params->nonce = nonce;
    d->seed_cur = L.h_params->seed;
    d->nonce_cur = nonce;

    // One graph launch instead of ~40 runtime calls per probe (matters when one host thread feeds 8 GPUs).
    // The graph is tied to the options it was captured with; any capture problem falls back to direct launches.
    const uint64_t graph_key = ((uint64_t)rv << 48) ^ ((uint64_t)cv << 40) ^ ((uint64_t)R << 24) ^ ((uint64_t)C << 8) ^
                               (overlap ? 1u : 0u) ^ (d->sweep_bytes << 1) ^
                               ((o.flags & CRO_F_TEST_INJECT) ? ((uint64_t)o.test_inject_after << 56) ^ (o.test_inject_word * 0x9E3779B97F4A7C15ull) ^ o.test_inject_mask : 0);
    if (c->knobs.get("CRO_USE_GRAPH") && !L.graph_failed) {
        if (L.graph_exec && L.graph_key != graph_key) {
            cudaGraphExecDestroy(L.graph_exec);
            L.graph_exec = nullptr;
        }
        if (!L.graph_exec) {
            Range nvc(c, "cro.probe.capture");
            // a probe still running on the stream does not matter: capture records, it does not execute — and it must
            // not wait either (one host thread feeds eight GPUs: a 10 ms wait here starves the other seven)
            cudaGraph_t graph = nullptr;
            bool ok = cudaStreamBeginCapture(d->stream, cudaStreamCaptureModeThreadLocal) == cudaSuccess;
            if (ok) {
                const int irc = issue(true);
                const cudaError_t ec = cudaStreamEndCapture(d->stream, &graph);
                ok = irc == CRO_OK && ec == cudaSuccess && graph != nullptr;
            }
            if (ok) ok = cudaGraphInstantiate(&L.graph_exec, graph, 0) == cudaSuccess;
            if (graph) cudaGraphDestroy(graph);
            if (!ok) {
                cudaGetLastError();
                L.graph_exec = nullptr;
                L.graph_failed = true;
            } else {
                L.graph_key = graph_key;
                L.graph_events = k;
            }
        }
    }
    if (L.graph_exec) {
        CU_TRY(c, cudaGraphLaunch(L.graph_exec, d->stream));
        k = L.graph_events;
    } else {
        int irc = issue(false);
        if (irc) return irc;
    }
    CU_TRY(c, cudaEventRecord(L.ev_done, d->stream));
    half_a_filled(d);
    if (C > 0) {                    // copy 0 wrote the pattern into B; the ping-pong keeps it in both halves
        d->half_known[1] = true;
        d->half_seed[1] = d->seed_cur;
    }
    c->launches += 3 + R + C;       // fill + closed form + sweeps + finalize
    L.events = k;
    L.reads = R;
    L.copies = C;
    L.timed = true;
    L.in_flight = true;
    L.since = std::chrono::steady_clock::now();
    return CRO_OK;
}

// Waits for a lane's probe, honouring opts.deadline_ms (see wait_stream).
static int wait_lane(cro_ctx* c, Lane& L) {
    if (c->opts.deadline_ms <= 0) {
        CU_TRY(c, cudaEventSynchronize(L.ev_done));
        return CRO_OK;
    }
    const auto until = std::chrono::steady_clock::now() + std::chrono::milliseconds(c->opts.deadline_ms);
    for (;;) {
        cudaError_t q = cudaEventQuery(L.ev_done);
        if (q == cudaSuccess) return CRO_OK;
        if (q != cudaErrorNotReady) {
            c->set_error(std::string("cudaEventQuery: ") + cudaGetErrorString(q));
            return CRO_ERR_CUDA;
        }
        if (std::chrono::steady_clock::now() > until) {
            c->set_error("probe deadline of " + std::to_string(c->opts.deadline_ms) + " ms exceeded");
            return CRO_ERR_DEADLINE;
        }
        std::this_thread::sleep_for(std::chrono::microseconds(50));
    }
}

// Caller holds d->mu.  Waits for the probe enqueued on lane L and hands out the struct the device wrote.
static int probe_finish(cro_ctx* c, Device* d, Lane& L, cro_probe_result* r) {
    CU_TRY(c, cudaSetDevice(d->ordinal));
    int rc = wait_lane(c, L);
    L.in_flight = false;
    d->last_lane = (int)(&L - d->lanes);
    if (rc) {
        memset(r, 0, sizeof *r);
        r->abi_version = CRO_ABI_VERSION;
        r->status = rc;
        return rc;
    }
    *r = *L.h_result;
    d->last = *r;
    d->have_last = true;
    c->m_probes++;
    if (r->status != CRO_OK) {
        c->m_probe_failures++;
        c->set_error(describe_failure(d, *r));
        // What the memory itself reported: uncorrected volatile ECC errors (nvmlDeviceGetTotalEccErrors).
        // NVML calls serialise across processes (with several ranks probing, enough to skew the ranks' all-gather), so the warm probe reuses the count read at init / at the last full-box probe and
        // only a FAILED probe pays for a fresh read — which then also goes into the device-resident copies.
        const uint32_t before = d->ecc_uncorrected;
        refresh_ecc(c, d);
        if (d->ecc_uncorrected != before) {
            r->ecc_errors = d->ecc_uncorrected;
            d->tmpl.ecc_errors = d->ecc_uncorrected;
            *L.h_result = *r;
            CU_TRY(c, cudaMemcpyAsync(L.d_result, L.h_result, sizeof *r, cudaMemcpyHostToDevice, d->stream));
            CU_TRY(c, cudaMemcpyAsync(d->d_tmpl, &d->tmpl, sizeof d->tmpl, cudaMemcpyHostToDevice, d->stream));
            CU_TRY(c, cudaStreamSynchronize(d->stream));
        }
    }
    return r->status;
}

void drain_pending(cro_ctx* c, Device* d) {
    while (d->lane_count > 0) {
        Lane& L = d->lanes[d->lane_head];
        Device::Collected col;
        col.rc = probe_finish(c, d, L, &col.r);
        col.at = std::chrono::steady_clock::now();
        d->done.push_back(col);
        d->lane_head ^= 1;
        --d->lane_count;
    }
}

int ctx_probe_device(cro_ctx* c, int idx, cro_probe_result* out) {
    Device* d = dev_at(c, idx);
    if (!d || !out) return CRO_ERR_INVALID_ARG;
    std::lock_guard<std::mutex> g(d->mu);
    drain_pending(c, d);
    d->done.clear();                  // a synchronous probe supersedes uncollected asynchronous ones
    d->lane_head = 0;
    Lane& L = d->lanes[0];            // always lane 0: its result buffer is the all-gather send buffer
    int rc = probe_enqueue(c, d, L);
    if (rc) {
        memset(out, 0, sizeof *out);
        out->abi_version = CRO_ABI_VERSION;
        out->status = rc;
        return rc;
    }
    return probe_finish(c, d, L, out);
}

// Asynchronous form: begin enqueues a probe and returns; end waits for the OLDEST one and evaluates it.  Up to two
// probes per device may be in flight — the second one's kernels are already queued behind the first's, so the GPU
// does not idle while the host collects one result and starts the next.  Lets ONE host thread (the reference's single
// reconcile worker) keep every attached GPU busy.
int ctx_probe_begin(cro_ctx* c, int idx) {
    Device* d = dev_at(c, idx);
    if (!d) return CRO_ERR_INVALID_ARG;
    std::lock_guard<std::mutex> g(d->mu);
    if (d->lane_count + (int)d->done.size() >= 2) return CRO_OK;   // two in flight (or waiting to be collected): no-op
    Lane& L = d->lanes[(d->lane_head + d->lane_count) & 1];
    if (L.in_flight) return CRO_OK;
    int rc = probe_enqueue(c, d, L);
    if (rc) return rc;
    ++d->lane_count;
    return CRO_OK;
}

// 1 when the oldest probe begun on this device has finished (or none is in flight), 0 while it runs.
int ctx_probe_poll(cro_ctx* c, int idx) {
    Device* d = dev_at(c, idx);
    if (!d) return 1;
    std::lock_guard<std::mutex> g(d->mu);
    if (!d->done.empty() || d->lane_count == 0) return 1;
    cudaSetDevice(d->ordinal);
    // anything but "still running" counts as finished: a failed stream must not keep a poller spinning —
    // cro_probe_end then reports the CUDA error
    return cudaEventQuery(d->lanes[d->lane_head].ev_done) == cudaErrorNotReady ? 0 : 1;
}

// Probes in flight or finished-but-uncollected on this device (0..2).
int ctx_probe_depth(cro_ctx* c, int idx) {
    Device* d = dev_at(c, idx);
    if (!d) return 0;
    std::lock_guard<std::mutex> g(d->mu);
    return d->lane_count + (int)d->done.size();
}

// Blocks until the oldest probe in flight on this device (if any) has finished; does not collect it.
int ctx_probe_wait(cro_ctx* c, int idx) {
    Device* d = dev_at(c, idx);
    if (!d) return CRO_ERR_INVALID_ARG;
    std::lock_guard<std::mutex> g(d->mu);
    if (!d->done.empty() || d->lane_count == 0) return CRO_OK;
    CU_TRY(c, cudaSetDevice(d->ordinal));
    CU_TRY(c, cudaEventSynchronize(d->lanes[d->lane_head].ev_done));
    return CRO_OK;
}

int ctx_probe_end(cro_ctx* c, int idx, cro_probe_result* out) {
    Device* d = dev_at(c, idx);
    if (!d || !out) return CRO_ERR_INVALID_ARG;
    std::lock_guard<std::mutex> g(d->mu);
    // a drained result nobody collected for more than a second says nothing about the device NOW
    while (!d->done.empty() && std::chrono::steady_clock::now() - d->done.front().at > std::chrono::seconds(1)) d->done.pop_front();
    if (d->done.empty()) {
        if (d->lane_count == 0) {      // nothing begun: behave like the synchronous call
            Lane& L0 = d->lanes[d->lane_head];
            int rc = probe_enqueue(c, d, L0);
            if (rc) return rc;
            ++d->lane_count;
        }
        Lane& L = d->lanes[d->lane_head];
        const int rc = probe_finish(c, d, L, out);
        d->lane_head ^= 1;
        --d->lane_count;
        return rc;
    }
    *out = d->done.front().r;
    const int rc = d->done.front().rc;
    d->done.pop_front();
    return rc;
}

// Prometheus text exposition of what the context has seen (SURVEY.md §5: the operator registers collectors with the
// controller-runtime metrics registry, cmd/main.go:66,119-125; a Go collector forwards these lines).
std::string ctx_metrics_text(cro_ctx* c) {
    std::string o;
    auto counter = [&](const char* name, const char* help, uint64_t v) {
        o += std::string("# HELP ") + name + " " + help + "\n# TYPE " + name + " counter\n" + name + " " + std::to_string(v) + "\n";
    };
    counter("cro_probe_total", "HBM probes collected by this context.", c->m_probes.load());
    counter("cro_probe_failures_total", "Probes whose device-side verdict was not ok.", c->m_probe_failures.load());
    counter("cro_fullbox_probe_total", "cro_probe_all calls (concurrent probes + NVLink rounds + all-gather).", c->m_fullbox.load());
    counter("cro_helper_probe_total", "Probes of devices attached after cuInit, run through the helper process.", c->m_helper_probes.load());
    counter("cro_helper_probe_failures_total", "Helper-process probes that failed or timed out.", c->m_helper_failures.load());
    counter("cro_inventory_rescans_total", "Times the node inventory was rebuilt from the driver registry.", c->inv_rescans.load());
    counter("cro_kernel_launches_total", "CUDA kernels launched by this context.", c->launches.load());
    struct G { const char* name; const char* help; };
    const G gauges[] = {{"cro_probe_status", "Status of the device's last probe (0 ok, <0 a CRO_ERR_* code)."},
                        {"cro_probe_hbm_read_bytes_per_second", "Best read sweep of the last probe."},
                        {"cro_probe_hbm_copy_bytes_per_second", "Best copy sweep of the last probe (read + written bytes)."},
                        {"cro_probe_hbm_fill_bytes_per_second", "Fill sweep of the last probe."},
                        {"cro_probe_copies_verified", "Copy sweeps of the last probe whose destination was re-read and matched."},
                        {"cro_probe_ecc_uncorrected", "Uncorrected volatile ECC errors as last read from NVML."},
                        {"cro_probe_nonce", "Probes run on the device by this context."}};
    for (const G& g : gauges) {
        o += std::string("# HELP ") + g.name + " " + g.help + "\n# TYPE " + g.name + " gauge\n";
        for (auto& dp : c->devs) {
            Device* d = dp.get();
            std::lock_guard<std::mutex> lk(d->mu);
            if (!d->have_last) continue;
            const cro_probe_result& r = d->last;
            const std::string uuid(r.gpu_uuid, strnlen(r.gpu_uuid, sizeof r.gpu_uuid));
            auto rate = [](uint64_t bytes, uint64_t ns) -> long long { return ns ? (long long)((unsigned __int128)bytes * 1000000000ull / ns) : 0; };
            long long v = 0;
            const std::string n = g.name;
            if (n == "cro_probe_status") v = r.status;
            else if (n == "cro_probe_hbm_read_bytes_per_second") v = rate(r.sweep_bytes, r.read_best_ns);
            else if (n == "cro_probe_hbm_copy_bytes_per_second") v = rate(2 * r.sweep_bytes, r.copy_best_ns);
            else if (n == "cro_probe_hbm_fill_bytes_per_second") v = rate(r.sweep_bytes, r.fill_ns);
            else if (n == "cro_probe_copies_verified") v = r.copy_verified;
            else if (n == "cro_probe_ecc_uncorrected") v = r.ecc_errors;
            else v = r.nonce;
            o += n + "{gpu_uuid=\"" + uuid + "\",minor=\"" + std::to_string(r.device_minor) + "\"} " + std::to_string(v) + "\n";
        }
    }
    return o;
}

// CUDA-event and %globaltimer times of the sweeps of the device's last collected probe.
int ctx_sweep_times(cro_ctx* c, int idx, cro_sweep_time* out, int cap, int* n_out) {
    DeviceGuard g = enter_device(c, idx, n_out != nullptr);
    if (g.rc) return g.rc;
    Device* d = g.d;
    Lane& L = d->lanes[d->last_lane];
    const int n = L.timed ? (int)(1 + L.copies + L.reads) : 0;
    *n_out = n;
    if (n == 0) return CRO_OK;
    if (!out || cap < n) return CRO_ERR_BUFFER_SMALL;
    for (int i = 0; i < n; ++i) {
        float ms = 0;
        CU_TRY(c, cudaEventElapsedTime(&ms, L.evpool[(size_t)i], L.evpool[(size_t)i + 1]));
        cro_sweep_time& t = out[i];
        memset(&t, 0, sizeof t);
        const SweepOut& s = L.h_out[i == 0 ? kSlotFill : kSlotSweep0 + i - 1];
        t.kind = i == 0 ? 0u : (i <= (int)L.copies ? 1u : 2u);
        t.index = i == 0 ? 0u : (t.kind == 1 ? (uint32_t)(i - 1) : (uint32_t)(i - 1 - (int)L.copies));
        t.bytes = t.kind == 1 ? 2 * d->sweep_bytes : d->sweep_bytes;
        t.event_ns = ms_to_ns(ms);
        t.timer_ns = s.t1 - s.t0;
    }
    return CRO_OK;
}

// ---------------------------------------------------------------------------
// the node's inventory, fresh on every query (inventory.hpp)
// ---------------------------------------------------------------------------
// The slow part of an inventory refresh: reads the registry's `information` files (each read goes through the
// driver) and, when the node holds other devices than this context, re-initialises NVML for nvidia-smi's ordering.
// Touches nothing of the context but its options, so it can run on a side thread.
static std::vector<cro_dev_info> build_inventory(const cro_ctx* c, const std::vector<cro_dev_info>& mine, bool have_proc,
                                                 bool* scanned_nvml) {
    const bool nvml_ok = !(c->opts.flags & CRO_F_NO_NVML);
    std::vector<identity::ProcGpu> proc;
    if (have_proc) proc = identity::ScanProc(c->proc_root);
    std::vector<inventory::Seen> seen;
    bool have_scan = have_proc;
    if (have_proc) {
        seen = inventory::FromProc(proc);
        // the common case — the node holds exactly the devices this context manages — needs nothing more
        bool same = seen.size() == mine.size();
        for (const auto& s : seen) {
            bool found = false;
            for (const auto& m : mine) found = found || s.uuid == std::string(m.gpu_uuid, strnlen(m.gpu_uuid, sizeof m.gpu_uuid));
            same = same && found;
        }
        if (same) have_scan = false;          // Merge then keeps the context's own (nvidia-smi) order
    }
    if (have_scan || !have_proc) {
        std::vector<identity::NvmlGpu> nv;
        if (nvml_ok && identity::ScanNvml(&nv, nullptr)) {   // init + shutdown: NVML sees hot-plugged devices only after a re-init
            *scanned_nvml = true;
            std::vector<inventory::Seen> ordered;
            for (const auto& g2 : nv) {                        // nvidia-smi lists in NVML index order
                bool on_node = !have_proc;
                for (const auto& s : seen) on_node = on_node || s.uuid == g2.uuid;
                if (!on_node) continue;
                inventory::Seen s;
                s.uuid = g2.uuid; s.bus_id = g2.bus_id; s.minor = g2.minor; s.source = 1;
                ordered.push_back(s);
            }
            for (const auto& s : seen) {                       // on the bus but not (yet) known to NVML: keep, at the end
                bool in = false;
                for (const auto& o2 : ordered) in = in || o2.uuid == s.uuid;
                if (!in) ordered.push_back(s);
            }
            seen = ordered;
            have_scan = true;
        }
    }
    return inventory::Merge(mine, have_scan, seen);
}

int ctx_inventory(cro_ctx* c, std::vector<cro_dev_info>* out, bool force) {
    if (!c || !out) return CRO_ERR_INVALID_ARG;
    std::vector<cro_dev_info> mine;
    for (auto& d : c->devs) mine.push_back(d->info);
    std::unique_lock<std::mutex> g(c->inv_mu);
    const bool nvml_ok = !(c->opts.flags & CRO_F_NO_NVML);
    // Every call looks at the node: the registry's directory listing (readdir + stat, no driver lock).  The
    // `information` files are read again
    //   * at once, when that listing differs from the last one or the caller insists (it was told about a UUID the
    //     list lacks);
    //   * in the BACKGROUND every 30 s — the reference's own requeue period (composableresource_controller.go:223,285)
    //     — because each such read goes through the driver's locks (slow for a full box while nvidia-smi polls) and
    //     a reconcile must not pay for a refresh that will almost always confirm what is known.
    std::string key = identity::ProcRegistryListing(c->proc_root);
    const bool have_proc = !key.empty();
    if (!have_proc) key = "-";
    const auto now = std::chrono::steady_clock::now();
    const bool nvml_due = !have_proc && nvml_ok && now - c->inv_nvml_at > std::chrono::seconds(1);
    if (c->inv_valid && key == c->inv_key && !nvml_due && !force) {
        if (have_proc && now - c->inv_full_at > std::chrono::seconds(30) && !c->inv_refreshing) {
            c->inv_refreshing = true;
            c->inv_full_at = now;
            c->inv_rescans++;
            if (c->inv_thread.joinable()) c->inv_thread.join();     // the previous refresh ended long ago
            c->inv_thread = std::thread([c, mine, key]() {
                bool nv = false;
                std::vector<cro_dev_info> fresh;
                try { fresh = build_inventory(c, mine, true, &nv); } catch (...) { fresh.clear(); nv = false; }
                std::lock_guard<std::mutex> lk(c->inv_mu);
                if (c->inv_key == key && (!fresh.empty() || c->inv.empty())) c->inv = fresh;   // a newer listing wins
                if (nv) c->inv_nvml_at = std::chrono::steady_clock::now();
                c->inv_refreshing = false;
            });
        }
        *out = c->inv;
        return CRO_OK;
    }
    c->inv_rescans++;
    c->inv_full_at = now;
    bool nv = false;
    c->inv = build_inventory(c, mine, have_proc, &nv);
    if (nv) c->inv_nvml_at = now;
    c->inv_key = key;
    c->inv_valid = true;
    *out = c->inv;
    return CRO_OK;
}

int find_on_node(cro_ctx* c, const std::string& uuid, cro_dev_info* hit) {
    std::vector<cro_dev_info> inv;
    int rc = ctx_inventory(c, &inv);
    if (rc) return rc;
    for (int attempt = 0; attempt < 2; ++attempt) {
        // told about a UUID the cached list lacks: look again, properly, before saying "not on this node"
        if (attempt == 1 && (rc = ctx_inventory(c, &inv, true))) return rc;
        for (const auto& d : inv)
            if (uuid == std::string(d.gpu_uuid, strnlen(d.gpu_uuid, sizeof d.gpu_uuid))) {
                *hit = d;
                return CRO_OK;
            }
    }
    c->set_error("device '" + uuid + "' is not on this node");
    return CRO_ERR_NO_DEVICE;
}

int ctx_probe_uuid(cro_ctx* c, const char* uuid, cro_probe_result* out) {
    if (!uuid || !out) return CRO_ERR_INVALID_ARG;
    const std::string want = uuid;
    uint64_t sweep = 1ull << 30;              // helper default: 1 GiB is far beyond the L2 and starts ~4x sooner than 4 GiB
    env::Values knobs;                        // no context: this caller's environment, defaults where it is illegal
    if (c) knobs = c->knobs;
    else env::read(&knobs, nullptr);
    int deadline = (int)knobs.get("CRO_HELPER_TIMEOUT_MS");
    if (c) {
        cro_dev_info hit{};
        const int rc = find_on_node(c, want, &hit);
        if (rc) return rc;
        if (hit.flags & CRO_DEV_IN_PROCESS) return ctx_probe_device(c, hit.dev_index, out);
        sweep = std::min<uint64_t>(c->opts.sweep_bytes, sweep);
        if (c->opts.deadline_ms > 0) deadline = c->opts.deadline_ms;
    }
    std::string err;
    if (c && c->nvtx) nvtxRangePushA("cro.probe.helper");
    const int rc = inventory::RunHelper("", want, sweep, deadline, out, &err);
    if (c && c->nvtx) nvtxRangePop();
    if (c) {
        c->m_helper_probes++;
        if (rc != CRO_OK) c->m_helper_failures++;
    }
    if (rc != CRO_OK && !err.empty()) {
        if (c) c->set_error(err);
        else set_thread_error(err);
    }
    return rc;
}

void set_call_error(cro_ctx* c, const std::string& m) {
    if (c) c->set_error(m);
    else set_thread_error(m);
}

uint64_t helper_seed_base(cro_ctx* c) {
    if (c) return c->opts.seed_base + ((c->helper_seeds.fetch_add(1) + 1) << 8);
    const uint64_t s = fresh_seed() & ~0xFFull;
    return s ? s : 0x100;         // 0 would ask the helper for the default base
}

// run_probe_helper reads a helper result's status from the first four bytes of its frame.
template <class R>
constexpr bool status_first() { return offsetof(R, status) == 0 && std::is_same<decltype(R::status), int32_t>::value; }
static_assert(status_first<cro_link_result>() && status_first<cro_compute_result>() && status_first<cro_precision_result>() &&
                  status_first<cro_scan_report>() && status_first<cro_sram_result>() && status_first<cro_l2_result>(),
              "every helper result begins with its int32_t status");

int run_probe_helper(cro_ctx* c, const std::string& uuid, const std::string& what, const char* range,
                     const std::vector<std::string>& args, int deadline_ms, size_t head, size_t rec, size_t cap,
                     uint64_t (*count)(const unsigned char* head), std::string* got, uint64_t* helper_ns) {
    env::Values knobs;                        // no context: this caller's environment, defaults where it is illegal
    if (c) knobs = c->knobs;
    else env::read(&knobs, nullptr);
    const int deadline = deadline_ms > 0 ? deadline_ms : (int)knobs.get("CRO_HELPER_TIMEOUT_MS");
    DeviceGuard g;
    if (c) {
        cro_dev_info hit{};
        const int rc = find_on_node(c, uuid, &hit);
        if (rc) return rc;
        if (hit.flags & CRO_DEV_IN_PROCESS) {     // no probe of this GPU runs beside the helper
            g = enter_device(c, hit.dev_index);
            if (g.rc) return g.rc;
        }
    }
    std::string err;
    if (c && c->nvtx) nvtxRangePushA(range);
    const uint64_t t_spawn = now_ns();
    const int rc = inventory::RunHelperRaw("", what, uuid, args, deadline, head, rec, cap, count, got, &err);
    *helper_ns = now_ns() - t_spawn;
    if (c && c->nvtx) nvtxRangePop();
    if (rc != CRO_OK) {
        if (!err.empty()) set_call_error(c, err);
        return rc;
    }
    int32_t status;
    memcpy(&status, got->data(), sizeof status);
    if (status != CRO_OK && status != CRO_ERR_CHECKSUM) set_call_error(c, what + " for " + uuid + ": " + cro_strerror(status));
    return CRO_OK;
}

}  // namespace cro
