// probe_internal.hpp — what the probe context's translation units share: error plumbing, the device guard, the sweep
// region's bookkeeping, the probe's enqueue / drain, and the owners of lazily allocated probe state.
#pragma once
#include <algorithm>
#include <chrono>
#include <cstring>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include <nvtx3/nvToolsExt.h>

#include "identity.hpp"
#include "probe.hpp"

namespace cro {

#define CU_TRY(ctx, expr)                                                              \
    do {                                                                               \
        cudaError_t e__ = (expr);                                                      \
        if (e__ != cudaSuccess) {                                                      \
            (ctx)->set_error(std::string(#expr) + ": " + cudaGetErrorString(e__));     \
            return e__ == cudaErrorMemoryAllocation ? CRO_ERR_OOM : CRO_ERR_CUDA;      \
        }                                                                              \
    } while (0)

inline uint64_t ms_to_ns(float ms) { return (uint64_t)((double)ms * 1.0e6 + 0.5); }
inline uint64_t now_ns() {
    return (uint64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

// NVTX ranges around the host-side phases (SURVEY.md §5); nsys / ncu --nvtx pick them up, nothing else pays.
struct Range {
    bool on;
    Range(const cro_ctx* c, const char* name) : on(c->nvtx) { if (on) nvtxRangePushA(name); }
    ~Range() { if (on) nvtxRangePop(); }
};

// A seed no earlier call shares: the wall clock, the process and a per-process call count through splitmix; never 0
// (hbm_scan.cu).
uint64_t fresh_seed();

inline Params imm_params(const Device* d) { return Params{ProbeParams{d->seed_cur, d->nonce_cur}, nullptr}; }

// The seed spaces of a device: seed j of call k in a space is seed_dev + offset + (per_call * k + j) * kNonceStride.
// No seed of one space is a seed of another while every count per_call * k + j stays below 2^52.  kNonceStride is
// odd, hence invertible mod 2^64, so seeds of offsets O != O' and counts n, n' are equal only when (n - n') *
// kNonceStride = O' - O (mod 2^64).  Every offset is 0 or a power of two from 2^52 up, so O' - O is a nonzero multiple
// of 2^52 mod 2^64, and so is n - n' (an odd factor keeps the power of two in a number): n or n' is at least 2^52.  The
// largest per_call, the register-file probe's 65536, keeps its counts 65536 k + j below 2^52 while k < 2^36.
// Within a space distinct counts give distinct seeds, so no call passes on what an earlier call left behind.
enum SeedSpace { kSeedNonce, kSeedRetest, kSeedLink, kSeedCompute, kSeedSram, kSeedL2, kSeedPrecision, kSeedSparse, kSeedRegfile,
                 kSeedWarpMma, kSeedXlane, kSeedAlu, kSeedBarrier };
struct SeedSpaceInfo {
    uint64_t offset, per_call;
};
constexpr SeedSpaceInfo kSeedSpaces[] = {
    {0, 1},             // kSeedNonce: probe nonce k (the HBM probe's pattern)
    {1ull << 63, 1},    // kSeedRetest: the fault locator's retest pattern (k = 0)
    {1ull << 62, 3},    // kSeedLink: host link patterns P1 .. P3
    {1ull << 61, 1},    // kSeedCompute: compute probe operands
    {1ull << 60, 8},    // kSeedSram: SRAM probe, one per cluster rank (the largest cluster)
    {1ull << 59, 2},    // kSeedL2: L2 probe march (j = 0) and atomics (j = 1)
    {1ull << 58, 1},    // kSeedPrecision: precision probe operands
    {1ull << 57, 1},    // kSeedSparse: sparse probe operands and pairs
    {1ull << 56, CRO_REGFILE_MAX_ITERATIONS},   // kSeedRegfile: register-file probe, one per iteration
    {1ull << 55, 1},    // kSeedWarpMma: warp-MMA probe operands and MOVE tile
    {1ull << 54, CRO_XLANE_MAX_ITERATIONS},     // kSeedXlane: cross-lane probe, one per iteration
    {1ull << 53, 1},    // kSeedAlu: ALU probe table, one per call (every iteration repeats it)
    {1ull << 52, 1},    // kSeedBarrier: barrier probe table, one per call (every iteration repeats it)
};
inline uint64_t space_seed(const Device* d, SeedSpace s, uint64_t k, uint64_t j = 0) {
    return d->seed_dev + kSeedSpaces[s].offset + (kSeedSpaces[s].per_call * k + j) * kNonceStride;
}

inline Device* dev_at(cro_ctx* c, int idx) {
    if (!c || idx < 0 || idx >= (int)c->devs.size()) return nullptr;
    return c->devs[(size_t)idx].get();
}

// Drains every probe still in flight on the device (oldest first) into d->done, so another operation may use the
// stream / the region.  Caller holds d->mu.
void drain_pending(cro_ctx* c, Device* d);

// One call's hold on device idx.  An index that is not a device of the context, or !args_ok (the call's own checks),
// is CRO_ERR_INVALID_ARG at once.  Otherwise d->mu is taken, every probe in flight drained (a probe in flight must be
// collected before anything else uses the stream or the region) and the device made current; rc is the error of that.
struct DeviceGuard {
    Device* d = nullptr;
    std::unique_lock<std::mutex> lock;
    int rc = CRO_OK;
};
DeviceGuard enter_device(cro_ctx* c, int idx, bool args_ok = true);

// CRO_ERR_INVALID_ARG for an index that is not a device of the context, with why the call needs one in the error text.
inline int unknown_device(cro_ctx* c, int idx, const char* why) {
    c->set_error("dev_index " + std::to_string(idx) + " is not a device of this context (" + why + ")");
    return CRO_ERR_INVALID_ARG;
}

inline int ensure_region(cro_ctx* c, Device* d) {
    if (d->region) return CRO_OK;
    CU_TRY(c, cudaSetDevice(d->ordinal));
    // A device that is already in use may not have 2*S free (the reference's own pre-check for that
    // is CheckNoGPULoads, internal/utils/gpus.go:88).  Degrade: halve S down to 64 MiB — still far
    // beyond the 50 MB L2 when doubled — and report the size actually swept in the result.
    const uint64_t asked = d->sweep_bytes;
    cudaError_t e = cudaErrorMemoryAllocation;
    for (uint64_t s = asked;; s = (s / 2) & ~(uint64_t)15) {
        e = cudaMalloc(&d->region, 2 * s);
        if (e == cudaSuccess) {
            if (s != d->sweep_bytes) {
                d->sweep_bytes = s;
                for (Lane& L : d->lanes)
                    if (L.graph_exec) { cudaGraphExecDestroy(L.graph_exec); L.graph_exec = nullptr; }
            }
            break;
        }
        cudaGetLastError();
        d->region = nullptr;
        if (e != cudaErrorMemoryAllocation || s <= (64ull << 20) || !(c->opts.flags & CRO_F_DEGRADE_ON_OOM)) {
            c->set_error("cudaMalloc of sweep region (" + std::to_string(2 * s) + " bytes, asked for " +
                         std::to_string(2 * asked) + ") failed: " + cudaGetErrorString(e));
            return CRO_ERR_OOM;
        }
    }
    d->filled = false;
    d->half_known[0] = d->half_known[1] = false;
    return CRO_OK;
}

// Half A now holds the pattern of seed_cur (a fill, or a probe's fill).
inline void half_a_filled(Device* d) {
    d->filled = true;
    d->half_known[0] = true;
    d->half_seed[0] = d->seed_cur;
}

inline int ensure_filled(cro_ctx* c, Device* d) {
    int rc = ensure_region(c, d);
    if (rc) return rc;
    if (d->filled) return CRO_OK;
    CU_TRY(c, launch_fill(d->plan, d->region, d->sweep_bytes, imm_params(d), d->scratch, nullptr, d->stream));
    c->launches++;
    half_a_filled(d);
    return CRO_OK;
}

// Waits for the stream, honouring opts.deadline_ms (kernels cannot be cancelled; on expiry the caller gets
// CRO_ERR_DEADLINE and the next call on this device synchronises first because it takes the same stream).
inline int wait_stream(cro_ctx* c, Device* d) {
    if (c->opts.deadline_ms <= 0) {
        CU_TRY(c, cudaStreamSynchronize(d->stream));
        return CRO_OK;
    }
    const auto until = std::chrono::steady_clock::now() + std::chrono::milliseconds(c->opts.deadline_ms);
    for (;;) {
        cudaError_t q = cudaStreamQuery(d->stream);
        if (q == cudaSuccess) return CRO_OK;
        if (q != cudaErrorNotReady) {
            c->set_error(std::string("cudaStreamQuery: ") + cudaGetErrorString(q));
            return CRO_ERR_CUDA;
        }
        if (std::chrono::steady_clock::now() > until) {
            c->set_error("probe deadline of " + std::to_string(c->opts.deadline_ms) + " ms exceeded");
            return CRO_ERR_DEADLINE;
        }
        std::this_thread::sleep_for(std::chrono::microseconds(50));
    }
}

inline int alloc_scratch(cro_ctx* c, SweepScratch* sc, int max_grid) {
    CU_TRY(c, cudaMalloc(&sc->partials, sizeof(ulonglong4) * (size_t)max_grid));
    CU_TRY(c, cudaMalloc(&sc->counter, sizeof(unsigned)));
    CU_TRY(c, cudaMalloc(&sc->tmin, sizeof(unsigned long long)));
    CU_TRY(c, cudaMalloc(&sc->tmax, sizeof(unsigned long long)));
    CU_TRY(c, cudaMalloc(&sc->tile_ctr, sizeof(unsigned long long)));
    CU_TRY(c, cudaMemset(sc->tile_ctr, 0, sizeof(unsigned long long)));
    CU_TRY(c, cudaMemset(sc->counter, 0, sizeof(unsigned)));
    CU_TRY(c, cudaMemset(sc->tmin, 0xFF, sizeof(unsigned long long)));
    CU_TRY(c, cudaMemset(sc->tmax, 0, sizeof(unsigned long long)));
    return CRO_OK;
}

inline void free_scratch(SweepScratch* sc) {
    cudaFree(sc->partials);
    cudaFree(sc->counter);
    cudaFree(sc->tmin);
    cudaFree(sc->tmax);
    cudaFree(sc->tile_ctr);
}

// Stages the fields of the result that the device cannot know (identity strings, NVML readings, options) into the
// template the finalize kernel starts from.  Caller has the device current.
inline int stage_template(cro_ctx* c, Device* d) {
    cro_probe_result& t = d->tmpl;
    memset(&t, 0, sizeof t);
    t.abi_version = CRO_ABI_VERSION;
    t.cuda_ordinal = d->ordinal;
    t.device_minor = d->info.device_minor;
    memcpy(t.gpu_uuid, d->info.gpu_uuid, sizeof t.gpu_uuid);
    memcpy(t.pci_bus_id, d->info.pci_bus_id, sizeof t.pci_bus_id);
    t.hbm_bytes_total = d->info.hbm_bytes_total;
    t.sweep_bytes = d->sweep_bytes;
    t.sm_count = d->info.sm_count;
    t.sm_clock_mhz = d->sm_clock_mhz;
    t.mem_clock_mhz = d->mem_clock_mhz;
    t.ecc_errors = d->ecc_uncorrected;
    t.rank = (uint8_t)(c->opts.rank_base + (uint32_t)d->index);
    t.world = (uint8_t)(c->opts.world_override ? c->opts.world_override : (uint32_t)c->devs.size());
    t.p2p_bytes = c->opts.p2p_bytes;
    if (c->peers_enabled)
        for (size_t j = 0; j < c->devs.size() && j < 8; ++j) {
            if ((int)j == d->index) continue;
            int can = 0;
            cudaDeviceCanAccessPeer(&can, d->ordinal, c->devs[j]->ordinal);
            t.p2p_access[j] = (uint8_t)can;
        }
    CU_TRY(c, cudaMemcpyAsync(d->d_tmpl, &t, sizeof t, cudaMemcpyHostToDevice, d->stream));
    CU_TRY(c, cudaStreamSynchronize(d->stream));    // `t` lives in pageable memory
    return CRO_OK;
}

// Caches the device's uncorrected volatile ECC count (0 when NVML is not the identity source or ECC is off).
inline void refresh_ecc(cro_ctx* c, Device* d) {
    if ((c->opts.flags & CRO_F_NO_NVML) || d->info.identity_source != 1) return;
    unsigned long long ecc = 0;
    if (identity::NvmlEccUncorrected(std::string(d->info.gpu_uuid, strnlen(d->info.gpu_uuid, sizeof d->info.gpu_uuid)), &ecc))
        d->ecc_uncorrected = (uint32_t)std::min<unsigned long long>(ecc, 0xFFFFFFFFull);
}

inline std::string describe_failure(const Device* d, const cro_probe_result& r) {
    const std::string who = std::string(d->info.gpu_uuid, strnlen(d->info.gpu_uuid, sizeof d->info.gpu_uuid));
    const std::string idx = std::to_string((unsigned)r.fail_index);
    switch (r.fail_code) {
        case CRO_FAIL_EXPECT: return "closed-form checksum slot on " + who + " is stale: the generator kernel did not run";
        case CRO_FAIL_COPY_SRC:
            return "HBM copy sweep " + idx + " on " + who + " read something else than the pattern" +
                   (r.fail_index ? " (the destination of sweep " + std::to_string((unsigned)r.fail_index - 1) + " is corrupt)" : " (the fill is corrupt)");
        case CRO_FAIL_READ: return "HBM read sweep " + idx + " on " + who + " does not reproduce the pattern checksum";
        case CRO_FAIL_P2P_READ: return "NVLink read of peer " + idx + " from " + who + " does not reproduce the pattern checksum";
        case CRO_FAIL_P2P_PUSH: return "NVLink push between " + who + " and peer " + idx + " did not land the pattern checksum";
        case CRO_FAIL_P2P_CHASE: return "NVLink pointer chase from " + who + " through peer " + idx + " ended on the wrong slot";
        case CRO_FAIL_STALE: return "sweep slot " + idx + " on " + who + " carries another probe's stamp: a kernel of the probe did not run";
        default: return "probe of " + who + " failed";
    }
}

int probe_enqueue(cro_ctx* c, Device* d, Lane& L);
// One latency table on the current device: permutation `perm` with slot i at table[i*16], the head of its own
// 128-byte line.
int upload_chase_table(cro_ctx* c, const std::vector<uint32_t>& perm, unsigned long long** table);

// Closed form of the complement of a pattern over n words, from the pattern's: ~p = -1 - p, and the weights
// 2i + 1 of n words sum to n^2.
inline SweepOut complement_fold(SweepOut f, uint64_t n) {
    f.x ^= (n & 1) ? ~0ull : 0ull;
    f.s = 0 - n - f.s;
    f.w = 0 - n * n - f.w;
    return f;
}

// Device memory of one call, freed on every way out.
template <class T>
struct DeviceMem {
    T* p = nullptr;
    DeviceMem() = default;
    DeviceMem(const DeviceMem&) = delete;
    DeviceMem& operator=(const DeviceMem&) = delete;
    ~DeviceMem() { cudaFree(p); }
};

// The per-SM probes' coverage loop (the compute and SRAM probes): one launch per round, relaunched while fewer than
// `want` SMs were seen and fewer than max_rounds rounds ran.  Each round arms the CTA records (all ones: a CTA that
// does not publish stays so), times launch() with ev, then fetch() enqueues the copies back, the stream is waited for
// and take(&covered) reads the round's records and says how many distinct SMs were seen so far.  *ns sums the rounds'
// event times.
template <class Launch, class Fetch, class Take>
int coverage_rounds(cro_ctx* c, Device* d, cudaEvent_t (&ev)[2], void* cta, size_t cta_bytes, uint32_t want, uint32_t max_rounds,
                    uint32_t* rounds, uint64_t* ns, Launch launch, Fetch fetch, Take take) {
    uint32_t covered = 0;
    do {
        CU_TRY(c, cudaMemsetAsync(cta, 0xFF, cta_bytes, d->stream));
        CU_TRY(c, cudaEventRecord(ev[0], d->stream));
        CU_TRY(c, launch());
        CU_TRY(c, cudaEventRecord(ev[1], d->stream));
        c->launches++;
        CU_TRY(c, fetch());
        const int e = wait_stream(c, d);
        if (e) return e;
        float ms = 0;
        CU_TRY(c, cudaEventElapsedTime(&ms, ev[0], ev[1]));
        *ns += ms_to_ns(ms);
        ++*rounds;
        const int rc = take(&covered);
        if (rc) return rc;
    } while (covered < want && *rounds < max_rounds);
    return CRO_OK;
}

// The typed parts of one copy of a MismatchBuffer: the device block or its host mirror.
struct MismatchView {
    LocateCounters* ctr;               // [check]
    unsigned long long* gran;          // [check * gran_words + word]
    SweepOut* slots;
    LocateRecord* rec;                 // [check * kLocateRecords + j]
    unsigned char* tail;
    uint64_t gran_words;               // bitmap words per check
    LocateBufs check(int k) const { return LocateBufs{ctr + k, rec + (size_t)k * kLocateRecords, gran + k * gran_words}; }
};

// What the word-checking kernels (launch_locate, launch_link_stream) write for N checks, in one device block with a
// pinned host mirror: per check its LocateCounters, its granule bitmap (one bit per CRO_LOCATE_GRANULE_BYTES of the
// `covered` bytes) and kLocateRecords records, plus result slots and a tail for the caller.  A call zeroes the
// counters, bitmaps and slots; the records are read only up to the claims.  It also owns the reduction scratch of the
// kernels that write it, one per role that runs at once.  Freed with the device: made at a probe's first call.
class MismatchBuffer {
  public:
    SweepScratch scratch[2]{};
    ~MismatchBuffer() {
        for (SweepScratch& sc : scratch) free_scratch(&sc);
        if (h_) cudaFreeHost(h_);
        cudaGetLastError();
    }
    // Lays the block out; allocates it, its mirror and `scratches` scratches of `grid` CTAs at the first call (next to
    // the region, never at its expense: no room is an error of the call).  A probe passes the same arguments at every
    // call: S is fixed once the region exists.
    int ensure(cro_ctx* c, int checks, uint64_t covered, int slots, size_t tail_bytes, int grid, int scratches) {
        int rc;
        gran_words_ = ((covered + CRO_LOCATE_GRANULE_BYTES - 1) / CRO_LOCATE_GRANULE_BYTES + 63) / 64;
        gran_ = checks * sizeof(LocateCounters);
        slots_ = (gran_ + checks * gran_words_ * 8 + 63) & ~(size_t)63;
        rec_ = slots_ + slots * sizeof(SweepOut);
        tail_ = rec_ + checks * (size_t)kLocateRecords * sizeof(LocateRecord);
        total_ = tail_ + tail_bytes;
        if (!d_.p) CU_TRY(c, cudaMalloc(&d_.p, total_));
        if (!h_) CU_TRY(c, cudaMallocHost(&h_, total_));
        for (int i = 0; i < scratches; ++i)
            if (!scratch[i].partials && (rc = alloc_scratch(c, &scratch[i], grid))) return rc;
        return CRO_OK;
    }
    int zero(cro_ctx* c, cudaStream_t st) const {
        CU_TRY(c, cudaMemsetAsync(d_.p, 0, rec_, st));
        return CRO_OK;
    }
    int fetch(cro_ctx* c, cudaStream_t st) const {      // into the mirror; the caller waits for the stream
        CU_TRY(c, cudaMemcpyAsync(h_, d_.p, total_, cudaMemcpyDeviceToHost, st));
        return CRO_OK;
    }
    MismatchView dev() const { return view(d_.p); }
    MismatchView host() const { return view(h_); }     // as of the last fetch

  private:
    MismatchView view(unsigned char* b) const {
        return MismatchView{reinterpret_cast<LocateCounters*>(b), reinterpret_cast<unsigned long long*>(b + gran_),
                            reinterpret_cast<SweepOut*>(b + slots_), reinterpret_cast<LocateRecord*>(b + rec_), b + tail_, gran_words_};
    }
    DeviceMem<unsigned char> d_;                        // its owner makes the buffer non-copyable
    unsigned char* h_ = nullptr;                        // pinned
    size_t gran_ = 0, slots_ = 0, rec_ = 0, tail_ = 0, total_ = 0;
    uint64_t gran_words_ = 0;
};

// The host link probe's per-device state (ctx_probe_host_link), made at its first call and freed with the device
// (host_link.cu): pinned host buffers H0 and H1 (cap bytes each) and the 8 MiB chase table, all mapped into the
// device's address space; the word checks' buffer, its tail the chase output; timing events.
struct LinkState {
    unsigned char* host[2] = {nullptr, nullptr};
    uint64_t cap = 0;
    unsigned char* chase = nullptr;
    MismatchBuffer buf;
    cudaEvent_t ev[14] = {};          // around the legs: CE d2h, SM read, CE h2d, SM write, SM duplex, CE duplex
    ~LinkState();
};

}  // namespace cro
