// kernels.cu — hand-written sm_90a kernels of the post-attach HBM / NVLink probe.
//
// The reference has no device code at all (its check is the UUID membership
// test at internal/utils/gpus.go:54-86); these kernels are new work in that
// slot (SURVEY.md §2b, §8d).  They are HBM-bound integer sweeps:
//
//   hbm_fill          S bytes written   w[i] = splitmix64-step(seed + i)
//   hbm_read_*        S bytes read      (XOR, wrapping sum, position-weighted sum) of all words; the probe's
//                                       reads also compare every word with its closed form and count mismatches
//   hbm_copy_fused    2S bytes moved    + the same checksum of the source stream, folded out of shared memory
//   hbm_copy_*        2S bytes moved    (plain variants, kept for comparison)
//   hbm_expected      0 bytes           the same checksum from the closed form
//   hbm_locate        S bytes read      the read sweep's checksum + every word compared with its closed form
//                                       (the fault locator, cro_locate_faults; not part of the probe)
//   link_stream       L bytes over PCIe mapped pinned host memory, read (fold + compare) and / or written
//                                       (the host link probe, cro_probe_host_link; not part of the probe)
//   chase             pointer chase over peer-resident permutations (latency)
//   compute_probe     0 bytes           the answer tile D = A * B on every SM, tensor cores and CUDA cores, checked
//                                       exactly (the compute probe, cro_probe_compute; not part of the probe)
//   probe_finalize / p2p_finalize       the verdict: the 512-byte result struct is written on the device
//
// Two data paths per sweep: 128-bit ld.global.nc / st.global vector accesses
// (also used on peer-mapped pointers for the NVLink probe), and 1-D TMA bulk
// copies (cp.async.bulk + mbarrier) through a shared-memory ring.
// The probe path has no tensor cores: there is no contraction on it.  The compute
// probe uses them on purpose: checking them is its job.
#include "kernels.cuh"
#include "sm_tile.cuh"
#include "warp_claim.cuh"

#include <cuda_bf16.h>
#include <cuda_fp8.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <type_traits>

namespace cro {

// ---------------------------------------------------------------------------
// small PTX helpers
// ---------------------------------------------------------------------------
__device__ __forceinline__ uint4 ldg_stream(const uint4* p) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p));
    return r;
}

// L2 eviction-priority policies for the bulk copies and the 32-byte loads (streaming data is touched once).
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
    return p;
}

// Batched streaming loads: ONE asm block so ptxas cannot interleave the
// consumers between the loads — every thread keeps the whole batch (128 B) in
// flight.  STRIDE is the byte distance between a thread's consecutive vectors.
template <int STRIDE>
__device__ __forceinline__ void ldg128_x8(const void* p, unsigned long long (&a)[8],
                                          unsigned long long (&b)[8]) {
    asm volatile(
        "ld.global.nc.L1::no_allocate.v2.u64 {%0,%1}, [%16];\n"
        "ld.global.nc.L1::no_allocate.v2.u64 {%2,%3}, [%16+%17];\n"
        "ld.global.nc.L1::no_allocate.v2.u64 {%4,%5}, [%16+%18];\n"
        "ld.global.nc.L1::no_allocate.v2.u64 {%6,%7}, [%16+%19];\n"
        "ld.global.nc.L1::no_allocate.v2.u64 {%8,%9}, [%16+%20];\n"
        "ld.global.nc.L1::no_allocate.v2.u64 {%10,%11}, [%16+%21];\n"
        "ld.global.nc.L1::no_allocate.v2.u64 {%12,%13}, [%16+%22];\n"
        "ld.global.nc.L1::no_allocate.v2.u64 {%14,%15}, [%16+%23];\n"
        : "=l"(a[0]), "=l"(b[0]), "=l"(a[1]), "=l"(b[1]), "=l"(a[2]), "=l"(b[2]), "=l"(a[3]),
          "=l"(b[3]), "=l"(a[4]), "=l"(b[4]), "=l"(a[5]), "=l"(b[5]), "=l"(a[6]), "=l"(b[6]),
          "=l"(a[7]), "=l"(b[7])
        : "l"(p), "n"(STRIDE), "n"(2 * STRIDE), "n"(3 * STRIDE), "n"(4 * STRIDE), "n"(5 * STRIDE),
          "n"(6 * STRIDE), "n"(7 * STRIDE));
}
// 32-byte flavour: four 32-byte vectors per thread, each fetched as two adjacent 128-bit loads (sm_90 has no
// 256-bit LDG), all eight in flight at once, under an L2 evict_first policy (`policy`, from createpolicy).
template <int STRIDE>
__device__ __forceinline__ void ldg256_x4(const void* p, uint64_t policy, unsigned long long (&w)[16]) {
    asm volatile(
        "ld.global.nc.L1::no_allocate.L2::cache_hint.v2.u64 {%0,%1}, [%16], %23;\n"
        "ld.global.nc.L1::no_allocate.L2::cache_hint.v2.u64 {%2,%3}, [%16+16], %23;\n"
        "ld.global.nc.L1::no_allocate.L2::cache_hint.v2.u64 {%4,%5}, [%16+%17], %23;\n"
        "ld.global.nc.L1::no_allocate.L2::cache_hint.v2.u64 {%6,%7}, [%16+%20], %23;\n"
        "ld.global.nc.L1::no_allocate.L2::cache_hint.v2.u64 {%8,%9}, [%16+%18], %23;\n"
        "ld.global.nc.L1::no_allocate.L2::cache_hint.v2.u64 {%10,%11}, [%16+%21], %23;\n"
        "ld.global.nc.L1::no_allocate.L2::cache_hint.v2.u64 {%12,%13}, [%16+%19], %23;\n"
        "ld.global.nc.L1::no_allocate.L2::cache_hint.v2.u64 {%14,%15}, [%16+%22], %23;\n"
        : "=l"(w[0]), "=l"(w[1]), "=l"(w[2]), "=l"(w[3]), "=l"(w[4]), "=l"(w[5]), "=l"(w[6]),
          "=l"(w[7]), "=l"(w[8]), "=l"(w[9]), "=l"(w[10]), "=l"(w[11]), "=l"(w[12]), "=l"(w[13]),
          "=l"(w[14]), "=l"(w[15])
        : "l"(p), "n"(STRIDE), "n"(2 * STRIDE), "n"(3 * STRIDE), "n"(STRIDE + 16), "n"(2 * STRIDE + 16),
          "n"(3 * STRIDE + 16), "l"(policy));
}

__device__ __forceinline__ void stg_stream(uint4* p, const uint4& v) {
    asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x),
                 "r"(v.y), "r"(v.z), "r"(v.w)
                 : "memory");
}

__device__ __forceinline__ unsigned long long lo64(const uint4& v) {
    return (unsigned long long)v.x | ((unsigned long long)v.y << 32);
}
__device__ __forceinline__ unsigned long long hi64(const uint4& v) {
    return (unsigned long long)v.z | ((unsigned long long)v.w << 32);
}

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
                 "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
// 1-D TMA: global -> shared, completion counted in bytes on an mbarrier.
__device__ __forceinline__ void tma_load_1d(void* smem_dst, const void* gsrc, uint32_t bytes,
                                            uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::
            "r"(smem_u32(smem_dst)),
        "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}
// 1-D TMA: shared -> global, tracked by bulk async-groups.
__device__ __forceinline__ void tma_store_1d(void* gdst, const void* smem_src, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst),
                 "r"(smem_u32(smem_src)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void tma_load_1d_hint(void* smem_dst, const void* gsrc, uint32_t bytes,
                                                 uint64_t* bar, uint64_t policy) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::
            "r"(smem_u32(smem_dst)),
        "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
        : "memory");
}
__device__ __forceinline__ void tma_store_1d_hint(void* gdst, const void* smem_src, uint32_t bytes,
                                                  uint64_t policy) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group.L2::cache_hint [%0], [%1], %2, %3;" ::"l"(gdst),
                 "r"(smem_u32(smem_src)), "r"(bytes), "l"(policy)
                 : "memory");
}
__device__ __forceinline__ void tma_commit() {
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
template <int N>
__device__ __forceinline__ void tma_wait_read() {
    asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void tma_wait_all() {
    asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

// ---------------------------------------------------------------------------
// Checksum accumulator.  A sweep over words w[0..n) yields (XOR, wrapping sum,
// wrapping sum of w[i] * (2i + 1)).  Threads fold 16-byte vectors (a, b) =
// (w[2v], w[2v+1]); with m = 2*(2v)+1 = 4v+1 the weighted part of the pair is
//   a*m + b*(m+2) = (a+b)*m + 2b,
// so one 64-bit multiply per VECTOR plus a running sum of the odd words.
// All three components are associative and commutative over words, so the
// result does not depend on grid shape or scheduling: bit-exact by construction.
// ---------------------------------------------------------------------------
struct Acc {
    unsigned long long x0 = 0, x1 = 0, s = 0, w = 0, d = 0;
};
__device__ __forceinline__ void fold2(Acc& A, unsigned long long a, unsigned long long b,
                                      unsigned long long m /* 4*vector_index + 1 */) {
    const unsigned long long c = a + b;
    A.x0 ^= a;
    A.x1 ^= b;
    A.s += c;
    A.w += c * m;
    A.d += b;
}
__device__ __forceinline__ unsigned long long acc_x(const Acc& A) { return A.x0 ^ A.x1; }
__device__ __forceinline__ unsigned long long acc_w(const Acc& A) { return A.w + 2ull * A.d; }

// ---------------------------------------------------------------------------
// CTA reduction + "last CTA publishes" epilogue shared by read / fused copy /
// expected.  The last CTA also re-arms the scratch (ticket, timers, dynamic
// tile counter), so no memset node sits between two sweeps.  COUNT (the read
// sweeps): m, the thread's count of mismatching words, is summed in the
// partials' fourth lane and published as out->mismatches.
// ---------------------------------------------------------------------------
template <bool COUNT = false>
__device__ __forceinline__ void publish(unsigned long long x, unsigned long long s, unsigned long long w,
                                        unsigned long long t_start, const SweepScratch sc,
                                        SweepOut* out, const ProbeParams& imm, const ProbeParams* pp,
                                        unsigned long long n_words, unsigned long long m = 0) {
    __shared__ unsigned long long sx[32], ss[32], sw[32];
    __shared__ unsigned long long sm[COUNT ? 32 : 1];
    __shared__ bool is_last;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        x ^= __shfl_xor_sync(0xffffffffu, x, o);
        s += __shfl_xor_sync(0xffffffffu, s, o);
        w += __shfl_xor_sync(0xffffffffu, w, o);
        if constexpr (COUNT) m += __shfl_xor_sync(0xffffffffu, m, o);
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int nwarps = (blockDim.x + 31) >> 5;
    if (lane == 0) {
        sx[warp] = x; ss[warp] = s; sw[warp] = w;
        if constexpr (COUNT) sm[warp] = m;
    }
    __syncthreads();
    if (warp == 0) {
        x = lane < nwarps ? sx[lane] : 0ull;
        s = lane < nwarps ? ss[lane] : 0ull;
        w = lane < nwarps ? sw[lane] : 0ull;
        if constexpr (COUNT) m = lane < nwarps ? sm[lane] : 0ull;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            x ^= __shfl_xor_sync(0xffffffffu, x, o);
            s += __shfl_xor_sync(0xffffffffu, s, o);
            w += __shfl_xor_sync(0xffffffffu, w, o);
            if constexpr (COUNT) m += __shfl_xor_sync(0xffffffffu, m, o);
        }
        if (lane == 0) {
            sc.partials[blockIdx.x] = make_ulonglong4(x, s, w, COUNT ? m : 0ull);
            atomicMin(sc.tmin, t_start);
            atomicMax(sc.tmax, globaltimer_ns());
            __threadfence();
            unsigned ticket = atomicAdd(sc.counter, 1u);
            is_last = (ticket == gridDim.x - 1);
        }
    }
    __syncthreads();
    if (!is_last) return;
    __threadfence();
    x = 0; s = 0; w = 0;
    if constexpr (COUNT) m = 0;
    for (unsigned i = threadIdx.x; i < gridDim.x; i += blockDim.x) {
        const ulonglong2* q = reinterpret_cast<const ulonglong2*>(&sc.partials[i]);
        const ulonglong2 p0 = __ldcg(q), p1 = __ldcg(q + 1);
        x ^= p0.x; s += p0.y; w += p1.x;
        if constexpr (COUNT) m += p1.y;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        x ^= __shfl_xor_sync(0xffffffffu, x, o);
        s += __shfl_xor_sync(0xffffffffu, s, o);
        w += __shfl_xor_sync(0xffffffffu, w, o);
        if constexpr (COUNT) m += __shfl_xor_sync(0xffffffffu, m, o);
    }
    __syncthreads();
    if (lane == 0) {
        sx[warp] = x; ss[warp] = s; sw[warp] = w;
        if constexpr (COUNT) sm[warp] = m;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        x = 0; s = 0; w = 0;
        for (int k = 0; k < nwarps; ++k) { x ^= sx[k]; s += ss[k]; w += sw[k]; }
        out->x = x;
        out->s = s;
        out->w = w;
        if constexpr (COUNT) {
            m = 0;
            for (int k = 0; k < nwarps; ++k) m += sm[k];
            out->mismatches = m;
        }
        out->t0 = *((volatile unsigned long long*)sc.tmin);
        out->t1 = *((volatile unsigned long long*)sc.tmax);
        out->stamp = pp ? pp->nonce : imm.nonce;
        out->n_words = n_words;
        *sc.counter = 0u;
        *sc.tmin = ~0ull;
        *sc.tmax = 0ull;
        if (sc.tile_ctr) *sc.tile_ctr = 0ull;
        __threadfence();
    }
}

// Epilogue of the sweeps that fold nothing (the fill, the plain copies): called by ONE thread per CTA once the CTA's
// work is done; the last CTA to get here publishes the sweep's %globaltimer window, stamp and word count with a zero
// checksum, and re-arms the ticket and the timers.
__device__ __forceinline__ void publish_window(unsigned long long t_start, const SweepScratch sc, SweepOut* out,
                                               const ProbeParams& imm, const ProbeParams* pp, unsigned long long n_words) {
    atomicMin(sc.tmin, t_start);
    atomicMax(sc.tmax, globaltimer_ns());
    __threadfence();
    const unsigned ticket = atomicAdd(sc.counter, 1u);
    if (ticket == gridDim.x - 1) {
        __threadfence();
        out->x = 0; out->s = 0; out->w = 0;
        out->t0 = *((volatile unsigned long long*)sc.tmin);
        out->t1 = *((volatile unsigned long long*)sc.tmax);
        out->stamp = pp ? pp->nonce : imm.nonce;
        out->n_words = n_words;
        *sc.counter = 0u;
        *sc.tmin = ~0ull;
        *sc.tmax = 0ull;
        __threadfence();
    }
}

// ---------------------------------------------------------------------------
// hbm_fill: S bytes written.  Thread t of a tile stores vectors t, t+T, ...
// so each warp-level store instruction covers 512 contiguous bytes.
// The CTAs also keep the sweep's %globaltimer window (first start, last store
// issued) so the device-written result needs no host-side event arithmetic.
// ---------------------------------------------------------------------------
// INVERT (the fault locator's complement retest) stores ~pattern; the probe's instantiation keeps the plain pattern.
template <int THREADS, int UNROLL, bool INVERT = false>
__global__ void __launch_bounds__(THREADS)
hbm_fill_kernel(uint4* __restrict__ base, unsigned long long n_vec, const ProbeParams imm,
                const ProbeParams* __restrict__ pp, SweepScratch sc, SweepOut* out) {
    const unsigned long long seed = pp ? pp->seed : imm.seed;
    constexpr unsigned long long inv = INVERT ? ~0ull : 0ull;
    unsigned long long t_start = 0;
    if (threadIdx.x == 0) t_start = globaltimer_ns();
    const unsigned long long tile_vecs = (unsigned long long)THREADS * UNROLL;
    const unsigned long long n_tiles = n_vec / tile_vecs;
    for (unsigned long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const unsigned long long v0 = tile * tile_vecs + threadIdx.x;
#pragma unroll
        for (int j = 0; j < UNROLL; ++j) {
            const unsigned long long v = v0 + (unsigned long long)j * THREADS;
            const unsigned long long a = pattern_word(seed, 2 * v) ^ inv;
            const unsigned long long b = pattern_word(seed, 2 * v + 1) ^ inv;
            stg_stream(base + v, make_uint4((unsigned)a, (unsigned)(a >> 32), (unsigned)b,
                                            (unsigned)(b >> 32)));
        }
    }
    // ragged tail (S not a multiple of the tile): plain grid-stride
    for (unsigned long long v = n_tiles * tile_vecs + (unsigned long long)blockIdx.x * THREADS +
                                threadIdx.x;
         v < n_vec; v += (unsigned long long)gridDim.x * THREADS) {
        const unsigned long long a = pattern_word(seed, 2 * v) ^ inv;
        const unsigned long long b = pattern_word(seed, 2 * v + 1) ^ inv;
        stg_stream(base + v,
                   make_uint4((unsigned)a, (unsigned)(a >> 32), (unsigned)b, (unsigned)(b >> 32)));
    }
    if (!out) return;
    __syncthreads();
    if (threadIdx.x == 0) publish_window(t_start, sc, out, imm, pp, 2 * n_vec);
}

// ---------------------------------------------------------------------------
// The word compare of the locator and the comparing read sweeps: vector
// v0 + j * vstride holds words (a[j], b[j]), which should be pattern words
// 2v and 2v + 1 (^ invert).  d[2j], d[2j + 1] get the differences; bit k of
// the result is set when d[k] != 0.
// ---------------------------------------------------------------------------
template <int J>
__device__ __forceinline__ unsigned compare_words(const unsigned long long (&a)[J], const unsigned long long (&b)[J],
                                                  unsigned long long v0, unsigned long long vstride,
                                                  unsigned long long seed, unsigned long long invert,
                                                  unsigned long long (&d)[2 * J]) {
    unsigned m = 0;
#pragma unroll
    for (int j = 0; j < J; ++j) {
        const unsigned long long v = v0 + (unsigned long long)j * vstride;
        d[2 * j] = a[j] ^ pattern_word(seed, 2 * v) ^ invert;
        d[2 * j + 1] = b[j] ^ pattern_word(seed, 2 * v + 1) ^ invert;
        m |= (d[2 * j] != 0 ? 1u : 0u) << (2 * j);
        m |= (d[2 * j + 1] != 0 ? 1u : 0u) << (2 * j + 1);
    }
    return m;
}

// A comparing read's count of the mismatching words among J vectors (compare_words).  A read keeps no records, so it
// needs neither the locator's ballot nor its atomics: each thread counts its own words and publish sums the counts.
template <int J>
__device__ __forceinline__ unsigned count_mismatches(const unsigned long long (&a)[J], const unsigned long long (&b)[J],
                                                     unsigned long long v0, unsigned long long vstride,
                                                     unsigned long long seed) {
    unsigned long long d[2 * J];
    return (unsigned)__popc(compare_words<J>(a, b, v0, vstride, seed, 0ull, d));
}

// ---------------------------------------------------------------------------
// hbm_read (LDG path): UNROLL independent 128-bit ld.global.nc per thread in
// flight, read-only path, no L1 allocation.  Also usable on a peer-mapped
// pointer (NVLink read).  CMP: every word is also compared with
// pattern_word(seed, i), i counted from base (count_mismatches); the exact
// count is published as out->mismatches (0 without CMP).
// ---------------------------------------------------------------------------
// The 16-byte flavour asks for two CTAs per SM: the compare's regeneration of the pattern is ALU work, and 32 warps
// per SM hide it behind the loads where the 16 its registers would otherwise allow do not (H100, 4 GiB: 3.07 against
// 2.42 TB/s).  The 32-byte flavour keeps its registers: held to two CTAs it read at 2.40 TB/s, not 2.84.
template <int THREADS, bool WIDE, bool CMP>
__global__ void __launch_bounds__(THREADS, WIDE ? 1 : 2)
hbm_read_ldg_kernel(const uint4* __restrict__ base, unsigned long long n_vec, const ProbeParams imm,
                    const ProbeParams* __restrict__ pp, SweepScratch sc, SweepOut* out) {
    const unsigned long long t_start = globaltimer_ns();
    const unsigned long long seed = CMP ? (pp ? pp->seed : imm.seed) : 0ull;
    unsigned long long mism = 0;
    Acc A, B;
    constexpr unsigned long long tile_vecs = (unsigned long long)THREADS * 8;  // 128 B / thread
    const unsigned long long n_tiles = n_vec / tile_vecs;
    const uint64_t pol = WIDE ? l2_policy_evict_first() : 0;
    for (unsigned long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        if (WIDE) {
            // thread t owns 32-byte vectors t, t+T, t+2T, t+3T of the tile (two 16-byte vectors each)
            const unsigned long long v0 = tile * tile_vecs + 2ull * threadIdx.x;
            const unsigned char* p = reinterpret_cast<const unsigned char*>(base + v0);
            unsigned long long w[16];
            ldg256_x4<THREADS * 32>(p, pol, w);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const unsigned long long v = v0 + 2ull * j * THREADS;
                fold2(A, w[4 * j], w[4 * j + 1], 4 * v + 1);
                fold2(B, w[4 * j + 2], w[4 * j + 3], 4 * (v + 1) + 1);
            }
            if constexpr (CMP) {
                // the even and the odd 16-byte vector of each 32-byte one: strides of 2T vectors
                const unsigned long long a0[4] = {w[0], w[4], w[8], w[12]}, b0[4] = {w[1], w[5], w[9], w[13]};
                const unsigned long long a1[4] = {w[2], w[6], w[10], w[14]}, b1[4] = {w[3], w[7], w[11], w[15]};
                mism += count_mismatches<4>(a0, b0, v0, 2ull * THREADS, seed);
                mism += count_mismatches<4>(a1, b1, v0 + 1, 2ull * THREADS, seed);
            }
        } else {
            const unsigned long long v0 = tile * tile_vecs + threadIdx.x;
            unsigned long long a[8], b[8];
            ldg128_x8<THREADS * 16>(base + v0, a, b);
#pragma unroll
            for (int j = 0; j < 8; j += 2) {
                fold2(A, a[j], b[j], 4 * (v0 + (unsigned long long)j * THREADS) + 1);
                fold2(B, a[j + 1], b[j + 1], 4 * (v0 + (unsigned long long)(j + 1) * THREADS) + 1);
            }
            if constexpr (CMP) mism += count_mismatches<8>(a, b, v0, THREADS, seed);
        }
    }
    for (unsigned long long i = n_tiles * tile_vecs + (unsigned long long)blockIdx.x * THREADS +
                                threadIdx.x;
         i < n_vec; i += (unsigned long long)gridDim.x * THREADS) {
        const uint4 v = ldg_stream(base + i);
        fold2(A, lo64(v), hi64(v), 4 * i + 1);
        if constexpr (CMP) {
            const unsigned long long a[1] = {lo64(v)}, b[1] = {hi64(v)};
            mism += count_mismatches<1>(a, b, i, 0ull, seed);
        }
    }
    publish<true>(acc_x(A) ^ acc_x(B), A.s + B.s, acc_w(A) + acc_w(B), t_start, sc, out, imm, pp, 2 * n_vec, mism);
}

// ---------------------------------------------------------------------------
// hbm_locate: the fault locator's compare pass over one half.  The loads and
// the fold are the LDG read sweep's; each word is also XORed with its expected
// value, regenerated in registers.  A warp whose words all match takes no other
// step.  Otherwise the warp (converged: every caller's loop is warp-uniform)
// records its mismatches with warp-aggregated updates:
//   count      one shared-memory add per warp, one global add per CTA at the end
//   records    one atomicAdd per warp claims a run of slots, only while the
//              buffer has room (a plain load checks first: a full buffer costs
//              no atomics, so a half that mismatches everywhere does not
//              serialise on the claim counter)
//   bit flips  per flipped bit position of the warp: a warp sum into shared
//              memory, flushed once per CTA
//   granules   a warp's words span < 2 MiB, so at most two granules: the warp
//              min and max, set with atomicOr only when not already set
// ---------------------------------------------------------------------------
struct LocateCtx {
    LocateBufs b;
    unsigned long long word0, seed, invert;
    unsigned long long* s_bits;     // shared, 64 entries
    unsigned long long* s_count;    // shared
};

__device__ __forceinline__ void mark_granule(unsigned long long* bitmap, unsigned g) {
    unsigned long long* p = bitmap + (g >> 6);
    const unsigned long long bit = 1ull << (g & 63u);
    if (!(*reinterpret_cast<volatile unsigned long long*>(p) & bit)) atomicOr(p, bit);
}

// d[k] = actual ^ expected of the lane's word k; bit k of m: word k mismatches.  Word k is half word
// 2 * (v0 + (k / 2) * vstride) + (k & 1).  The whole warp calls this (some lane has m != 0).
template <int K>
__device__ __forceinline__ void locate_record(const unsigned long long (&d)[K], unsigned m, unsigned long long v0,
                                              unsigned long long vstride, const LocateCtx& L) {
    const unsigned lane = threadIdx.x & 31u;
    unsigned long long base = warp_claim(__popc(m), &L.b.ctr->claims, kLocateRecords,
                                         [&](unsigned n_warp) { atomicAdd(L.s_count, (unsigned long long)n_warp); });
    unsigned long long flips = 0;
    unsigned gmin = ~0u, gmax = 0;
#pragma unroll
    for (int k = 0; k < K; ++k) {
        if (!((m >> k) & 1u)) continue;
        const unsigned long long w = 2 * (v0 + (unsigned long long)(k >> 1) * vstride) + (k & 1);
        if (base < kLocateRecords) {
            const unsigned long long e = pattern_word(L.seed, w) ^ L.invert;
            L.b.rec[base] = LocateRecord{L.word0 + w, e, e ^ d[k]};
        }
        ++base;
        flips |= d[k];
        const unsigned g = (unsigned)(((L.word0 + w) * 8ull) >> kLocateGranuleShift);
        gmin = min(gmin, g);
        gmax = max(gmax, g);
    }
    gmin = __reduce_min_sync(0xffffffffu, gmin);
    gmax = __reduce_max_sync(0xffffffffu, gmax);
    if (lane == 0) {
        mark_granule(L.b.granules, gmin);
        if (gmax != gmin) mark_granule(L.b.granules, gmax);
    }
    unsigned long long wor = (unsigned long long)__reduce_or_sync(0xffffffffu, (unsigned)flips) |
                             ((unsigned long long)__reduce_or_sync(0xffffffffu, (unsigned)(flips >> 32)) << 32);
    while (wor) {                       // warp-uniform
        const int bit = __ffsll((long long)wor) - 1;
        wor &= wor - 1;
        unsigned c = 0;
#pragma unroll
        for (int k = 0; k < K; ++k) c += ((m >> k) & 1u) ? (unsigned)((d[k] >> bit) & 1ull) : 0u;
        c = __reduce_add_sync(0xffffffffu, c);
        if (lane == 0) atomicAdd(&L.s_bits[bit], (unsigned long long)c);
    }
}

template <int THREADS>
__global__ void __launch_bounds__(THREADS)
hbm_locate_kernel(const uint4* __restrict__ base, unsigned long long n_vec, unsigned long long word0,
                  unsigned long long seed, unsigned long long invert, LocateBufs lb, const ProbeParams imm,
                  SweepScratch sc, SweepOut* out) {
    __shared__ unsigned long long s_bits[64];
    __shared__ unsigned long long s_count;
    const unsigned long long t_start = globaltimer_ns();
    for (unsigned i = threadIdx.x; i < 64; i += THREADS) s_bits[i] = 0;
    if (threadIdx.x == 0) s_count = 0;
    __syncthreads();
    const LocateCtx L{lb, word0, seed, invert, s_bits, &s_count};
    Acc A, B;
    constexpr unsigned long long tile_vecs = (unsigned long long)THREADS * 8;  // 128 B / thread
    const unsigned long long n_tiles = n_vec / tile_vecs;
    for (unsigned long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const unsigned long long v0 = tile * tile_vecs + threadIdx.x;
        unsigned long long a[8], b[8];
        ldg128_x8<THREADS * 16>(base + v0, a, b);
#pragma unroll
        for (int j = 0; j < 8; j += 2) {
            fold2(A, a[j], b[j], 4 * (v0 + (unsigned long long)j * THREADS) + 1);
            fold2(B, a[j + 1], b[j + 1], 4 * (v0 + (unsigned long long)(j + 1) * THREADS) + 1);
        }
        unsigned long long d[16];
        const unsigned m = compare_words<8>(a, b, v0, THREADS, seed, invert, d);
        if (__ballot_sync(0xffffffffu, m != 0)) locate_record<16>(d, m, v0, THREADS, L);
    }
    // ragged tail: warp-uniform trip count, so the ballot sees the whole warp
    const unsigned lane = threadIdx.x & 31u;
    for (unsigned long long vw = n_tiles * tile_vecs + (unsigned long long)blockIdx.x * THREADS + (threadIdx.x - lane);
         vw < n_vec; vw += (unsigned long long)gridDim.x * THREADS) {
        const unsigned long long v = vw + lane;
        unsigned long long d[2] = {0, 0};
        unsigned m = 0;
        if (v < n_vec) {
            const uint4 q = ldg_stream(base + v);
            fold2(A, lo64(q), hi64(q), 4 * v + 1);
            d[0] = lo64(q) ^ pattern_word(seed, 2 * v) ^ invert;
            d[1] = hi64(q) ^ pattern_word(seed, 2 * v + 1) ^ invert;
            m = (d[0] != 0 ? 1u : 0u) | (d[1] != 0 ? 2u : 0u);
        }
        if (__ballot_sync(0xffffffffu, m != 0)) locate_record<2>(d, m, v, 0, L);
    }
    __syncthreads();
    if (s_count) {                      // CTA-uniform: read after the barrier
        if (threadIdx.x == 0) atomicAdd(&lb.ctr->mismatches, s_count);
        if (threadIdx.x < 64 && s_bits[threadIdx.x]) atomicAdd(&lb.ctr->bits[threadIdx.x], s_bits[threadIdx.x]);
    }
    publish(acc_x(A) ^ acc_x(B), A.s + B.s, acc_w(A) + acc_w(B), t_start, sc, out, imm, nullptr, 2 * n_vec);
}

// ---------------------------------------------------------------------------
// link_stream: the host link probe's SM legs over mapped pinned host memory.
// Warps [0, rd.warps) of a CTA read (fold + compare, the locator's ballot and
// warp-aggregated records), warps [rd.warps, rd.warps + wr.warps) write; one
// launch with both roles keeps both directions of the link busy from the same
// SMs.  Warp tiles are 32 lanes x 8 vectors (4 KiB): every warp-level access
// covers 512 contiguous bytes.  Each role's CTA partial and window go through
// its own scratch; the last CTA of a role publishes the role's slot.
// ---------------------------------------------------------------------------
__device__ __forceinline__ void link_publish(const LinkRole& r, unsigned long long x, unsigned long long s,
                                             unsigned long long w, unsigned long long t0, unsigned long long t1,
                                             unsigned long long stamp) {
    const SweepScratch& sc = r.sc;
    sc.partials[blockIdx.x] = make_ulonglong4(x, s, w, 0ull);
    atomicMin(sc.tmin, t0);
    atomicMax(sc.tmax, t1);
    __threadfence();
    if (atomicAdd(sc.counter, 1u) != gridDim.x - 1) return;
    __threadfence();
    x = 0; s = 0; w = 0;
    for (unsigned i = 0; i < gridDim.x; ++i) {
        const ulonglong2* q = reinterpret_cast<const ulonglong2*>(&sc.partials[i]);
        const ulonglong2 p0 = __ldcg(q), p1 = __ldcg(q + 1);
        x ^= p0.x; s += p0.y; w += p1.x;
    }
    r.out->x = x;
    r.out->s = s;
    r.out->w = w;
    r.out->t0 = *((volatile unsigned long long*)sc.tmin);
    r.out->t1 = *((volatile unsigned long long*)sc.tmax);
    r.out->stamp = stamp;
    r.out->n_words = r.bytes >> 3;
    *sc.counter = 0u;
    *sc.tmin = ~0ull;
    *sc.tmax = 0ull;
    __threadfence();
}

__global__ void __launch_bounds__(64 * kLinkWarps)
link_stream_kernel(const LinkRole rd, const LinkRole wr, LocateBufs lb, unsigned long long stamp) {
    __shared__ unsigned long long s_bits[64];
    __shared__ unsigned long long s_count;
    __shared__ unsigned long long s_x[kLinkWarps], s_s[kLinkWarps], s_w[kLinkWarps];
    __shared__ unsigned long long s_t0[2], s_t1[2];
    const unsigned warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
    for (unsigned i = threadIdx.x; i < 64; i += blockDim.x) s_bits[i] = 0;
    if (threadIdx.x < 2) { s_t0[threadIdx.x] = ~0ull; s_t1[threadIdx.x] = 0; }
    if (threadIdx.x == 0) s_count = 0;
    __syncthreads();
    const unsigned long long t_start = globaltimer_ns();
    constexpr unsigned long long tile_vecs = 32 * 8;
    const bool reader = warp < rd.warps;
    if (reader) {
        const uint4* base = static_cast<const uint4*>(rd.buf);
        const unsigned long long n_vec = rd.bytes >> 4, seed = rd.seed;
        const LocateCtx L{lb, 0ull, seed, 0ull, s_bits, &s_count};
        const unsigned long long gw = (unsigned long long)blockIdx.x * rd.warps + warp, nw = (unsigned long long)gridDim.x * rd.warps;
        const unsigned long long n_tiles = n_vec / tile_vecs;
        Acc A, B;
        for (unsigned long long tile = gw; tile < n_tiles; tile += nw) {
            const unsigned long long v0 = tile * tile_vecs + lane;
            unsigned long long a[8], b[8];
            ldg128_x8<32 * 16>(base + v0, a, b);
            unsigned long long d[16];
            unsigned m = 0;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const unsigned long long v = v0 + (unsigned long long)j * 32;
                fold2((j & 1) ? B : A, a[j], b[j], 4 * v + 1);
                d[2 * j] = a[j] ^ pattern_word(seed, 2 * v);
                d[2 * j + 1] = b[j] ^ pattern_word(seed, 2 * v + 1);
                m |= (d[2 * j] != 0 ? 1u : 0u) << (2 * j);
                m |= (d[2 * j + 1] != 0 ? 1u : 0u) << (2 * j + 1);
            }
            if (__ballot_sync(0xffffffffu, m != 0)) locate_record<16>(d, m, v0, 32, L);
        }
        // ragged tail: warp-uniform trip count, so the ballot sees the whole warp
        for (unsigned long long vw = n_tiles * tile_vecs + gw * 32; vw < n_vec; vw += nw * 32) {
            const unsigned long long v = vw + lane;
            unsigned long long d[2] = {0, 0};
            unsigned m = 0;
            if (v < n_vec) {
                const uint4 q = ldg_stream(base + v);
                fold2(A, lo64(q), hi64(q), 4 * v + 1);
                d[0] = lo64(q) ^ pattern_word(seed, 2 * v);
                d[1] = hi64(q) ^ pattern_word(seed, 2 * v + 1);
                m = (d[0] != 0 ? 1u : 0u) | (d[1] != 0 ? 2u : 0u);
            }
            if (__ballot_sync(0xffffffffu, m != 0)) locate_record<2>(d, m, v, 0, L);
        }
        unsigned long long x = acc_x(A) ^ acc_x(B), s = A.s + B.s, w = acc_w(A) + acc_w(B);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            x ^= __shfl_xor_sync(0xffffffffu, x, o);
            s += __shfl_xor_sync(0xffffffffu, s, o);
            w += __shfl_xor_sync(0xffffffffu, w, o);
        }
        if (lane == 0) { s_x[warp] = x; s_s[warp] = s; s_w[warp] = w; }
    } else {
        uint4* base = static_cast<uint4*>(wr.buf);
        const unsigned long long n_vec = wr.bytes >> 4, seed = wr.seed;
        const unsigned long long gw = (unsigned long long)blockIdx.x * wr.warps + (warp - rd.warps),
                                 nw = (unsigned long long)gridDim.x * wr.warps;
        const unsigned long long n_tiles = n_vec / tile_vecs;
        for (unsigned long long tile = gw; tile < n_tiles; tile += nw) {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const unsigned long long v = tile * tile_vecs + lane + (unsigned long long)j * 32;
                const unsigned long long a = pattern_word(seed, 2 * v), b = pattern_word(seed, 2 * v + 1);
                stg_stream(base + v, make_uint4((unsigned)a, (unsigned)(a >> 32), (unsigned)b, (unsigned)(b >> 32)));
            }
        }
        for (unsigned long long v = n_tiles * tile_vecs + gw * 32 + lane; v < n_vec; v += nw * 32) {
            const unsigned long long a = pattern_word(seed, 2 * v), b = pattern_word(seed, 2 * v + 1);
            stg_stream(base + v, make_uint4((unsigned)a, (unsigned)(a >> 32), (unsigned)b, (unsigned)(b >> 32)));
        }
    }
    const unsigned long long t_end = globaltimer_ns();
    if (lane == 0) {
        atomicMin(&s_t0[reader ? 0 : 1], t_start);
        atomicMax(&s_t1[reader ? 0 : 1], t_end);
    }
    __syncthreads();
    if (rd.warps && s_count) {          // CTA-uniform: read after the barrier
        if (threadIdx.x == 0) atomicAdd(&lb.ctr->mismatches, s_count);
        if (threadIdx.x < 64 && s_bits[threadIdx.x]) atomicAdd(&lb.ctr->bits[threadIdx.x], s_bits[threadIdx.x]);
    }
    if (threadIdx.x == 0 && rd.warps) {
        unsigned long long x = 0, s = 0, w = 0;
        for (unsigned k = 0; k < rd.warps; ++k) { x ^= s_x[k]; s += s_s[k]; w += s_w[k]; }
        link_publish(rd, x, s, w, s_t0[0], s_t1[0], stamp);
    }
    if (threadIdx.x == 32 * rd.warps && wr.warps) link_publish(wr, 0, 0, 0, s_t0[1], s_t1[1], stamp);
}

__global__ void force_words_kernel(unsigned long long* base, unsigned long long first, unsigned long long count,
                                   unsigned long long and_mask, unsigned long long or_mask) {
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < count;
         i += (unsigned long long)gridDim.x * blockDim.x)
        base[first + i] = (base[first + i] & and_mask) | or_mask;
}

// Consumer side shared by the TMA read kernel and the checksumming copy: folds
// one landed tile out of shared memory with conflict-free LDS.128.
// v_tile = index (in 16-byte vectors, relative to the sweep's base) of the tile's first vector.
// CMP (the comparing read): every word is also compared with its pattern word of `seed`, and *mism counts the ones
// that differ.
template <bool CMP = false>
__device__ __forceinline__ void fold_tile(Acc& A, Acc& B, const uint4* sp, unsigned nvec, unsigned ctid,
                                          unsigned n_cons, unsigned long long v_tile,
                                          unsigned long long seed = 0, unsigned long long* mism = nullptr) {
    unsigned i = ctid;
    // 4 independent LDS.128 per trip
    for (; i + 3 * n_cons < nvec; i += 4 * n_cons) {
        const uint4 a = sp[i], b = sp[i + n_cons], c = sp[i + 2 * n_cons], d = sp[i + 3 * n_cons];
        const unsigned long long m = 4 * (v_tile + i) + 1, step = 4ull * n_cons;
        fold2(A, lo64(a), hi64(a), m);
        fold2(B, lo64(b), hi64(b), m + step);
        fold2(A, lo64(c), hi64(c), m + 2 * step);
        fold2(B, lo64(d), hi64(d), m + 3 * step);
        if constexpr (CMP) {
            const unsigned long long lo[4] = {lo64(a), lo64(b), lo64(c), lo64(d)}, hi[4] = {hi64(a), hi64(b), hi64(c), hi64(d)};
            *mism += count_mismatches<4>(lo, hi, v_tile + i, n_cons, seed);
        }
    }
    for (; i < nvec; i += n_cons) {
        const uint4 a = sp[i];
        fold2(A, lo64(a), hi64(a), 4 * (v_tile + i) + 1);
        if constexpr (CMP) {
            const unsigned long long lo[1] = {lo64(a)}, hi[1] = {hi64(a)};
            *mism += count_mismatches<1>(lo, hi, v_tile + i, 0ull, seed);
        }
    }
}

// ---------------------------------------------------------------------------
// hbm_read (TMA path): warp 0 / lane 0 is the producer, issuing 1-D bulk
// copies of `tile_bytes` into a `stages`-deep shared-memory ring; the consumer
// warps fold each landed tile and hand the slot back through an "empty"
// mbarrier.  Bytes in flight per SM = stages*tile.  CMP: the consumers also
// compare every word (fold_tile<true>), as the LDG read does.
// ---------------------------------------------------------------------------
template <bool CMP>
__global__ void __launch_bounds__(1024, 1)
hbm_read_tma_kernel(const unsigned char* __restrict__ base, unsigned long long bytes,
                    unsigned tile_bytes, unsigned stages, unsigned chunk,
                    unsigned long long* tile_ctr, const ProbeParams imm, const ProbeParams* __restrict__ pp,
                    SweepScratch sc, SweepOut* out) {
    extern __shared__ __align__(128) unsigned char ring[];
    __shared__ __align__(8) uint64_t full_bar[16];
    __shared__ __align__(8) uint64_t empty_bar[16];
    __shared__ unsigned long long tile_of[16];
    const unsigned long long t_start = globaltimer_ns();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const unsigned n_cons_warps = (blockDim.x >> 5) - 1;
    const unsigned long long n_tiles = (bytes + tile_bytes - 1) / tile_bytes;
    const unsigned hint = chunk >> 16;   // bit 0: L2 evict_first on the loads
    chunk &= 0xFFFFu;
    const unsigned long long seed = CMP ? (pp ? pp->seed : imm.seed) : 0ull;
    unsigned long long mism = 0;

    if (threadIdx.x == 0) {
        for (unsigned s = 0; s < stages; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], n_cons_warps);
        }
        mbar_fence_init();
    }
    __syncthreads();

    Acc A, B;
    constexpr unsigned long long kEnd = ~0ull;
    if (warp == 0) {
        if (lane == 0) {
            // Producer.  Tiles come from a device-wide atomic counter (dynamic:
            // fast SMs take more tiles, the in-flight window stays compact) or
            // from static striding when tile_ctr is null.
            unsigned stage = 0, phase = 0;
            unsigned long long cur = 0, end = 0;   // claimed-but-unissued tiles [cur, end)
            for (unsigned long long k = 0;; ++k) {
                unsigned long long tile;
                if (tile_ctr) {
                    if (cur == end) { cur = atomicAdd(tile_ctr, (unsigned long long)chunk); end = cur + chunk; }
                    tile = cur++;
                } else {
                    tile = blockIdx.x + k * (unsigned long long)gridDim.x;
                }
                mbar_wait(&empty_bar[stage], phase ^ 1u);
                if (tile >= n_tiles) {
                    tile_of[stage] = kEnd;
                    mbar_arrive(&full_bar[stage]);      // completes the phase with no bytes
                    break;
                }
                tile_of[stage] = tile;
                const unsigned long long off = tile * tile_bytes;
                const unsigned long long left = bytes - off;
                const unsigned nb = left < tile_bytes ? (unsigned)left : tile_bytes;
                mbar_expect_tx(&full_bar[stage], nb);  // release: publishes tile_of[stage]
                if (hint & 1u)
                    tma_load_1d_hint(ring + (size_t)stage * tile_bytes, base + off, nb, &full_bar[stage],
                                     l2_policy_evict_first());
                else
                    tma_load_1d(ring + (size_t)stage * tile_bytes, base + off, nb, &full_bar[stage]);
                if (++stage == stages) { stage = 0; phase ^= 1u; }
            }
        }
    } else {
        const unsigned ctid = threadIdx.x - 32;
        const unsigned n_cons = n_cons_warps * 32;
        unsigned stage = 0, phase = 0;
        for (;;) {
            mbar_wait(&full_bar[stage], phase);
            const unsigned long long tile = *reinterpret_cast<volatile unsigned long long*>(&tile_of[stage]);
            if (tile == kEnd) break;
            const unsigned long long off = tile * tile_bytes;
            const unsigned long long left = bytes - off;
            const unsigned nvec = (left < tile_bytes ? (unsigned)left : tile_bytes) >> 4;
            fold_tile<CMP>(A, B, reinterpret_cast<const uint4*>(ring + (size_t)stage * tile_bytes), nvec, ctid, n_cons, off >> 4,
                           seed, &mism);
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty_bar[stage]);
            if (++stage == stages) { stage = 0; phase ^= 1u; }
        }
    }
    publish<true>(acc_x(A) ^ acc_x(B), A.s + B.s, acc_w(A) + acc_w(B), t_start, sc, out, imm, pp, bytes >> 3, mism);
}

// ---------------------------------------------------------------------------
// hbm_copy (LDG/STG path)
// ---------------------------------------------------------------------------
template <int THREADS, int UNROLL>
__global__ void __launch_bounds__(THREADS)
hbm_copy_ldg_kernel(uint4* __restrict__ dst, const uint4* __restrict__ src,
                    unsigned long long n_vec, const ProbeParams imm, const ProbeParams* __restrict__ pp,
                    SweepScratch sc, SweepOut* out) {
    unsigned long long t_start = 0;
    if (threadIdx.x == 0) t_start = globaltimer_ns();
    const unsigned long long tile_vecs = (unsigned long long)THREADS * UNROLL;
    const unsigned long long n_tiles = n_vec / tile_vecs;
    for (unsigned long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const unsigned long long o = tile * tile_vecs + threadIdx.x;
        static_assert(UNROLL == 8, "batched loader is written for 8 vectors per thread");
        unsigned long long a[8], b[8];
        ldg128_x8<THREADS * 16>(src + o, a, b);
#pragma unroll
        for (int j = 0; j < UNROLL; ++j)
            stg_stream(dst + o + j * THREADS,
                       make_uint4((unsigned)a[j], (unsigned)(a[j] >> 32), (unsigned)b[j],
                                  (unsigned)(b[j] >> 32)));
    }
    for (unsigned long long i = n_tiles * tile_vecs + (unsigned long long)blockIdx.x * THREADS +
                                threadIdx.x;
         i < n_vec; i += (unsigned long long)gridDim.x * THREADS)
        stg_stream(dst + i, ldg_stream(src + i));
    if (!out) return;
    __syncthreads();
    if (threadIdx.x == 0) publish_window(t_start, sc, out, imm, pp, 2 * n_vec);
}

// ---------------------------------------------------------------------------
// hbm_copy (TMA path): one thread per CTA drives everything.  Tiles go
// global -> smem (bulk load, mbarrier) -> global (bulk store, bulk group);
// data never touches the register file.  Moves bytes, checks nothing; the
// window it publishes ends once its last bulk store has completed.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(32, 1)
hbm_copy_tma_kernel(unsigned char* __restrict__ dst, const unsigned char* __restrict__ src,
                    unsigned long long bytes, unsigned tile_bytes, unsigned stages, unsigned chunk,
                    unsigned long long* tile_ctr, const ProbeParams imm, const ProbeParams* __restrict__ pp,
                    SweepScratch sc, SweepOut* out) {
    extern __shared__ __align__(128) unsigned char ring[];
    __shared__ __align__(8) uint64_t full_bar[16];
    __shared__ unsigned long long tile_of[16];
    if (threadIdx.x != 0) return;
    const unsigned long long t_start = globaltimer_ns();
    for (unsigned s = 0; s < stages; ++s) mbar_init(&full_bar[s], 1);
    mbar_fence_init();
    // bit 0: evict_first loads, bit 1: evict_first stores, bit 2: evict_last stores
    const unsigned hint = chunk >> 16;
    chunk &= 0xFFFFu;
    const uint64_t pol_first = l2_policy_evict_first(), pol_last = l2_policy_evict_last();

    const unsigned long long n_tiles = (bytes + tile_bytes - 1) / tile_bytes;
    unsigned long long fetched = 0;   // tiles this CTA has asked for
    bool dry = false;                 // the counter ran past the last tile
    unsigned long long cur = 0, end = 0;   // claimed-but-unissued tiles [cur, end)
    auto fetch = [&]() -> unsigned long long {
        unsigned long long t;
        if (tile_ctr) {
            if (cur == end) { cur = atomicAdd(tile_ctr, (unsigned long long)chunk); end = cur + chunk; }
            t = cur++;
        } else {
            t = blockIdx.x + fetched * (unsigned long long)gridDim.x;
        }
        ++fetched;
        if (t >= n_tiles) dry = true;
        return t;
    };
    auto tile_len = [&](unsigned long long off) {
        const unsigned long long left = bytes - off;
        return left < tile_bytes ? (unsigned)left : tile_bytes;
    };
    auto issue_load = [&](unsigned st, unsigned long long tile) {
        const unsigned long long off = tile * tile_bytes;
        const unsigned nb = tile_len(off);
        tile_of[st] = tile;
        mbar_expect_tx(&full_bar[st], nb);
        if (hint & 1u) tma_load_1d_hint(ring + (size_t)st * tile_bytes, src + off, nb, &full_bar[st], pol_first);
        else tma_load_1d(ring + (size_t)st * tile_bytes, src + off, nb, &full_bar[st]);
    };
    // prologue: fill the ring
    unsigned long long loaded = 0;
    for (unsigned s = 0; s < stages && !dry; ++s) {
        const unsigned long long t = fetch();
        if (!dry) { issue_load(s, t); ++loaded; }
    }
    for (unsigned long long k = 0; k < loaded; ++k) {
        const unsigned st = (unsigned)(k % stages);
        const unsigned phase = (unsigned)((k / stages) & 1ull);
        mbar_wait(&full_bar[st], phase);
        const unsigned long long off = tile_of[st] * tile_bytes;
        if (hint & 6u)
            tma_store_1d_hint(dst + off, ring + (size_t)st * tile_bytes, tile_len(off), (hint & 2u) ? pol_first : pol_last);
        else
            tma_store_1d(dst + off, ring + (size_t)st * tile_bytes, tile_len(off));
        tma_commit();
        // refill the slot whose store was issued one trip ago
        if (k >= 1 && !dry) {
            const unsigned long long t = fetch();
            if (!dry) {
                tma_wait_read<1>();   // all but the newest store have finished reading smem
                issue_load((unsigned)((k - 1) % stages), t);
                ++loaded;
            }
        }
    }
    tma_wait_all();
    if (out) publish_window(t_start, sc, out, imm, pp, bytes >> 3);
}

// ---------------------------------------------------------------------------
// hbm_copy, checksumming (the probe's default copy): the tile that the bulk
// load lands in shared memory is (1) handed to the bulk store and (2) folded
// by the consumer warps, both straight out of the same shared-memory slot.
// The sweep therefore yields the checksum of its SOURCE as actually read at
// no extra HBM traffic.  The probe runs its copy sweeps ping-pong (A->B, B->A,
// ...), so the fold of sweep k+1 is the verification of what sweep k WROTE.
// It compares no word: a multi-word fault the fold cannot see (DESIGN.md §3) is
// carried into every later copy, and the comparing read of that half finds it.
//   warp 0 lane 0: producer — claims tiles, issues bulk loads, issues the bulk
//                  store of a tile as soon as it has landed, refills a slot
//                  once both its store has read it (bulk-group wait) and the
//                  consumers have released it (empty mbarrier)
//   warps 1..n   : consumers — LDS.128 fold of each landed tile
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(1024, 1)
hbm_copy_fused_kernel(unsigned char* __restrict__ dst, const unsigned char* __restrict__ src,
                      unsigned long long bytes, unsigned tile_bytes, unsigned stages, unsigned chunk,
                      unsigned long long* tile_ctr, const ProbeParams imm, const ProbeParams* __restrict__ pp,
                      SweepScratch sc, SweepOut* out) {
    extern __shared__ __align__(128) unsigned char ring[];
    __shared__ __align__(8) uint64_t full_bar[16];
    __shared__ __align__(8) uint64_t empty_bar[16];
    __shared__ unsigned long long tile_of[16];
    const unsigned long long t_start = globaltimer_ns();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const unsigned n_cons_warps = (blockDim.x >> 5) - 1;
    const unsigned long long n_tiles = (bytes + tile_bytes - 1) / tile_bytes;
    chunk &= 0xFFFFu;

    if (threadIdx.x == 0) {
        for (unsigned s = 0; s < stages; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], n_cons_warps);
        }
        mbar_fence_init();
    }
    __syncthreads();

    Acc A, B;
    constexpr unsigned long long kEnd = ~0ull;
    if (warp == 0) {
        if (lane == 0) {
            unsigned long long fetched = 0;
            bool dry = false;
            unsigned long long cur = 0, end = 0;
            auto fetch = [&]() -> unsigned long long {
                unsigned long long t;
                if (tile_ctr) {
                    if (cur == end) { cur = atomicAdd(tile_ctr, (unsigned long long)chunk); end = cur + chunk; }
                    t = cur++;
                } else {
                    t = blockIdx.x + fetched * (unsigned long long)gridDim.x;
                }
                ++fetched;
                if (t >= n_tiles) dry = true;
                return t;
            };
            auto tile_len = [&](unsigned long long off) {
                const unsigned long long left = bytes - off;
                return left < tile_bytes ? (unsigned)left : tile_bytes;
            };
            // use number u of slot st (u-th tile through it): consumers must have released use u-1
            auto issue_load = [&](unsigned st, unsigned long long use, unsigned long long tile) {
                if (use > 0) mbar_wait(&empty_bar[st], (unsigned)((use - 1) & 1ull));
                const unsigned long long off = tile * tile_bytes;
                const unsigned nb = tile_len(off);
                tile_of[st] = tile;
                mbar_expect_tx(&full_bar[st], nb);   // release: publishes tile_of[st]
                tma_load_1d(ring + (size_t)st * tile_bytes, src + off, nb, &full_bar[st]);
            };
            unsigned long long loaded = 0;
            for (unsigned s = 0; s < stages && !dry; ++s) {
                const unsigned long long t = fetch();
                if (!dry) { issue_load(s, 0, t); ++loaded; }
            }
            for (unsigned long long k = 0; k < loaded; ++k) {
                const unsigned st = (unsigned)(k % stages);
                mbar_wait(&full_bar[st], (unsigned)((k / stages) & 1ull));
                const unsigned long long off = tile_of[st] * tile_bytes;
                tma_store_1d(dst + off, ring + (size_t)st * tile_bytes, tile_len(off));
                tma_commit();
                if (k >= 1 && !dry) {
                    const unsigned long long t = fetch();
                    if (!dry) {
                        tma_wait_read<1>();   // the store of trip k-1 has finished reading its slot
                        issue_load((unsigned)((k - 1) % stages), (k - 1) / stages + 1, t);
                        ++loaded;
                    }
                }
            }
            // tell the consumers there is nothing more: the slot after the last tile carries the end mark
            {
                const unsigned st = (unsigned)(loaded % stages);
                const unsigned long long use = loaded / stages;
                if (use > 0) {
                    // that slot's previous store must have drained before the mark reuses its barrier phase
                    mbar_wait(&empty_bar[st], (unsigned)((use - 1) & 1ull));
                }
                tile_of[st] = kEnd;
                mbar_arrive(&full_bar[st]);
            }
            tma_wait_all();
        }
    } else {
        const unsigned ctid = threadIdx.x - 32;
        const unsigned n_cons = n_cons_warps * 32;
        unsigned stage = 0, phase = 0;
        for (;;) {
            mbar_wait(&full_bar[stage], phase);
            const unsigned long long tile = *reinterpret_cast<volatile unsigned long long*>(&tile_of[stage]);
            if (tile == kEnd) break;
            const unsigned long long off = tile * tile_bytes;
            const unsigned long long left = bytes - off;
            const unsigned nvec = (left < tile_bytes ? (unsigned)left : tile_bytes) >> 4;
            fold_tile(A, B, reinterpret_cast<const uint4*>(ring + (size_t)stage * tile_bytes), nvec, ctid, n_cons, off >> 4);
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty_bar[stage]);
            if (++stage == stages) { stage = 0; phase ^= 1u; }
        }
    }
    publish(acc_x(A) ^ acc_x(B), A.s + B.s, acc_w(A) + acc_w(B), t_start, sc, out, imm, pp, bytes >> 3);
}

// ---------------------------------------------------------------------------
// hbm_expected: the checksum of the pattern from its closed form, no HBM.
// An independent generator: a fill or read bug cannot cancel out.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
hbm_expected_kernel(unsigned long long n_words, const ProbeParams imm,
                    const ProbeParams* __restrict__ pp, SweepScratch sc, SweepOut* out) {
    const unsigned long long seed = pp ? pp->seed : imm.seed;
    const unsigned long long t_start = globaltimer_ns();
    unsigned long long x = 0, s = 0, w = 0;
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
         i < n_words; i += (unsigned long long)gridDim.x * blockDim.x) {
        const unsigned long long v = pattern_word(seed, i);
        x ^= v; s += v; w += v * (2 * i + 1);
    }
    publish(x, s, w, t_start, sc, out, imm, pp, n_words);
}

__global__ void xor_words_kernel(unsigned long long* base, unsigned long long first, unsigned long long count,
                                 unsigned long long mask) {
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < count;
         i += (unsigned long long)gridDim.x * blockDim.x)
        base[first + i] ^= mask;
}

// Latency: dependent loads, system scope, one slot per 128-byte line.  Warp j
// (its lane 0) walks table j; the warps run concurrently, one outstanding load
// each, so n-1 peers are measured in the time of one chase.
__global__ void __launch_bounds__(32 * CRO_MAX_DEVICES)
chase_kernel(const ChaseArgs a, unsigned long long* __restrict__ out) {
    const unsigned j = threadIdx.x >> 5;
    if ((threadIdx.x & 31) != 0 || j >= a.n) return;
    const unsigned long long* next = a.table[j];
    if (!next) return;
    unsigned long long idx = a.start[j];
    // warm the TLB / first line
    {
        unsigned long long v;
        asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(next + idx * 16));
        if (v == ~0ull) out[2 * j] = v;   // keep the warm-up load alive
    }
    const unsigned long long t0 = globaltimer_ns();
    for (unsigned h = 0; h < a.hops; ++h) {
        unsigned long long v;
        asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(next + idx * 16));
        idx = v;
    }
    const unsigned long long t1 = globaltimer_ns();
    out[2 * j] = idx;
    out[2 * j + 1] = t1 - t0;
}

// ---------------------------------------------------------------------------
// finalize: the verdict, on the device.  One CTA; thread 0 does the (tiny)
// arithmetic after the CTA has copied the identity template.
// ---------------------------------------------------------------------------
__device__ __forceinline__ bool same_fold(const SweepOut& a, const SweepOut& b) {
    return a.x == b.x && a.s == b.s && a.w == b.w;
}
__device__ void best_and_median(const unsigned long long* t, unsigned n, unsigned long long* best,
                                unsigned long long* median) {
    unsigned long long v[kMaxSweepsEach];
    for (unsigned i = 0; i < n; ++i) {      // insertion sort, n <= 30
        unsigned long long x = t[i];
        unsigned k = i;
        while (k > 0 && v[k - 1] > x) { v[k] = v[k - 1]; --k; }
        v[k] = x;
    }
    *best = n ? v[0] : 0ull;
    *median = n ? v[n / 2] : 0ull;
}

__global__ void __launch_bounds__(128)
probe_finalize_kernel(const FinalizeArgs a) {
    // identity, options and whatever the host staged: 512 bytes, one uint4 per thread
    if (threadIdx.x < sizeof(cro_probe_result) / 16)
        reinterpret_cast<uint4*>(a.out)[threadIdx.x] = reinterpret_cast<const uint4*>(a.tmpl)[threadIdx.x];
    __syncthreads();
    if (threadIdx.x != 0) return;
    cro_probe_result* r = a.out;
    const SweepOut* sl = a.slots;
    const unsigned long long nonce = a.pp->nonce;
    const unsigned long long n_words = a.sweep_bytes >> 3;
    const unsigned C = a.copy_sweeps, R = a.read_sweeps;
    const SweepOut& E = sl[kSlotExpect];
    int status = CRO_OK;
    unsigned fail_code = CRO_FAIL_NONE, fail_index = 0;
    auto fail = [&](unsigned code, unsigned index) {
        if (status == CRO_OK) { status = CRO_ERR_CHECKSUM; fail_code = code; fail_index = index; }
    };
    r->seed = a.pp->seed;
    r->nonce = (uint32_t)nonce;
    r->sweep_bytes = a.sweep_bytes;
    r->read_sweeps = (uint8_t)R;
    r->copy_sweeps = (uint8_t)C;
    r->read_variant = (uint8_t)a.read_variant;
    r->copy_variant = (uint8_t)a.copy_variant;
    r->expect_xor = E.x; r->expect_sum = E.s; r->expect_wsum = E.w;
    if (E.stamp != nonce || E.n_words != n_words) fail(CRO_FAIL_EXPECT, 0);
    if (sl[kSlotFill].stamp != nonce || sl[kSlotFill].n_words != n_words) fail(CRO_FAIL_STALE, 0);

    unsigned long long tc[kMaxSweepsEach], tr[kMaxSweepsEach];
    unsigned verified = 0;
    // every copy publishes its slot: a stale one did not run.  The checksumming copy i also folds what sweep i-1 wrote
    // (sweep 0 reads the fill): its fold IS the check of that data.  A plain copy's data is checked by the next sweep.
    for (unsigned i = 0; i < C; ++i) {
        const SweepOut& s = sl[kSlotSweep0 + i];
        tc[i] = s.t1 - s.t0;
        if (s.stamp != nonce || s.n_words != n_words) fail(CRO_FAIL_STALE, 1 + i);
        else if (!a.fused) continue;
        else if (!same_fold(s, E)) fail(CRO_FAIL_COPY_SRC, i);
        else if (i > 0) ++verified;            // sweep i-1's destination reproduced the pattern
    }
    // read sweep 0 reads the last copy's destination.  A read also compares every word: its fold can match while words
    // differ (a multi-word fault that cancels in the fold, carried through every copy), and then its count does not.
    const SweepOut* shown = &sl[kSlotSweep0 + C];
    for (unsigned i = 0; i < R; ++i) {
        const SweepOut& s = sl[kSlotSweep0 + C + i];
        tr[i] = s.t1 - s.t0;
        bool ok = true;
        if (s.stamp != nonce || s.n_words != n_words) { if (status == CRO_OK) shown = &s; fail(CRO_FAIL_STALE, 1 + C + i); ok = false; }
        else if (!same_fold(s, E) || s.mismatches != 0) { if (status == CRO_OK) shown = &s; fail(CRO_FAIL_READ, i); ok = false; }
        if (i == 0 && ok && C > 0) ++verified;
    }
    r->checksum_xor = shown->x; r->checksum_sum = shown->s; r->checksum_wsum = shown->w;
    if (C > 0 && R > 0) {
        const SweepOut& d = sl[kSlotSweep0 + C];
        r->copy_checksum_xor = d.x; r->copy_checksum_sum = d.s; r->copy_checksum_wsum = d.w;
    }
    r->copy_verified = (uint8_t)verified;
    r->fill_ns = sl[kSlotFill].t1 - sl[kSlotFill].t0;
    unsigned long long best, med;
    best_and_median(tr, R, &best, &med);
    r->read_best_ns = best; r->read_median_ns = med;
    best_and_median(tc, C, &best, &med);
    r->copy_best_ns = best; r->copy_median_ns = med;
    unsigned long long t_end = sl[kSlotFill].t1;
    for (unsigned i = 0; i < C + R; ++i) t_end = sl[kSlotSweep0 + i].t1 > t_end ? sl[kSlotSweep0 + i].t1 : t_end;
    r->t_start_ns = sl[kSlotFill].t0;
    r->total_ns = t_end - sl[kSlotFill].t0;
    r->fail_code = (uint8_t)fail_code;
    r->fail_index = (uint8_t)fail_index;
    r->status = status;
}

__global__ void __launch_bounds__(32)
p2p_finalize_kernel(const P2PFinalizeArgs a) {
    if (threadIdx.x != 0) return;
    cro_probe_result* r = a.out;
    int status = r->status;
    unsigned fail_code = r->fail_code, fail_index = r->fail_index;
    auto fail = [&](unsigned code, unsigned index) {
        if (status == CRO_OK) { status = CRO_ERR_CHECKSUM; fail_code = code; fail_index = index; }
    };
    unsigned ok_mask = 0;
    r->p2p_bytes = a.p2p_bytes;
    for (unsigned j = 0; j < a.n && j < 8; ++j) {
        if (j == a.self || !r->p2p_access[j] || !a.peer_slots[j]) continue;
        bool ok = true;
        const SweepOut& rd = a.slots[kSlotP2P0 + 3 * j];
        // what the owner itself says its first p2p_bytes must fold to (its closed-form slot, read over NVLink)
        const SweepOut want = a.peer_slots[j][kSlotPrefix];
        r->p2p_read_ns[j] = rd.t1 - rd.t0;
        r->p2p_checksum_xor[j] = rd.x;
        if (want.stamp != a.peer_stamp[j] || want.n_words != (a.p2p_bytes >> 3)) { fail(CRO_FAIL_EXPECT, j); ok = false; }
        if (rd.stamp != a.stamp || !same_fold(rd, want)) { fail(CRO_FAIL_P2P_READ, j); ok = false; }
        const SweepOut& ps = a.slots[kSlotP2P0 + 3 * j + 1];          // my push into j (fold of my own prefix as read)
        if (ps.stamp == a.stamp) r->p2p_write_ns[j] = ps.t1 - ps.t0;
        if (a.have_push) {
            const SweepOut& rr = a.slots[kSlotP2P0 + 3 * j + 2];      // my re-read of what j pushed into me
            const SweepOut mine = a.slots[kSlotPrefix];
            if (a.push_folded && (ps.stamp != a.stamp || !same_fold(ps, mine))) { fail(CRO_FAIL_P2P_PUSH, j); ok = false; }
            if (rr.stamp != a.stamp || !same_fold(rr, want)) { fail(CRO_FAIL_P2P_PUSH, j); ok = false; }
        }
        if (a.hops) {
            const unsigned long long end = a.chase_out[2 * j], ns = a.chase_out[2 * j + 1];
            // ns * 16 would wrap at 2^60 ns and up; such a chase saturates the 32-bit field anyway (hops < 2^32)
            const unsigned long long x16 = ns > (~0ull >> 4) ? ~0ull : ns * 16ull / a.hops;
            r->p2p_latency_ns_x16[j] = (uint32_t)(x16 > 0xFFFFFFFFull ? 0xFFFFFFFFull : x16);
            if (end != a.chase_expect[j]) { fail(CRO_FAIL_P2P_CHASE, j); ok = false; }
        }
        if (ok) ok_mask |= 1u << j;
    }
    r->p2p_ok = (uint8_t)ok_mask;
    r->fail_code = (uint8_t)fail_code;
    r->fail_index = (uint8_t)fail_index;
    r->status = status;
}

// ---------------------------------------------------------------------------
// compute_probe: every SM computes the answer tile D = A * B (M x N x K of
// include/croprobe.h) `iterations` times from operands it generates into its own
// shared memory, and checks what it got (the compute probe, cro_probe_compute;
// not part of the HBM probe).  One template per leg:
//   S8, BF16, E4M3   wgmma.mma_async m64n256 (IGMMA / HGMMA / QGMMA), each of the
//                    two warpgroups owning 64 rows, chained over K with scale-d = 0
//                    on the first instruction of every iteration
//   FFMA, IMAD       the same accumulator fragment computed by scalar FMA / IMAD
//                    chains on the CUDA cores
// Operands sit in the canonical K-major no-swizzle layout the wgmma shared-memory
// descriptors read (kmajor_off, sm_tile.cuh).  B is held transposed (N rows of K),
// as the K-major form requires.
// After each iteration every thread adds sum_j value_j * (2j + 1) to a running
// fold (float values after cvt.rni.s32.f32); at the end it compares the fold with
// iterations * the fold of the expected values, and the last answer element by
// element with the expected tile (global memory, L2-resident, shared by all CTAs).
// Mismatches are recorded with the locator's idiom: a ballot keeps clean warps off
// the atomics, one atomicAdd per warp claims a run of record slots, and only while
// a plain load shows room.
// ---------------------------------------------------------------------------
constexpr unsigned kCM = CRO_COMPUTE_M, kCN = CRO_COMPUTE_N, kCK = CRO_COMPUTE_K;
constexpr size_t kComputeSmem = (size_t)(kCM + kCN) * kCK * 2;     // the bf16 operands: 192 KiB, one CTA per SM

template <unsigned LEG> struct ComputeLeg {
    static constexpr bool kTensor = LEG <= CRO_COMPUTE_LEG_E4M3;
    static constexpr bool kFloat = LEG == CRO_COMPUTE_LEG_BF16 || LEG == CRO_COMPUTE_LEG_E4M3 || LEG == CRO_COMPUTE_LEG_FFMA;
    static constexpr unsigned kElem = (LEG == CRO_COMPUTE_LEG_BF16 || LEG == CRO_COMPUTE_LEG_FFMA) ? 2 : 1;   // bytes
    using Acc = typename std::conditional<kFloat, float, int>::type;
};

SM_TILE_WGMMA(wgmma_s8, int, 128, "+r", "m64n256k32.s32.s8.s8", "")
SM_TILE_WGMMA(wgmma_bf16, float, 128, "+f", "m64n256k16.f32.bf16.bf16", ", 1, 1, 0, 0")
SM_TILE_WGMMA(wgmma_e4m3, float, 128, "+f", "m64n256k32.f32.e4m3.e4m3", ", 1, 1")

// The operand byte read as each leg's element type: s8 as int8; small-int (byte & 7) - 4 as bf16 or e4m3.
template <unsigned LEG>
__device__ __forceinline__ void store_operand(unsigned char* p, unsigned byte) {
    if constexpr (LEG == CRO_COMPUTE_LEG_S8 || LEG == CRO_COMPUTE_LEG_IMAD) {
        *p = (unsigned char)byte;
    } else if constexpr (LEG == CRO_COMPUTE_LEG_E4M3) {
        *p = (unsigned char)__nv_cvt_float_to_fp8((float)((int)(byte & 7u) - 4), __NV_SATFINITE, __NV_E4M3);
    } else {
        *reinterpret_cast<__nv_bfloat16*>(p) = __float2bfloat16_rn((float)((int)(byte & 7u) - 4));
    }
}

template <unsigned LEG>
__device__ __forceinline__ int compute_value(typename ComputeLeg<LEG>::Acc v) {
    if constexpr (ComputeLeg<LEG>::kFloat) return __float2int_rn(v);      // cvt.rni.s32.f32: exact for these integers
    else return v;
}

// Element k (0 .. 16 / ELEM - 1) of 16 operand bytes, as the ALU legs multiply it.
template <unsigned LEG>
__device__ __forceinline__ typename ComputeLeg<LEG>::Acc alu_elem(const unsigned (&w)[4], int k) {
    if constexpr (LEG == CRO_COMPUTE_LEG_FFMA) {
        const unsigned x = w[k >> 1];
        return __uint_as_float((k & 1) ? (x & 0xFFFF0000u) : (x << 16));
    } else {
        return (int)(signed char)(w[k >> 2] >> (8 * (k & 3)));
    }
}

// Records the warp's mismatching elements of chunk C (accumulator values 32 C .. 32 C + 31; bit q of m: value
// 32 C + q mismatches).  The whole warp calls this (some lane has m != 0).
template <unsigned LEG, int C>
__device__ __forceinline__ void compute_record(const typename ComputeLeg<LEG>::Acc (&acc)[128], unsigned m, unsigned r0,
                                               unsigned c0, unsigned smid, const ComputeArgs& a) {
    unsigned long long base = warp_claim(__popc(m), a.claims, CRO_COMPUTE_RECORDS, [](unsigned) {});
#pragma unroll
    for (int q = 0; q < 32; ++q) {
        const int j = 32 * C + q;
        if (!((m >> q) & 1u)) continue;
        if (base < CRO_COMPUTE_RECORDS) {
            const unsigned row = r0 + 8u * ((j >> 1) & 1), col = 8u * (j >> 2) + c0 + (j & 1);
            a.rec[base] = cro_compute_fault{LEG, smid, row, col, __ldg(a.expect + row * kCN + col),
                                            compute_value<LEG>(acc[j])};
        }
        ++base;
    }
}

template <unsigned LEG, int C>
__device__ __forceinline__ unsigned compute_compare(const typename ComputeLeg<LEG>::Acc (&acc)[128], unsigned r0, unsigned c0,
                                                    unsigned smid, const ComputeArgs& a, unsigned long long* efold) {
    unsigned m = 0;
#pragma unroll
    for (int q = 0; q < 32; ++q) {
        const int j = 32 * C + q;
        const unsigned row = r0 + 8u * ((j >> 1) & 1), col = 8u * (j >> 2) + c0 + (j & 1);
        const int e = __ldg(a.expect + row * kCN + col);
        *efold += (unsigned long long)(long long)e * (unsigned long long)(2 * j + 1);
        if (compute_value<LEG>(acc[j]) != e) m |= 1u << q;
    }
    if (__ballot_sync(0xffffffffu, m != 0)) compute_record<LEG, C>(acc, m, r0, c0, smid, a);
    return __popc(m);
}

template <unsigned LEG>
__global__ void __launch_bounds__(kComputeThreads, 1) compute_probe_kernel(const ComputeArgs a) {
    using L = ComputeLeg<LEG>;
    using Acc = typename L::Acc;
    constexpr unsigned ELEM = L::kElem;
    extern __shared__ __align__(128) unsigned char cmp_smem[];
    __shared__ unsigned long long s_mism, s_fold_mism, s_fold;
    unsigned char* const sA = cmp_smem;
    unsigned char* const sB = cmp_smem + kCM * kCK * ELEM;
    const unsigned tid = threadIdx.x;
    if (tid == 0) s_mism = s_fold_mism = s_fold = 0;

    // operands: element e is byte e % 8 of pattern_word(seed, e / 8); A[m][k] at e = m * K + k, B[k][n] at
    // e = M * K + k * N + n
    for (unsigned w = tid; w < (kCM * kCK + kCK * kCN) / 8; w += kComputeThreads) {
        const unsigned long long v = pattern_word(a.seed, w);
#pragma unroll
        for (unsigned b = 0; b < 8; ++b) {
            const unsigned e = 8 * w + b;
            const unsigned byte = (unsigned)(v >> (8 * b)) & 0xFFu;
            if (e < kCM * kCK) store_operand<LEG>(sA + kmajor_off<ELEM, kCK>(e / kCK, e % kCK), byte);
            else store_operand<LEG>(sB + kmajor_off<ELEM, kCK>((e - kCM * kCK) % kCN, (e - kCM * kCK) / kCN), byte);
        }
    }
    if constexpr (L::kTensor) asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");
    __syncthreads();

    unsigned smid, nsmid;
    asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
    asm volatile("mov.u32 %0, %%nsmid;" : "=r"(nsmid));
    const unsigned wg = tid >> 7, lane = tid & 31u;
    const unsigned r0 = 64u * wg + 16u * ((tid >> 5) & 3u) + (lane >> 2), c0 = 2u * (lane & 3u);
    const Injection inj = resolve_injection(a, r0, smid);

    Acc acc[128];
#pragma unroll
    for (int j = 0; j < 128; ++j) acc[j] = 0;
    unsigned long long run = 0;
    const unsigned long long t0 = globaltimer_ns();
    const long long k0 = clock64();
    for (unsigned it = 0; it < a.iterations; ++it) {
        if constexpr (L::kTensor) {
            constexpr unsigned SBO = 8u * kCK * ELEM;
            const unsigned long long da = wgmma_desc(smem_u32(sA) + wg * 64u * kCK * ELEM, SBO);
            const unsigned long long db = wgmma_desc(smem_u32(sB), SBO);
            asm volatile("wgmma.fence.sync.aligned;\n" ::: "memory");
#pragma unroll
            for (unsigned s = 0; s < kCK * ELEM / 32; ++s) {      // 32 bytes of K per instruction: +256 bytes, >> 4
                if constexpr (LEG == CRO_COMPUTE_LEG_S8) wgmma_s8(acc, da + 16u * s, db + 16u * s, s != 0);
                else if constexpr (LEG == CRO_COMPUTE_LEG_BF16) wgmma_bf16(acc, da + 16u * s, db + 16u * s, s != 0);
                else wgmma_e4m3(acc, da + 16u * s, db + 16u * s, s != 0);
            }
            asm volatile("wgmma.commit_group.sync.aligned;\n" ::: "memory");
            asm volatile("wgmma.wait_group.sync.aligned 0;\n" ::: "memory");
#pragma unroll
            for (int j = 0; j < 128; ++j) {
                if constexpr (L::kFloat) asm volatile("" : "+f"(acc[j])::"memory");
                else asm volatile("" : "+r"(acc[j])::"memory");
            }
        } else {
#pragma unroll
            for (int j = 0; j < 128; ++j) acc[j] = 0;
            constexpr int KC = 16 / ELEM;                          // elements per 16-byte core-matrix row
#pragma unroll 1
            for (unsigned kc = 0; kc < kCK; kc += KC) {
                const uint4 x0 = *reinterpret_cast<const uint4*>(sA + kmajor_off<ELEM, kCK>(r0, kc));
                const uint4 x1 = *reinterpret_cast<const uint4*>(sA + kmajor_off<ELEM, kCK>(r0 + 8, kc));
                const unsigned a0[4] = {x0.x, x0.y, x0.z, x0.w}, a1[4] = {x1.x, x1.y, x1.z, x1.w};
#pragma unroll
                for (int g = 0; g < 32; ++g) {
                    const uint4 y0 = *reinterpret_cast<const uint4*>(sB + kmajor_off<ELEM, kCK>(8u * g + c0, kc));
                    const uint4 y1 = *reinterpret_cast<const uint4*>(sB + kmajor_off<ELEM, kCK>(8u * g + c0 + 1, kc));
                    const unsigned b0[4] = {y0.x, y0.y, y0.z, y0.w}, b1[4] = {y1.x, y1.y, y1.z, y1.w};
#pragma unroll
                    for (int k = 0; k < KC; ++k) {
                        const Acc p = alu_elem<LEG>(a0, k), q = alu_elem<LEG>(a1, k);
                        const Acc u = alu_elem<LEG>(b0, k), v = alu_elem<LEG>(b1, k);
                        if constexpr (L::kFloat) {
                            acc[4 * g] = fmaf(p, u, acc[4 * g]);
                            acc[4 * g + 1] = fmaf(p, v, acc[4 * g + 1]);
                            acc[4 * g + 2] = fmaf(q, u, acc[4 * g + 2]);
                            acc[4 * g + 3] = fmaf(q, v, acc[4 * g + 3]);
                        } else {
                            acc[4 * g] += p * u;
                            acc[4 * g + 1] += p * v;
                            acc[4 * g + 2] += q * u;
                            acc[4 * g + 3] += q * v;
                        }
                    }
                }
            }
        }
        if (it == inj.iter) {                                        // test only: one compare on the clean path
#pragma unroll
            for (int j = 0; j < 128; ++j) {
                const unsigned col = 8u * (j >> 2) + c0 + (j & 1);
                if (((inj.rows >> ((j >> 1) & 1)) & 1u) && (a.inj_col < 0 || (unsigned)a.inj_col == col)) {
                    if constexpr (L::kFloat) acc[j] = __uint_as_float(__float_as_uint(acc[j]) ^ a.inj_mask);
                    else acc[j] ^= (int)a.inj_mask;
                }
            }
        }
        __syncwarp();
        unsigned long long f = 0;
#pragma unroll
        for (int j = 0; j < 128; ++j)
            f += (unsigned long long)(long long)compute_value<LEG>(acc[j]) * (unsigned long long)(2 * j + 1);
        run += f;
    }
    const long long k1 = clock64();
    const unsigned long long t1 = globaltimer_ns();

    unsigned long long efold = 0;
    unsigned mism = compute_compare<LEG, 0>(acc, r0, c0, smid, a, &efold);
    mism += compute_compare<LEG, 1>(acc, r0, c0, smid, a, &efold);
    mism += compute_compare<LEG, 2>(acc, r0, c0, smid, a, &efold);
    mism += compute_compare<LEG, 3>(acc, r0, c0, smid, a, &efold);
    const unsigned fold_bad = run != (unsigned long long)a.iterations * efold ? 1u : 0u;
    publish_cta<CRO_COMPUTE_MAX_SMS>(a, mism, fold_bad, run, t0, t1, k0, k1, smid, nsmid, s_mism, s_fold_mism, s_fold);
}

// ---------------------------------------------------------------------------
// host side: plan + launch wrappers
// ---------------------------------------------------------------------------
namespace {
constexpr int kFillThreads = 512, kFillUnroll = 4;
constexpr int kReadThreads = 512;
constexpr int kCopyThreads = 512, kCopyUnroll = 8;
// Grid of the host link probe's SM legs (8 warps per role and CTA): see DESIGN.md "host link" for the measurement.
constexpr int kLinkDefaultCtas = 32;
}  // namespace

cudaError_t plan_kernels(int device, const env::Values& knobs, KernelPlan* plan, std::string* why) {
    cudaError_t e;
    int sms = 0, optin = 0;
    if ((e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device)) != cudaSuccess)
        return e;
    if ((e = cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device)) != cudaSuccess)
        return e;
    plan->sm_count = sms;
    int occ = 0;
    auto knob = [&](const char* name) { return knobs.get(name); };

    auto fill = hbm_fill_kernel<kFillThreads, kFillUnroll>;
    if ((e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, fill, kFillThreads, 0)) != cudaSuccess)
        return e;
    plan->fill = {sms * (occ > 0 ? occ : 1) * (int)knob("CRO_FILL_WAVES"), kFillThreads, 0};

    auto rd = hbm_read_ldg_kernel<kReadThreads, false, true>;
    if ((e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, rd, kReadThreads, 0)) != cudaSuccess)
        return e;
    plan->read_ldg = {sms * (occ > 0 ? occ : 1) * (int)knob("CRO_READ_WAVES"), kReadThreads, 0};
    auto rdw = hbm_read_ldg_kernel<kReadThreads, true, true>;
    if ((e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, rdw, kReadThreads, 0)) != cudaSuccess)
        return e;
    plan->read_ldg256 = {sms * (occ > 0 ? occ : 1) * (int)knob("CRO_READ_WAVES"), kReadThreads, 0};
    auto loc = hbm_locate_kernel<kReadThreads>;
    if ((e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, loc, kReadThreads, 0)) != cudaSuccess)
        return e;
    plan->locate = {sms * (occ > 0 ? occ : 1) * (int)knob("CRO_READ_WAVES"), kReadThreads, 0};
    plan->link_grid = kLinkDefaultCtas;

    auto cp = hbm_copy_ldg_kernel<kCopyThreads, kCopyUnroll>;
    if ((e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, cp, kCopyThreads, 0)) != cudaSuccess)
        return e;
    plan->copy_ldg = {sms * (occ > 0 ? occ : 1) * (int)knob("CRO_COPY_WAVES"), kCopyThreads, 0};

    // A ring kernel's dynamic shared-memory ceiling belongs to the function in the whole process, not to a context: it
    // is set to everything the device lets a CTA own beside the kernel's static shared memory, the same value for every
    // context, so a context planned with a small ring cannot shrink it under another one's larger ring.  Launches and
    // occupancy use the context's own ring.  A ring that does not fit, or fits no CTA on an SM, is refused by its tile
    // knob.
    auto plan_ring = [&](const void* fn, const char* tile_knob, size_t ring, int threads) -> cudaError_t {
        cudaFuncAttributes fa;
        cudaError_t r;
        if ((r = cudaFuncGetAttributes(&fa, fn)) != cudaSuccess) return r;
        const size_t room = (size_t)optin > fa.sharedSizeBytes ? (size_t)optin - fa.sharedSizeBytes : 0;
        if (ring > room) {
            *why = env::refusal(tile_knob, std::to_string(knob(tile_knob)));
            return cudaErrorInvalidValue;
        }
        if ((r = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)room)) != cudaSuccess) return r;
        if ((r = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, fn, threads, ring)) != cudaSuccess) return r;
        if (occ < 1) {
            *why = env::refusal(tile_knob, std::to_string(knob(tile_knob)));
            return cudaErrorInvalidValue;
        }
        return cudaSuccess;
    };
    {
        plan->read_tile = knob("CRO_TMA_READ_TILE");
        plan->read_stages = knob("CRO_TMA_READ_STAGES");
        plan->read_chunk = (knob("CRO_TMA_READ_CHUNK") & 0xFFFFu) | (knob("CRO_TMA_READ_HINT") << 16);
        plan->read_dyn = knob("CRO_TMA_READ_DYN");
        const int threads = (int)knob("CRO_TMA_READ_THREADS");
        const size_t smem = (size_t)plan->read_tile * plan->read_stages;
        // both instances: the comparing one sets the occupancy the grid is planned for
        if ((e = plan_ring((const void*)hbm_read_tma_kernel<false>, "CRO_TMA_READ_TILE", smem, threads)) != cudaSuccess ||
            (e = plan_ring((const void*)hbm_read_tma_kernel<true>, "CRO_TMA_READ_TILE", smem, threads)) != cudaSuccess)
            return e;
        plan->read_tma = {sms * occ * (int)knob("CRO_TMA_READ_WAVES"), threads, smem};
    }
    {
        plan->copy_tile = knob("CRO_TMA_COPY_TILE");
        plan->copy_stages = knob("CRO_TMA_COPY_STAGES");
        plan->copy_chunk = (knob("CRO_TMA_COPY_CHUNK") & 0xFFFFu) | (knob("CRO_TMA_COPY_HINT") << 16);
        plan->copy_dyn = knob("CRO_TMA_COPY_DYN");
        const size_t smem = (size_t)plan->copy_tile * plan->copy_stages;
        if ((e = plan_ring((const void*)hbm_copy_tma_kernel, "CRO_TMA_COPY_TILE", smem, 32)) != cudaSuccess)
            return e;
        plan->copy_tma = {sms * occ * (int)knob("CRO_TMA_COPY_WAVES"), 32, smem};
    }
    {
        plan->fused_tile = knob("CRO_FUSED_TILE");
        plan->fused_stages = knob("CRO_FUSED_STAGES");
        plan->fused_chunk = knob("CRO_FUSED_CHUNK") & 0xFFFFu;
        plan->fused_threads = knob("CRO_FUSED_THREADS");
        const size_t smem = (size_t)plan->fused_tile * plan->fused_stages;
        if ((e = plan_ring((const void*)hbm_copy_fused_kernel, "CRO_FUSED_TILE", smem, (int)plan->fused_threads)) != cudaSuccess)
            return e;
        plan->copy_fused = {sms * occ, (int)plan->fused_threads, smem};
    }
    // An SM changes its L1 / shared-memory split only when it is empty, so a kernel that asks for the default split
    // keeps the copy's CTA (128 KiB of shared memory) off every SM it occupies, and the first copy sweep waits for the
    // whole generator.  The generator and the kernels it may run beside therefore ask for the SAME split, the largest
    // shared memory.  That includes the fill: in cro_probe_all it runs beside the generator of the NVLink prefix.  Not
    // the LDG kernels: they never run beside a generator, and they want the L1 the smallest split would take away.
    for (const void* fn : {(const void*)hbm_expected_kernel, (const void*)hbm_read_tma_kernel<false>,
                           (const void*)hbm_read_tma_kernel<true>, (const void*)hbm_copy_fused_kernel,
                           (const void*)hbm_copy_tma_kernel, (const void*)probe_finalize_kernel})
        if ((e = cudaFuncSetAttribute(fn, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared)) != cudaSuccess)
            return e;
    if (knob("CRO_CARVEOUT_FILL"))     // the fill: it does run beside a generator in cro_probe_all (the p2p prefix's)
        if ((e = cudaFuncSetAttribute((const void*)hbm_fill_kernel<kFillThreads, kFillUnroll>, cudaFuncAttributePreferredSharedMemoryCarveout,
                                      cudaSharedmemCarveoutMaxShared)) != cudaSuccess)
            return e;
    if ((e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, hbm_expected_kernel, 256, 0)) !=
        cudaSuccess)
        return e;
    // The generator runs BESIDE the copy sweeps: it may not fill the SM, or the copy's CTA (160 threads, 128 KiB of
    // shared memory) would have to wait for it to drain; and the fewer of its warps compete with the copy's consumer
    // warps for issue slots the better: one CTA of 256 threads per SM by default (CRO_EXPECT_CTAS).
    plan->expect = {sms * std::min<int>(occ > 0 ? occ : 1, (int)knob("CRO_EXPECT_CTAS")), 256, 0};
    return cudaSuccess;
}

// No more CTAs than there are tiles: a small sweep should not pay for a grid sized for 4 GiB.
static int clamp_grid(int planned, uint64_t bytes, uint64_t tile_bytes) {
    const uint64_t tiles = (bytes + tile_bytes - 1) / tile_bytes;
    return (int)std::max<uint64_t>(1, std::min<uint64_t>((uint64_t)planned, tiles));
}

cudaError_t launch_fill(const KernelPlan& p, void* base, uint64_t bytes, const Params& pr,
                        const SweepScratch& sc, SweepOut* out, cudaStream_t st, bool invert) {
    // Few tiles per CTA: with a fixed grid a 16 GiB fill strides 14 tiles per CTA, the SMs drift apart and the DRAM
    // window spreads and the rate drops as the sweep grows; the grid therefore grows with the sweep.
    constexpr uint64_t kTile = (uint64_t)kFillThreads * kFillUnroll * 16;
    const uint64_t tiles = (bytes + kTile - 1) / kTile;
    const int planned = (int)std::min<uint64_t>(std::max<uint64_t>((uint64_t)p.fill.grid, tiles / 4), 0x7FFFFFFFull);
    if (invert)
        hbm_fill_kernel<kFillThreads, kFillUnroll, true><<<clamp_grid(planned, bytes, kTile), p.fill.block, 0, st>>>(
            static_cast<uint4*>(base), bytes >> 4, pr.imm, pr.pp, sc, out);
    else
        hbm_fill_kernel<kFillThreads, kFillUnroll><<<clamp_grid(planned, bytes, kTile), p.fill.block, 0, st>>>(
            static_cast<uint4*>(base), bytes >> 4, pr.imm, pr.pp, sc, out);
    return cudaGetLastError();
}

cudaError_t launch_locate(const KernelPlan& p, const void* half, uint64_t bytes, uint64_t word0, uint64_t seed,
                          uint64_t invert, const LocateBufs& lb, const SweepScratch& sc, SweepOut* out, cudaStream_t st) {
    hbm_locate_kernel<kReadThreads><<<clamp_grid(p.locate.grid, bytes, kReadThreads * 128), p.locate.block, 0, st>>>(
        static_cast<const uint4*>(half), bytes >> 4, word0, seed, invert, lb, ProbeParams{seed, 0}, sc, out);
    return cudaGetLastError();
}

cudaError_t launch_force_words(void* base, uint64_t first, uint64_t count, uint64_t and_mask, uint64_t or_mask,
                               int sm_count, cudaStream_t st) {
    if (count == 0) return cudaSuccess;
    const uint64_t blocks = std::min<uint64_t>((count + 255) / 256, (uint64_t)std::max(sm_count, 1) * 8);
    force_words_kernel<<<(unsigned)blocks, 256, 0, st>>>(static_cast<unsigned long long*>(base), first, count, and_mask,
                                                        or_mask);
    return cudaGetLastError();
}

cudaError_t launch_link_stream(const LinkRole& rd, const LinkRole& wr, const LocateBufs& lb, int grid, uint64_t stamp,
                               cudaStream_t st) {
    if ((rd.warps != 0 && rd.warps != kLinkWarps) || (wr.warps != 0 && wr.warps != kLinkWarps) || !(rd.warps | wr.warps) ||
        grid < 1)
        return cudaErrorInvalidValue;
    link_stream_kernel<<<grid, 32 * (rd.warps + wr.warps), 0, st>>>(rd, wr, lb, stamp);
    return cudaGetLastError();
}

cudaError_t launch_read(const KernelPlan& p, unsigned variant, const void* base, uint64_t bytes,
                        const Params& pr, const SweepScratch& sc, SweepOut* out, cudaStream_t st, bool compare) {
    if (variant == READ_TMA) {
        auto k = compare ? hbm_read_tma_kernel<true> : hbm_read_tma_kernel<false>;
        k<<<clamp_grid(p.read_tma.grid, bytes, p.read_tile), p.read_tma.block, p.read_tma.smem, st>>>(
            static_cast<const unsigned char*>(base), bytes, p.read_tile, p.read_stages, p.read_chunk,
            (p.read_dyn && sc.tile_ctr) ? sc.tile_ctr : nullptr, pr.imm, pr.pp, sc, out);
    } else {
        const bool wide = variant == READ_LDG256;
        auto k = wide ? (compare ? hbm_read_ldg_kernel<kReadThreads, true, true> : hbm_read_ldg_kernel<kReadThreads, true, false>)
                      : (compare ? hbm_read_ldg_kernel<kReadThreads, false, true> : hbm_read_ldg_kernel<kReadThreads, false, false>);
        k<<<clamp_grid((wide ? p.read_ldg256 : p.read_ldg).grid, bytes, kReadThreads * 128), kReadThreads, 0, st>>>(
            static_cast<const uint4*>(base), bytes >> 4, pr.imm, pr.pp, sc, out);
    }
    return cudaGetLastError();
}

cudaError_t launch_copy(const KernelPlan& p, unsigned variant, void* dst, const void* src, uint64_t bytes,
                        const Params& pr, const SweepScratch& sc, SweepOut* out, cudaStream_t st) {
    if (variant == COPY_TMA_FUSED) {
        if (!out) return cudaErrorInvalidValue;
        hbm_copy_fused_kernel<<<clamp_grid(p.copy_fused.grid, bytes, p.fused_tile), p.copy_fused.block, p.copy_fused.smem, st>>>(
            static_cast<unsigned char*>(dst), static_cast<const unsigned char*>(src), bytes, p.fused_tile,
            p.fused_stages, p.fused_chunk, sc.tile_ctr, pr.imm, pr.pp, sc, out);
    } else if (variant == COPY_TMA) {
        unsigned long long* ctr = nullptr;
        if (p.copy_dyn && sc.tile_ctr) {     // this kernel has no epilogue that could re-arm the counter
            ctr = sc.tile_ctr;
            cudaError_t e = cudaMemsetAsync(ctr, 0, sizeof(unsigned long long), st);
            if (e != cudaSuccess) return e;
        }
        hbm_copy_tma_kernel<<<clamp_grid(p.copy_tma.grid, bytes, p.copy_tile), p.copy_tma.block, p.copy_tma.smem, st>>>(
            static_cast<unsigned char*>(dst), static_cast<const unsigned char*>(src), bytes, p.copy_tile,
            p.copy_stages, p.copy_chunk, ctr, pr.imm, pr.pp, sc, out);
        if (ctr) {
            cudaError_t e = cudaMemsetAsync(ctr, 0, sizeof(unsigned long long), st);   // leave it armed for the self-resetting kernels
            if (e != cudaSuccess) return e;
        }
    } else {
        hbm_copy_ldg_kernel<kCopyThreads, kCopyUnroll><<<clamp_grid(p.copy_ldg.grid, bytes, kCopyThreads * kCopyUnroll * 16), p.copy_ldg.block, 0, st>>>(
            static_cast<uint4*>(dst), static_cast<const uint4*>(src), bytes >> 4, pr.imm, pr.pp, sc, out);
    }
    return cudaGetLastError();
}

cudaError_t launch_expected(const KernelPlan& p, uint64_t bytes, const Params& pr,
                            const SweepScratch& sc, SweepOut* out, cudaStream_t st) {
    hbm_expected_kernel<<<p.expect.grid, p.expect.block, 0, st>>>(bytes >> 3, pr.imm, pr.pp, sc, out);
    return cudaGetLastError();
}

cudaError_t launch_xor_words(void* base, uint64_t first, uint64_t count, uint64_t mask, cudaStream_t st) {
    if (count == 0) return cudaSuccess;
    const uint64_t blocks = std::min<uint64_t>((count + 255) / 256, 1024);
    xor_words_kernel<<<(unsigned)blocks, 256, 0, st>>>(static_cast<unsigned long long*>(base), first, count, mask);
    return cudaGetLastError();
}

cudaError_t launch_chase(const ChaseArgs& a, unsigned long long* out, cudaStream_t st) {
    if (a.n == 0 || a.n > CRO_MAX_DEVICES) return cudaErrorInvalidValue;
    chase_kernel<<<1, 32 * a.n, 0, st>>>(a, out);
    return cudaGetLastError();
}

cudaError_t arm_chase_out(unsigned long long* out, cudaStream_t st) {
    static_assert(kChaseArmed == ~0ull, "the armed word is all 0xFF bytes");
    return cudaMemsetAsync(out, 0xFF, kChaseOutWords * sizeof(unsigned long long), st);
}

cudaError_t launch_finalize(const FinalizeArgs& a, cudaStream_t st) {
    probe_finalize_kernel<<<1, 128, 0, st>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_p2p_finalize(const P2PFinalizeArgs& a, cudaStream_t st) {
    p2p_finalize_kernel<<<1, 32, 0, st>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_compute(unsigned leg, const ComputeArgs& a, int grid, cudaStream_t st) {
    void (*k)(ComputeArgs) = leg == CRO_COMPUTE_LEG_S8     ? compute_probe_kernel<CRO_COMPUTE_LEG_S8>
                             : leg == CRO_COMPUTE_LEG_BF16 ? compute_probe_kernel<CRO_COMPUTE_LEG_BF16>
                             : leg == CRO_COMPUTE_LEG_E4M3 ? compute_probe_kernel<CRO_COMPUTE_LEG_E4M3>
                             : leg == CRO_COMPUTE_LEG_FFMA ? compute_probe_kernel<CRO_COMPUTE_LEG_FFMA>
                             : leg == CRO_COMPUTE_LEG_IMAD ? compute_probe_kernel<CRO_COMPUTE_LEG_IMAD>
                                                           : nullptr;
    if (!k || grid < 1) return cudaErrorInvalidValue;
    cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kComputeSmem);
    if (e != cudaSuccess) return e;
    k<<<grid, kComputeThreads, kComputeSmem, st>>>(a);
    return cudaGetLastError();
}

}  // namespace cro
