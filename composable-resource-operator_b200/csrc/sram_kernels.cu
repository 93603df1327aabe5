// sram_kernels.cu — the SRAM probe's kernels (cro_probe_sram): March C- over every SM's shared memory, and the same
// words written and read across the SM-to-SM network of a thread-block cluster (distributed shared memory).
//
//   sram_smem    one CTA per SM: M0 .. M5 (include/croprobe.h) over the CTA's n_words, every read compared with the
//                word generated in registers, M5's reads folded
//   sram_dsmem   clusters of C CTAs: D0 local write, D1 every peer read over the network, D2 write into the next peer
//                over the network, D3 local read back
//
// Thread t of kSramThreads owns words t, t + T, t + 2T, ...: a warp's 32 lanes touch 32 consecutive 64-bit words, so
// its shared-memory accesses are conflict-free.  The march's order holds per word and per thread; between words of
// different threads only the barriers between elements order it.
#include "kernels.cuh"
#include "warp_claim.cuh"

#include <algorithm>

namespace cro {

namespace {

__device__ __forceinline__ unsigned long long timer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

// Every shared-memory access of the march is one of these: volatile (local) or .relaxed.cluster (network) inline PTX,
// which the compiler can neither drop, merge nor forward from an earlier store.
__device__ __forceinline__ unsigned long long ld_local(unsigned addr) {
    unsigned long long v;
    asm volatile("ld.volatile.shared.u64 %0, [%1];" : "=l"(v) : "r"(addr) : "memory");
    return v;
}
__device__ __forceinline__ void st_local(unsigned addr, unsigned long long v) {
    asm volatile("st.volatile.shared.u64 [%0], %1;" ::"r"(addr), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_remote(unsigned addr) {
    unsigned long long v;
    asm volatile("ld.relaxed.cluster.shared::cluster.u64 %0, [%1];" : "=l"(v) : "r"(addr) : "memory");
    return v;
}
__device__ __forceinline__ void st_remote(unsigned addr, unsigned long long v) {
    asm volatile("st.relaxed.cluster.shared::cluster.u64 [%0], %1;" ::"r"(addr), "l"(v) : "memory");
}
// The address of the same shared-memory offset in the CTA of cluster rank `rank`.
__device__ __forceinline__ unsigned map_rank(unsigned addr, unsigned rank) {
    unsigned r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank));
    return r;
}
__device__ __forceinline__ void cluster_barrier() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}

struct SramShared {
    unsigned long long count[CRO_SRAM_ELEMENTS];
    unsigned long long last;
    unsigned long long fx, fs, fw;
};

// The CTA's view of one launch: who it is and whether the test injection applies to it.
struct Cta {
    unsigned smid, nsmid, rank, base;           // base: shared address of word 0 of the CTA's own words
    bool inj;
};

__device__ __forceinline__ Cta cta_of(const SramArgs& a, unsigned rank, unsigned base) {
    Cta c;
    asm volatile("mov.u32 %0, %%smid;" : "=r"(c.smid));
    asm volatile("mov.u32 %0, %%nsmid;" : "=r"(c.nsmid));
    c.rank = rank;
    c.base = base;
    c.inj = a.inj_mask && (a.inj_sm < 0 || (unsigned)a.inj_sm == c.smid);
    return c;
}

// The test injection into word w of element el in iteration it (nothing unless the host armed it for this CTA).
__device__ __forceinline__ unsigned long long injected(const SramArgs& a, const Cta& c, unsigned long long v, unsigned w,
                                                       unsigned el, unsigned it) {
    if (c.inj && el == a.inj_element && it == a.inj_iter && (a.inj_word < 0 || (unsigned)a.inj_word == w)) v ^= a.inj_mask;
    return v;
}

// One compare of word w: v as read (injected) against e.  Counts and records a mismatch; the whole warp calls it.
__device__ __forceinline__ unsigned check(const SramArgs& a, const Cta& c, unsigned long long v, unsigned long long e,
                                          unsigned w, unsigned el, unsigned it, unsigned peer_block) {
    const bool bad = v != e;
    if (__ballot_sync(0xffffffffu, bad)) {
        const unsigned long long slot = warp_claim(bad ? 1u : 0u, a.claims, CRO_SRAM_RECORDS, [](unsigned) {});
        if (bad && slot < CRO_SRAM_RECORDS) a.rec[slot] = SramRecord{el, it, c.smid, peer_block, a.round, w, e, v};
    }
    return bad ? 1u : 0u;
}

// f(w) for the thread's words, ascending or descending.  n_words is a multiple of 32 and at least kSramThreads, so
// every lane of a warp runs the same trips.  Not unrolled: each element is one load and / or one store in the SASS,
// which tests/test_sram_abi.py counts.
template <bool DESC, class F>
__device__ __forceinline__ void each_word(unsigned n_words, F f) {
    if (!DESC) {
#pragma unroll 1
        for (unsigned w = threadIdx.x; w < n_words; w += kSramThreads) f(w);
    } else {
#pragma unroll 1
        for (int w = (int)(threadIdx.x + (n_words - 1 - threadIdx.x) / kSramThreads * kSramThreads); w >= 0; w -= kSramThreads)
            f((unsigned)w);
    }
}

// M1 .. M4: read the word against pattern ^ inv, then write its complement.
template <bool DESC>
__device__ __forceinline__ unsigned march_rw(const SramArgs& a, const Cta& c, unsigned el, unsigned long long inv, unsigned it) {
    unsigned n = 0;
    each_word<DESC>(a.n_words, [&](unsigned w) {
        const unsigned long long e = pattern_word(a.seed, w) ^ inv;
        const unsigned long long v = injected(a, c, ld_local(c.base + 8u * w), w, el, it);
        n += check(a, c, v, e, w, el, it, 0);
        st_local(c.base + 8u * w, ~e);
    });
    __syncthreads();
    return n;
}

// Adds the thread's per-element counts of one iteration to the CTA's; the iteration's total when it is the last.
__device__ __forceinline__ void add_counts(SramShared& s, const unsigned (&n)[CRO_SRAM_ELEMENTS], bool last) {
    unsigned sum = 0;
#pragma unroll
    for (int e = 0; e < CRO_SRAM_ELEMENTS; ++e) {
        const unsigned t = __reduce_add_sync(0xffffffffu, n[e]);
        if ((threadIdx.x & 31u) == 0 && t) atomicAdd(&s.count[e], (unsigned long long)t);
        sum += t;
    }
    if (last && (threadIdx.x & 31u) == 0 && sum) atomicAdd(&s.last, (unsigned long long)sum);
}

__device__ __forceinline__ void publish(const SramArgs& a, const Cta& c, SramShared& s, unsigned long long fx,
                                        unsigned long long fs, unsigned long long fw, unsigned long long t0,
                                        unsigned long long t1, long long k0, long long k1) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        fx ^= __shfl_xor_sync(0xffffffffu, fx, o);
        fs += __shfl_xor_sync(0xffffffffu, fs, o);
        fw += __shfl_xor_sync(0xffffffffu, fw, o);
    }
    if ((threadIdx.x & 31u) == 0) {
        atomicXor(&s.fx, fx);
        atomicAdd(&s.fs, fs);
        atomicAdd(&s.fw, fw);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        SramCta& o = a.cta[blockIdx.x];
        o.t0 = t0;
        o.t1 = t1;
        o.cycles = (unsigned long long)(k1 - k0);
        for (int e = 0; e < CRO_SRAM_ELEMENTS; ++e) o.count[e] = s.count[e];
        o.last = s.last;
        o.fold_x = s.fx;
        o.fold_s = s.fs;
        o.fold_w = s.fw;
        o.smid = c.smid;
        o.nsmid = c.nsmid;
        o.rank = c.rank;
        o.block = blockIdx.x;
        __threadfence();
        o.stamp = a.stamp;
    }
}

__device__ __forceinline__ void clear_shared(SramShared& s) {
    if (threadIdx.x < sizeof(SramShared) / 8) reinterpret_cast<unsigned long long*>(&s)[threadIdx.x] = 0;
    __syncthreads();
}

__global__ void __launch_bounds__(kSramThreads, 1) sram_smem_kernel(const SramArgs a) {
    extern __shared__ __align__(16) unsigned long long sram_words[];
    __shared__ SramShared s;
    clear_shared(s);
    const Cta c = cta_of(a, 0, (unsigned)__cvta_generic_to_shared(sram_words));
    unsigned long long fx = 0, fs = 0, fw = 0;
    const unsigned long long t0 = timer_ns();
    const long long k0 = clock64();
    for (unsigned it = 0; it < a.iterations; ++it) {
        unsigned n[CRO_SRAM_ELEMENTS] = {0, 0, 0, 0, 0, 0};
        each_word<false>(a.n_words, [&](unsigned w) { st_local(c.base + 8u * w, pattern_word(a.seed, w)); });   // M0
        __syncthreads();
        n[1] = march_rw<false>(a, c, 1, 0ull, it);
        n[2] = march_rw<false>(a, c, 2, ~0ull, it);
        n[3] = march_rw<true>(a, c, 3, 0ull, it);
        n[4] = march_rw<true>(a, c, 4, ~0ull, it);
        each_word<false>(a.n_words, [&](unsigned w) {                                                                 // M5
            const unsigned long long e = pattern_word(a.seed, w);
            const unsigned long long v = injected(a, c, ld_local(c.base + 8u * w), w, 5, it);
            n[5] += check(a, c, v, e, w, 5, it, 0);
            fx ^= v;
            fs += v;
            fw += v * (2ull * w + 1);
        });
        __syncthreads();
        add_counts(s, n, it + 1 == a.iterations);
    }
    const long long k1 = clock64();
    const unsigned long long t1 = timer_ns();
    publish(a, c, s, fx, fs, fw, t0, t1, k0, k1);
}

__global__ void __launch_bounds__(kSramThreads, 1) sram_dsmem_kernel(const SramArgs a) {
    extern __shared__ __align__(16) unsigned long long sram_words[];
    __shared__ SramShared s;
    clear_shared(s);
    unsigned rank, size;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(rank));
    asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(size));
    const Cta c = cta_of(a, rank, (unsigned)__cvta_generic_to_shared(sram_words));
    const unsigned block0 = blockIdx.x - rank, next = (rank + 1) % size, prev = (rank + size - 1) % size;
    const unsigned long long seed = a.seed + rank * kNonceStride, next_seed = a.seed + next * kNonceStride;
    const unsigned next_base = map_rank(c.base, next);
    const unsigned long long t0 = timer_ns();
    const long long k0 = clock64();
    for (unsigned it = 0; it < a.iterations; ++it) {
        unsigned n[CRO_SRAM_ELEMENTS] = {0, 0, 0, 0, 0, 0};
        each_word<false>(a.n_words, [&](unsigned w) { st_local(c.base + 8u * w, pattern_word(seed, w)); });     // D0
        cluster_barrier();
        for (unsigned q = 1; q < size; ++q) {                                                                    // D1
            const unsigned peer = (rank + q) % size, peer_base = map_rank(c.base, peer);
            const unsigned long long peer_seed = a.seed + peer * kNonceStride;
            each_word<false>(a.n_words, [&](unsigned w) {
                const unsigned long long e = pattern_word(peer_seed, w);
                const unsigned long long v = injected(a, c, ld_remote(peer_base + 8u * w), w, 1, it);
                n[1] += check(a, c, v, e, w, 1, it, block0 + peer);
            });
        }
        cluster_barrier();
        each_word<false>(a.n_words, [&](unsigned w) {                                                            // D2
            st_remote(next_base + 8u * w, injected(a, c, ~pattern_word(next_seed, w), w, 2, it));
        });
        cluster_barrier();
        each_word<false>(a.n_words, [&](unsigned w) {                                                            // D3
            const unsigned long long e = ~pattern_word(seed, w);
            n[3] += check(a, c, ld_local(c.base + 8u * w), e, w, 3, it, block0 + prev);
        });
        // No barrier before the next D0: it writes only the CTA's own words, which no peer touches until the
        // barrier after it.  After the last D3 no peer touches them at all, so the CTA may exit.
        __syncthreads();
        add_counts(s, n, it + 1 == a.iterations);
    }
    const long long k1 = clock64();
    const unsigned long long t1 = timer_ns();
    publish(a, c, s, 0, 0, 0, t0, t1, k0, k1);
}

cudaLaunchConfig_t cluster_config(int grid, unsigned cluster, unsigned n_words, cudaStream_t st,
                                  cudaLaunchAttribute* attr) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)grid);
    cfg.blockDim = dim3(kSramThreads);
    cfg.dynamicSmemBytes = (size_t)n_words * 8;
    cfg.stream = st;
    attr->id = cudaLaunchAttributeClusterDimension;
    attr->val.clusterDim.x = cluster;
    attr->val.clusterDim.y = 1;
    attr->val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cfg;
}

}  // namespace

cudaError_t sram_plan(int device, unsigned* n_words) {
    int optin = 0;
    cudaError_t e = cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device);
    if (e) return e;
    cudaFuncAttributes fa[2];
    if ((e = cudaFuncGetAttributes(&fa[0], sram_smem_kernel)) || (e = cudaFuncGetAttributes(&fa[1], sram_dsmem_kernel))) return e;
    const size_t fixed = std::max(fa[0].sharedSizeBytes, fa[1].sharedSizeBytes);
    if ((size_t)optin < fixed + 8 * kSramThreads) return cudaErrorInvalidConfiguration;
    const size_t dyn = ((size_t)optin - fixed) & ~(size_t)255;
    for (const void* k : {(const void*)sram_smem_kernel, (const void*)sram_dsmem_kernel}) {
        if ((e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dyn)) ||
            (e = cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared)))
            return e;
    }
    *n_words = (unsigned)(dyn / 8);
    return cudaSuccess;
}

cudaError_t launch_sram_smem(const SramArgs& a, int grid, cudaStream_t st) {
    sram_smem_kernel<<<grid, kSramThreads, (size_t)a.n_words * 8, st>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_sram_dsmem(const SramArgs& a, int grid, unsigned cluster, cudaStream_t st) {
    cudaLaunchAttribute attr;
    const cudaLaunchConfig_t cfg = cluster_config(grid, cluster, a.n_words, st, &attr);
    return cudaLaunchKernelEx(&cfg, sram_dsmem_kernel, a);
}

cudaError_t sram_max_clusters(unsigned cluster, unsigned n_words, int* clusters) {
    cudaLaunchAttribute attr;
    const cudaLaunchConfig_t cfg = cluster_config((int)cluster, cluster, n_words, nullptr, &attr);
    return cudaOccupancyMaxActiveClusters(clusters, sram_dsmem_kernel, &cfg);
}

}  // namespace cro
