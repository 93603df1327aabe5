// l2_kernels.cu — the L2 probe's kernels (cro_probe_l2): March C- over an L2-resident buffer whose blocks change hands
// between SMs from element to element, and the L2 atomic units checked against answers computed without atomics.
//
//   l2_march      one element of one iteration; one CTA per SM, CTA j handling the blocks b with
//                 (b + element * delta) mod G == j, thread t the 16-byte vector t of each (descending elements: the
//                 blocks and the vectors in reverse)
//   l2_a1         red.add.u64 / red.xor.b64 of every CTA's pattern words into the A1 counters
//   l2_a1_check   one thread per A1 counter: its sum and xor over every CTA, recomputed
//   l2_a2         one warp of every CTA per A2 counter takes atom.add.u32 tickets and stores them
//   l2_a2_check   one warp per A2 counter: marks each ticket present and counts the holes
//   l2_release    after the call: every line of the buffer discarded from the L2, so none keeps its evict-last mark
//
// Nothing here waits on another CTA or loops on a value read from memory: a broken L2 or atomic unit gives a wrong
// answer, never a hang.
#include "l2_kernels.cuh"
#include "warp_claim.cuh"

namespace cro {

namespace {

__device__ __forceinline__ unsigned long long timer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

// Every access of the march is one of these: 128-bit .relaxed.gpu inline PTX, which bypasses L1 and which the compiler
// can neither drop, merge nor forward from an earlier store, with an L2::evict_last policy so that the buffer stays in
// the L2 while it fits (without touching the persisting set-aside, which every tenant of the GPU shares).
__device__ __forceinline__ unsigned long long evict_last_policy() {
    unsigned long long p;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ ulonglong2 ld_l2(const ulonglong2* p, unsigned long long pol) {
    ulonglong2 v;
    asm volatile("ld.relaxed.gpu.global.L2::cache_hint.v2.u64 {%0, %1}, [%2], %3;" : "=l"(v.x), "=l"(v.y) : "l"(p), "l"(pol) : "memory");
    return v;
}
__device__ __forceinline__ void st_l2(ulonglong2* p, unsigned long long x, unsigned long long y, unsigned long long pol) {
    asm volatile("st.relaxed.gpu.global.L2::cache_hint.v2.u64 [%0], {%1, %2}, %3;" ::"l"(p), "l"(x), "l"(y), "l"(pol) : "memory");
}

struct L2Shared {
    unsigned long long count, fx, fs, fw;
};

// The CTA's view of one launch.
struct Launch {
    unsigned el, it, smid, writer;
    bool inj;
};

// One compare of the vector holding words w and w + 1: v as read (injected) against e.  Counts and records the
// mismatches; the whole warp calls it.
__device__ __forceinline__ unsigned check(const L2Args& a, const Launch& L, ulonglong2 v, unsigned long long e0,
                                          unsigned long long e1, unsigned long long w) {
    const bool b0 = v.x != e0, b1 = v.y != e1;
    const unsigned n = (b0 ? 1u : 0u) + (b1 ? 1u : 0u);
    if (__ballot_sync(0xffffffffu, n)) {
        unsigned long long slot = warp_claim(n, a.claims, CRO_L2_RECORDS, [](unsigned) {});
        if (b0) {
            if (slot < CRO_L2_RECORDS) a.rec[slot] = cro_l2_fault{L.el, L.it, L.smid, blockIdx.x, L.writer, 0u, w, e0, v.x, 0u, 0u};
            ++slot;
        }
        if (b1 && slot < CRO_L2_RECORDS) a.rec[slot] = cro_l2_fault{L.el, L.it, L.smid, blockIdx.x, L.writer, 0u, w + 1, e1, v.y, 0u, 0u};
    }
    return n;
}

constexpr unsigned kL2Batch = 4;       // blocks a thread has in flight: four loads issued before the first compare

__global__ void __launch_bounds__(kL2Threads, 1) l2_march_kernel(const L2Args a, unsigned el, unsigned it) {
    __shared__ L2Shared s;
    if (threadIdx.x < sizeof(L2Shared) / 8) reinterpret_cast<unsigned long long*>(&s)[threadIdx.x] = 0;
    __syncthreads();
    const unsigned long long t0 = timer_ns();
    Launch L;
    unsigned nsmid;
    asm volatile("mov.u32 %0, %%smid;" : "=r"(L.smid));
    asm volatile("mov.u32 %0, %%nsmid;" : "=r"(nsmid));
    const unsigned G = a.G, j = blockIdx.x;
    L.el = el;
    L.it = it;
    L.writer = (j + G - a.delta % G) % G;                   // the owner of this CTA's blocks in the element before
    L.inj = a.inj_mask && el != 0 && it == a.inj_iter && (a.inj_sm < 0 || (unsigned)a.inj_sm == L.smid) &&
            (a.inj_element < 0 || (unsigned)a.inj_element == el);
    const unsigned b0 = (j + G - (unsigned)((unsigned long long)el * a.delta % G)) % G;
    const unsigned nb = b0 < a.blocks ? (a.blocks - 1 - b0) / G + 1 : 0;      // blocks b0, b0 + G, ...
    const bool desc = el == 3 || el == 4, reads = el != 0, writes = el != 5;
    const unsigned long long inv = (el == 2 || el == 4) ? ~0ull : 0ull;       // M2, M4 read Q; M1, M3, M5 read P
    const unsigned vec = desc ? kL2Threads - 1 - threadIdx.x : threadIdx.x;
    const unsigned long long pol = evict_last_policy();
    unsigned long long n = 0, fx = 0, fs = 0, fw = 0;
#pragma unroll 1
    for (unsigned q0 = 0; q0 < nb; q0 += kL2Batch) {
        unsigned long long w[kL2Batch];
        ulonglong2 v[kL2Batch];
#pragma unroll
        for (unsigned u = 0; u < kL2Batch; ++u) {
            const unsigned q = desc ? nb - 1 - (q0 + u) : q0 + u;
            w[u] = (unsigned long long)(b0 + q * G) * kL2BlockWords + 2ull * vec;
            v[u] = make_ulonglong2(0, 0);
            if (reads && q0 + u < nb) v[u] = ld_l2(a.buf + w[u] / 2, pol);
        }
#pragma unroll
        for (unsigned u = 0; u < kL2Batch; ++u) {
            if (q0 + u >= nb) break;                        // uniform over the CTA
            const unsigned long long e0 = pattern_word(a.seed, w[u]) ^ inv, e1 = pattern_word(a.seed, w[u] + 1) ^ inv;
            if (reads) {
                if (L.inj && (a.inj_word < 0 || (unsigned long long)a.inj_word == w[u])) v[u].x ^= a.inj_mask;
                if (L.inj && (a.inj_word < 0 || (unsigned long long)a.inj_word == w[u] + 1)) v[u].y ^= a.inj_mask;
                n += check(a, L, v[u], e0, e1, w[u]);
            }
            if (el == 5) {
                fx ^= v[u].x ^ v[u].y;
                fs += v[u].x + v[u].y;
                fw += v[u].x * (2 * w[u] + 1) + v[u].y * (2 * w[u] + 3);
            }
            // M0 writes P; M1 .. M4 write the complement of what they read
            if (writes) st_l2(a.buf + w[u] / 2, reads ? ~e0 : e0, reads ? ~e1 : e1, pol);
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        n += __shfl_xor_sync(0xffffffffu, n, o);
        fx ^= __shfl_xor_sync(0xffffffffu, fx, o);
        fs += __shfl_xor_sync(0xffffffffu, fs, o);
        fw += __shfl_xor_sync(0xffffffffu, fw, o);
    }
    if ((threadIdx.x & 31u) == 0) {
        if (n) atomicAdd(&s.count, n);
        atomicXor(&s.fx, fx);
        atomicAdd(&s.fs, fs);
        atomicAdd(&s.fw, fw);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        L2Cta& o = a.cta[((size_t)it * CRO_L2_ELEMENTS + el) * G + j];
        o.t0 = t0;
        o.t1 = timer_ns();
        o.count = s.count;
        o.fx = s.fx;
        o.fs = s.fs;
        o.fw = s.fw;
        o.smid = L.smid;
        o.nsmid = nsmid;
        __threadfence();
        o.stamp = a.stamp;
    }
}

__device__ __forceinline__ void red_add(unsigned long long* p, unsigned long long v) {
    asm volatile("red.relaxed.gpu.global.add.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ void red_xor(unsigned long long* p, unsigned long long v) {
    asm volatile("red.relaxed.gpu.global.xor.b64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned atom_add(unsigned* p, unsigned v) {
    unsigned r;
    asm volatile("atom.relaxed.gpu.global.add.u32 %0, [%1], %2;" : "=r"(r) : "l"(p), "r"(v) : "memory");
    return r;
}

__global__ void __launch_bounds__(kL2Threads) l2_a1_kernel(const L2AtomicArgs a) {
    const unsigned j = blockIdx.x;
    for (unsigned i = threadIdx.x; i < a.a1; i += kL2Threads) {
        unsigned long long v = pattern_word(a.seed, (unsigned long long)j * a.a1 + i);
        if (a.inj_leg == CRO_L2_A1 && j == 0 && i == a.inj_counter) v ^= a.inj_mask;
        red_add(a.a1_sum + i, v);
        red_xor(a.a1_xor + i, v);
    }
}

__global__ void __launch_bounds__(kL2Threads) l2_a1_check_kernel(const L2AtomicArgs a) {
    const unsigned i = blockIdx.x * kL2Threads + threadIdx.x;
    bool bad = false;
    if (i < a.a1) {
        unsigned long long s = 0, x = 0;
        for (unsigned j = 0; j < a.G; ++j) {
            const unsigned long long v = pattern_word(a.seed, (unsigned long long)j * a.a1 + i);
            s += v;
            x ^= v;
        }
        bad = __ldcg(a.a1_sum + i) != s || __ldcg(a.a1_xor + i) != x;
        a.a1_bad[i] = bad ? 1 : 0;
    }
    const int n = __syncthreads_count(bad);
    if (threadIdx.x == 0) a.a1_partial[blockIdx.x] = (unsigned long long)n;
}

__global__ void __launch_bounds__(kL2Threads) l2_a2_kernel(const L2AtomicArgs a) {
    const unsigned lane = threadIdx.x & 31u, warp = threadIdx.x >> 5, j = blockIdx.x, per = 32 * a.G;
    for (unsigned t = warp; t < a.a2; t += kL2Threads / 32) {
        unsigned got = atom_add(a.a2_ctr + 32ull * t, 1u);
        if (a.inj_leg == CRO_L2_A2 && j == 0 && lane == 0 && t == a.inj_counter) got ^= (unsigned)a.inj_mask;
        a.tickets[(size_t)t * per + 32 * j + lane] = got;
    }
}

__global__ void __launch_bounds__(kL2Threads) l2_a2_check_kernel(const L2AtomicArgs a) {
    __shared__ unsigned long long holes_of[kL2Threads / 32], bad_of[kL2Threads / 32];
    const unsigned lane = threadIdx.x & 31u, warp = threadIdx.x >> 5, t = blockIdx.x * (kL2Threads / 32) + warp, per = 32 * a.G;
    unsigned holes = 0;
    bool bad = false;
    if (t < a.a2) {
        const unsigned* tk = a.tickets + (size_t)t * per;
        unsigned char* pr = a.present + (size_t)t * per;
        for (unsigned k = lane; k < per; k += 32) {
            const unsigned v = __ldcg(tk + k);
            if (v < per) pr[v] = 1;                         // a ticket out of range marks nothing: a hole stays
        }
        __syncwarp();
        for (unsigned k = lane; k < per; k += 32) holes += *reinterpret_cast<volatile unsigned char*>(pr + k) ? 0u : 1u;
        holes = __reduce_add_sync(0xffffffffu, holes);
        bad = holes || __ldcg(a.a2_ctr + 32ull * t) != per;
        if (lane == 0) a.a2_bad[t] = bad ? 1 : 0;
    }
    if (lane == 0) {
        holes_of[warp] = holes;
        bad_of[warp] = bad ? 1 : 0;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long h = 0, b = 0;
        for (int k = 0; k < kL2Threads / 32; ++k) {
            h += holes_of[k];
            b += bad_of[k];
        }
        a.a2_partial[2 * blockIdx.x] = h;
        a.a2_partial[2 * blockIdx.x + 1] = b;
    }
}

// The march leaves its whole buffer in the L2 marked evict-last, and nothing would demote those lines after the call:
// on a GPU other tenants share they would keep their priority over other data until the driver reuses the memory.
// The buffer is dead once the march is checked, so each 128-byte line is discarded (invalidated without a write-back).
__global__ void __launch_bounds__(256) l2_release_kernel(const char* buf, unsigned long long lines) {
    for (unsigned long long i = blockIdx.x * 256ull + threadIdx.x; i < lines; i += (unsigned long long)gridDim.x * 256)
        asm volatile("discard.global.L2 [%0], 128;" ::"l"(buf + 128 * i) : "memory");
}

}  // namespace

cudaError_t launch_l2_release(const void* buf, unsigned long long bytes, int grid, cudaStream_t st) {
    l2_release_kernel<<<grid, 256, 0, st>>>(static_cast<const char*>(buf), bytes / 128);
    return cudaGetLastError();
}

cudaError_t l2_plan(int device, size_t* dyn) {
    int optin = 0;
    cudaError_t e = cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device);
    if (e) return e;
    cudaFuncAttributes fa;
    if ((e = cudaFuncGetAttributes(&fa, l2_march_kernel))) return e;
    // the most a CTA may ask for: more than half of any SM's shared memory, so no two CTAs of a launch share an SM
    *dyn = ((size_t)optin - fa.sharedSizeBytes) & ~(size_t)1023;
    return cudaFuncSetAttribute(l2_march_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)*dyn);
}

cudaError_t launch_l2_march(const L2Args& a, unsigned el, unsigned it, size_t dyn, cudaStream_t st) {
    l2_march_kernel<<<a.G, kL2Threads, dyn, st>>>(a, el, it);
    return cudaGetLastError();
}

cudaError_t launch_l2_a1(const L2AtomicArgs& a, cudaStream_t st) {
    l2_a1_kernel<<<a.G, kL2Threads, 0, st>>>(a);
    return cudaGetLastError();
}
cudaError_t launch_l2_a1_check(const L2AtomicArgs& a, cudaStream_t st) {
    l2_a1_check_kernel<<<l2_a1_check_ctas(a.a1), kL2Threads, 0, st>>>(a);
    return cudaGetLastError();
}
cudaError_t launch_l2_a2(const L2AtomicArgs& a, cudaStream_t st) {
    l2_a2_kernel<<<a.G, kL2Threads, 0, st>>>(a);
    return cudaGetLastError();
}
cudaError_t launch_l2_a2_check(const L2AtomicArgs& a, cudaStream_t st) {
    l2_a2_check_kernel<<<l2_a2_check_ctas(a.a2), kL2Threads, 0, st>>>(a);
    return cudaGetLastError();
}

}  // namespace cro
