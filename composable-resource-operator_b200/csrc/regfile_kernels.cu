// regfile_kernels.cu — the register-file probe's kernel (cro_probe_regfile): every thread of one CTA per SM holds
// CRO_REGFILE_SLOTS words of a known pattern in as many registers across two barriers, and compares every one.
//
// One element of an iteration, every step a whole-CTA phase:
//   1 generate   each thread writes its own K source words (the pattern, complemented in E1, test injection last)
//   2 barrier
//   3 load       K words into K registers: fully unrolled ld.volatile.shared.v4, constant indices only
//   4 barrier
//   5 overwrite  every source word set to 0; thread 0 publishes the element's key (seed, complement, fold mask)
//   6 barrier
//   7 compare    the key read back from shared memory, every slot compared with the pattern recomputed from it
//
// Why the value compared is the value held: the loads are volatile, so neither the compiler nor ptxas may issue them
// again, and after step 5 a reload would read 0.  The expected words derive from the key, which is read only after the
// barrier of step 6, so no compare, and nothing else that could stand in for a held register, can move above it.
// tests/test_regfile_abi.py checks this on the SASS.  The element body is one non-unrolled loop body, so slot k is the
// same physical register in every element and iteration.
//
// Source layout: word k of thread t is 32-bit word (k / 4 * T + t) * 4 + k % 4 of the CTA's dynamic shared memory, so
// one warp's 16-byte loads of one slot group cover 512 consecutive bytes (conflict-free).
#include "kernels.cuh"
#include "warp_claim.cuh"

namespace cro {

namespace {

constexpr unsigned kK = CRO_REGFILE_SLOTS;
constexpr unsigned kT = CRO_REGFILE_THREADS;
constexpr unsigned kGroups = kK / 4;
static_assert(kK % 4 == 0 && kT % 32 == 0, "whole 16-byte slot groups, whole warps");

__device__ __forceinline__ unsigned long long timer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

__device__ __forceinline__ void st4(unsigned addr, unsigned x, unsigned y, unsigned z, unsigned w) {
    asm volatile("st.volatile.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(x), "r"(y), "r"(z), "r"(w) : "memory");
}
__device__ __forceinline__ void ld4(unsigned addr, unsigned& x, unsigned& y, unsigned& z, unsigned& w) {
    asm volatile("ld.volatile.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(x), "=r"(y), "=r"(z), "=r"(w) : "r"(addr) : "memory");
}
__device__ __forceinline__ void st1(unsigned addr, unsigned v) {
    asm volatile("st.volatile.shared.u32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned ld1(unsigned addr) {
    unsigned v;
    asm volatile("ld.volatile.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
    return v;
}
__device__ __forceinline__ void st64(unsigned addr, unsigned long long v) {
    asm volatile("st.volatile.shared.u64 [%0], %1;" ::"r"(addr), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld64(unsigned addr) {
    unsigned long long v;
    asm volatile("ld.volatile.shared.u64 %0, [%1];" : "=l"(v) : "r"(addr) : "memory");
    return v;
}

// P(t, k) of an element's seed (include/croprobe.h), before the complement.
__device__ __forceinline__ unsigned pattern32(unsigned long long seed, unsigned t, unsigned k) {
    return (unsigned)pattern_word(seed, (unsigned long long)t * kK + k);
}

// The element's key, written by thread 0 in step 5 and read by every thread after the barrier of step 6.
struct Key {
    unsigned long long seed;
    unsigned inv;                               // 0 in E0, all ones in E1
    unsigned fold;                              // all ones in the last iteration's E1: its held words are folded
};
struct RegfileShared {
    Key key;
    unsigned long long count[CRO_REGFILE_ELEMENTS];
    unsigned long long last;
    unsigned long long fx, fs, fw;
};

__global__ void __launch_bounds__(kT, 1) regfile_kernel(const RegfileArgs a) {
    extern __shared__ __align__(16) unsigned regfile_src[];
    __shared__ RegfileShared s;
    if (threadIdx.x < sizeof(RegfileShared) / 8) reinterpret_cast<unsigned long long*>(&s)[threadIdx.x] = 0;
    __syncthreads();
    unsigned smid, nsmid;
    asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
    asm volatile("mov.u32 %0, %%nsmid;" : "=r"(nsmid));
    const unsigned t = threadIdx.x, warp = t >> 5, lane = t & 31u;
    const bool inj = a.inj_mask && (a.inj_sm < 0 || (unsigned)a.inj_sm == smid) && (a.inj_warp < 0 || (unsigned)a.inj_warp == warp) &&
                     (a.inj_lane < 0 || (unsigned)a.inj_lane == lane);
    const unsigned src = (unsigned)__cvta_generic_to_shared(regfile_src) + 16u * t;   // + 16 * kT * g: slot group g
    const unsigned key = (unsigned)__cvta_generic_to_shared(&s.key);
    unsigned long long c0 = 0, c1 = 0, last = 0, fx = 0, fs = 0, fw = 0;
    const unsigned long long t0 = timer_ns();
    const long long k0 = clock64();
#pragma unroll 1
    for (unsigned step = 0; step < 2 * a.iterations; ++step) {
        const unsigned it = step >> 1, el = step & 1u;
        const unsigned long long seed = a.seed + it * kNonceStride;
        const unsigned inv = el ? ~0u : 0u;
        const unsigned mask = inj && el == a.inj_element && it == a.inj_iter ? a.inj_mask : 0u;

        // 1 generate
#pragma unroll 1
        for (unsigned g = 0; g < kGroups; ++g) {
            unsigned w[4];
#pragma unroll
            for (unsigned j = 0; j < 4; ++j) {
                const unsigned k = 4 * g + j;
                w[j] = pattern32(seed, t, k) ^ inv ^ (a.inj_slot < 0 || (unsigned)a.inj_slot == k ? mask : 0u);
            }
            st4(src + 16u * kT * g, w[0], w[1], w[2], w[3]);
        }
        __syncthreads();                                                    // 2

        // 3 load: K registers
        unsigned r[kK];
#pragma unroll
        for (unsigned g = 0; g < kGroups; ++g) ld4(src + 16u * kT * g, r[4 * g], r[4 * g + 1], r[4 * g + 2], r[4 * g + 3]);
        __syncthreads();                                                    // 4

        // 5 overwrite, and the key
#pragma unroll 1
        for (unsigned g = 0; g < kGroups; ++g) st4(src + 16u * kT * g, 0u, 0u, 0u, 0u);
        if (t == 0) {
            st64(key, seed);
            st1(key + 8, inv);
            st1(key + 12, el && it + 1 == a.iterations ? ~0u : 0u);
        }
        __syncthreads();                                                    // 6

        // 7 compare: a mismatching slot leaves its difference in its (zeroed) source word for the records below
        const unsigned long long kseed = ld64(key);
        const unsigned kinv = ld1(key + 8), kfold = ld1(key + 12);
        unsigned n = 0;
#pragma unroll
        for (unsigned k = 0; k < kK; ++k) {
            const unsigned d = r[k] ^ pattern32(kseed, t, k) ^ kinv;
            n += d != 0u;
            if (d) st1(src + 16u * kT * (k / 4) + 4u * (k % 4), d);
            const unsigned f = r[k] & kfold;
            fx ^= f;
            fs += f;
            fw += (unsigned long long)f * (2u * k + 1u);
        }
        if (__any_sync(0xffffffffu, n)) {
#pragma unroll 1
            for (unsigned k = 0; k < kK; ++k) {
                const unsigned d = ld1(src + 16u * kT * (k / 4) + 4u * (k % 4));
                const bool bad = d != 0u;
                if (__ballot_sync(0xffffffffu, bad)) {
                    const unsigned long long slot = warp_claim(bad ? 1u : 0u, a.claims, CRO_REGFILE_RECORDS, [](unsigned) {});
                    const unsigned e = pattern32(kseed, t, k) ^ kinv;
                    if (bad && slot < CRO_REGFILE_RECORDS) a.rec[slot] = cro_regfile_fault{el, it, smid, warp, lane, k, e, e ^ d};
                }
            }
        }
        c0 += el ? 0u : n;
        c1 += el ? n : 0u;
        last += it + 1 == a.iterations ? n : 0u;
    }
    const long long k1 = clock64();
    const unsigned long long t1 = timer_ns();

#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        c0 += __shfl_xor_sync(0xffffffffu, c0, o);
        c1 += __shfl_xor_sync(0xffffffffu, c1, o);
        last += __shfl_xor_sync(0xffffffffu, last, o);
        fx ^= __shfl_xor_sync(0xffffffffu, fx, o);
        fs += __shfl_xor_sync(0xffffffffu, fs, o);
        fw += __shfl_xor_sync(0xffffffffu, fw, o);
    }
    if (lane == 0) {
        atomicAdd(&s.count[0], c0);
        atomicAdd(&s.count[1], c1);
        atomicAdd(&s.last, last);
        atomicXor(&s.fx, fx);
        atomicAdd(&s.fs, fs);
        atomicAdd(&s.fw, fw);
    }
    __syncthreads();
    if (t == 0) {
        cro_regfile_cta& o = a.cta[blockIdx.x];
        o.t0 = t0;
        o.t1 = t1;
        o.cycles = (unsigned long long)(k1 - k0);
        o.count[0] = s.count[0];
        o.count[1] = s.count[1];
        o.last = s.last;
        o.fold_x = s.fx;
        o.fold_s = s.fs;
        o.fold_w = s.fw;
        o.smid = smid;
        o.nsmid = nsmid;
        o.block = blockIdx.x;
        o.reserved = 0;
        __threadfence();
        o.stamp = a.stamp;
    }
}

constexpr size_t kSrcBytes = 4ull * kK * kT;

}  // namespace

cudaError_t regfile_plan(int device, cudaFuncAttributes* fa) {
    int optin = 0;
    cudaError_t e = cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device);
    if (e || (e = cudaFuncGetAttributes(fa, regfile_kernel))) return e;
    if ((size_t)optin < fa->sharedSizeBytes + kSrcBytes) return cudaErrorInvalidConfiguration;
    if ((e = cudaFuncSetAttribute(regfile_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSrcBytes))) return e;
    return cudaFuncSetAttribute(regfile_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
}

cudaError_t launch_regfile(const RegfileArgs& a, int grid, cudaStream_t st) {
    regfile_kernel<<<grid, kT, kSrcBytes, st>>>(a);
    return cudaGetLastError();
}

}  // namespace cro
