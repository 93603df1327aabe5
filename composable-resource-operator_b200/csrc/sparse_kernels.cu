// sparse_kernels.cu — the sparse probe's kernels (cro_probe_sparse): every SM computes its leg's answer tile D = A * B
// `iterations` times with wgmma.mma_async.sp, A 2:4 sparse (TF32: 1:2), from a compressed A, B and metadata it
// generates itself, and checks every value against the exact answer (include/croprobe.h, "SM sparse").  One template
// per leg:
//   S8                 m64n256k64 .s32.s8.s8 (IGMMA.SP), selector 0
//   E4M3, E5M2         m64n256k64 .f32.e4m3 / .e5m2 (QGMMA.SP), selector 0
//   BF16, F16          m64n256k32 .f32.bf16 / .f16 (HGMMA.SP), selectors 0 and 1 on alternate K steps
//   TF32               m64n256k16 .f32.tf32 (HGMMA.SP), selectors 0 and 1 on alternate K steps
// Each of the two warpgroups owns 64 rows and chains eight instructions over K, scale-d = 0 on the first of every
// iteration.  The compressed A (M x K/2) and B^T (N x K) sit in the canonical K-major no-swizzle layout (kmajor_off,
// sm_tile.cuh): one instruction reads 32 bytes of K of A and 64 of B.
// Metadata: one 32-bit register per thread and instruction, eight nibbles, nibble = i | j << 2 for the kept pair (i, j)
// of a group.  Which nibble of which thread decodes which (row, group) was measured on an H100 and is pinned by the
// sparse probe's GPU tests: with r0 = 16 * (warp % 4) + lane / 4 and q = lane % 4, nibble n of instruction s
// covers
//   8-bit forms (16 groups per row and instruction):  row r0 + 8 * (q % 2), group 16 s + 8 * (q / 2) + n
//   16- and 32-bit forms (8 groups):                  row r0 + 8 * (n / 4), group 8 s + 4 * (q % 2) + n % 4
// where for the 16- and 32-bit forms the threads with q / 2 == selector supply the register.  The other pair of each
// quad holds a different legal register (every pair advanced by one), so a clean call passes only if the instruction
// reads the pair its selector names: the clean calls pin the selector mapping, the substitutions the nibble mapping.
// After each iteration every thread adds sum_j canon(value_j) * (2e_j + 1) to a running fold (e_j = row * N + col); at
// the end it compares the fold with iterations * the fold of the expected values, and the last answer element by
// element with the expected tile (global memory, L2-resident, shared by all CTAs), recording mismatches with the
// compute probe's idiom (warp_claim).
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_fp8.h>

#include <type_traits>

#include "sm_tile.cuh"
#include "sparse_kernels.cuh"
#include "warp_claim.cuh"

namespace cro {

namespace {

template <unsigned LEG> struct SLeg {
    static constexpr bool kInt = LEG == CRO_SPARSE_LEG_S8;
    static constexpr unsigned kElem = LEG <= CRO_SPARSE_LEG_E5M2 ? 1 : LEG == CRO_SPARSE_LEG_TF32 ? 4 : 2;
    static constexpr unsigned M = CRO_SPARSE_M, N = CRO_SPARSE_N;
    static constexpr unsigned K = kElem == 1 ? CRO_SPARSE_K : kElem == 2 ? CRO_SPARSE_K16 : CRO_SPARSE_TF32_K;   // logical
    static constexpr unsigned KC = K / 2;                       // compressed A's elements per row
    static constexpr unsigned G = kElem == 4 ? 2 : 4;           // K positions per group (one metadata nibble)
    static constexpr unsigned P = kElem == 4 ? 2 : 6;           // legal pairs of a group
    static constexpr unsigned kCodes = kElem == 4 ? 0xE4u : 0xED9C84u;   // nibble of pair p: bits 4p .. 4p + 3
    static constexpr unsigned kBlocks = (K / G + P - 1) / P;   // pair bytes per row
    static constexpr unsigned kSteps = 8;                       // .sp instructions per warpgroup and iteration
    static constexpr size_t kSmem = (size_t)(M * KC + N * K) * kElem;
    using Acc = typename std::conditional<kInt, int, float>::type;
};
static_assert(SLeg<CRO_SPARSE_LEG_S8>::kSmem == 160 * 1024 && SLeg<CRO_SPARSE_LEG_F16>::kSmem == 160 * 1024 &&
                  SLeg<CRO_SPARSE_LEG_TF32>::kSmem == 160 * 1024,
              "every leg's operands take 160 KiB of an H100 SM's shared memory");

SM_TILE_WGMMA_SP(wgmma_sp_s8, int, "+r", "m64n256k64.s32.s8.s8", "0", "")
SM_TILE_WGMMA_SP(wgmma_sp_e4m3, float, "+f", "m64n256k64.f32.e4m3.e4m3", "0", ", 1, 1")
SM_TILE_WGMMA_SP(wgmma_sp_e5m2, float, "+f", "m64n256k64.f32.e5m2.e5m2", "0", ", 1, 1")
SM_TILE_WGMMA_SP(wgmma_sp_bf16_0, float, "+f", "m64n256k32.f32.bf16.bf16", "0", ", 1, 1, 0, 0")
SM_TILE_WGMMA_SP(wgmma_sp_bf16_1, float, "+f", "m64n256k32.f32.bf16.bf16", "1", ", 1, 1, 0, 0")
SM_TILE_WGMMA_SP(wgmma_sp_f16_0, float, "+f", "m64n256k32.f32.f16.f16", "0", ", 1, 1, 0, 0")
SM_TILE_WGMMA_SP(wgmma_sp_f16_1, float, "+f", "m64n256k32.f32.f16.f16", "1", ", 1, 1, 0, 0")
SM_TILE_WGMMA_SP(wgmma_sp_tf32_0, float, "+f", "m64n256k16.f32.tf32.tf32", "0", ", 1, 1")
SM_TILE_WGMMA_SP(wgmma_sp_tf32_1, float, "+f", "m64n256k16.f32.tf32.tf32", "1", ", 1, 1")

// Byte e of the operands of `seed` (include/croprobe.h).
__device__ __forceinline__ unsigned operand_byte(unsigned long long seed, unsigned e) {
    return (unsigned)(pattern_word(seed, e / 8) >> (8 * (e % 8))) & 0xFFu;
}

// The pair of group g of row m: an index into the leg's pair order.
template <unsigned LEG>
__device__ __forceinline__ unsigned pair_of(unsigned long long seed, unsigned m, unsigned g) {
    using L = SLeg<LEG>;
    return (g + operand_byte(seed, L::M * L::KC + L::K * L::N + m * L::kBlocks + g / L::P)) % L::P;
}

// The value v as each leg's element type.
template <unsigned LEG>
__device__ __forceinline__ void store_operand(unsigned char* p, int v) {
    if constexpr (LEG == CRO_SPARSE_LEG_S8) *reinterpret_cast<signed char*>(p) = (signed char)v;
    else if constexpr (LEG == CRO_SPARSE_LEG_E4M3) *p = (unsigned char)__nv_cvt_float_to_fp8((float)v, __NV_SATFINITE, __NV_E4M3);
    else if constexpr (LEG == CRO_SPARSE_LEG_E5M2) *p = (unsigned char)__nv_cvt_float_to_fp8((float)v, __NV_SATFINITE, __NV_E5M2);
    else if constexpr (LEG == CRO_SPARSE_LEG_BF16) *reinterpret_cast<__nv_bfloat16*>(p) = __float2bfloat16_rn((float)v);
    else if constexpr (LEG == CRO_SPARSE_LEG_F16) *reinterpret_cast<__half*>(p) = __int2half_rn(v);
    else *reinterpret_cast<float*>(p) = (float)v;
}

// Raw bits of value j, canon (the f32 legs take -0 as 0), the expected value's bits, the compare, injection.
template <unsigned LEG>
__device__ __forceinline__ unsigned value_bits(const typename SLeg<LEG>::Acc (&acc)[128], int j) {
    if constexpr (SLeg<LEG>::kInt) return (unsigned)acc[j];
    else return __float_as_uint(acc[j]);
}
template <unsigned LEG>
__device__ __forceinline__ unsigned canon(unsigned bits) {
    if constexpr (SLeg<LEG>::kInt) return bits;
    else return bits == 0x80000000u ? 0u : bits;
}
template <unsigned LEG>
__device__ __forceinline__ unsigned expected_bits(int e) {
    if constexpr (SLeg<LEG>::kInt) return (unsigned)e;
    else return __float_as_uint((float)e);
}
template <unsigned LEG>
__device__ __forceinline__ bool value_equal(unsigned bits, int e) {
    if constexpr (SLeg<LEG>::kInt) return (int)bits == e;
    else return __uint_as_float(bits) == (float)e;
}
template <unsigned LEG>
__device__ __forceinline__ void inject(typename SLeg<LEG>::Acc (&acc)[128], int j, unsigned mask) {
    if constexpr (SLeg<LEG>::kInt) acc[j] = (int)((unsigned)acc[j] ^ mask);
    else acc[j] = __uint_as_float(__float_as_uint(acc[j]) ^ mask);
}

// Records the warp's mismatching values of chunk C (values 32 C .. 32 C + 31; bit q of m: value 32 C + q).  The whole
// warp calls this (some lane has m != 0).
template <unsigned LEG, int C>
__device__ __forceinline__ void record(const typename SLeg<LEG>::Acc (&acc)[128], unsigned m, unsigned r0, unsigned c0,
                                       unsigned smid, const SparseArgs& a) {
    constexpr unsigned N = SLeg<LEG>::N;
    unsigned long long base = warp_claim(__popc(m), a.claims, CRO_SPARSE_RECORDS, [](unsigned) {});
#pragma unroll
    for (int q = 0; q < 32; ++q) {
        const int j = 32 * C + q;
        if (!((m >> q) & 1u)) continue;
        if (base < CRO_SPARSE_RECORDS) {
            const unsigned row = r0 + 8u * ((j >> 1) & 1), col = 8u * (j >> 2) + c0 + (j & 1);
            a.rec[base] = cro_sparse_fault{LEG, smid, row, col, __ldg(a.expect + row * N + col), value_bits<LEG>(acc, j)};
        }
        ++base;
    }
}

template <unsigned LEG, int C>
__device__ __forceinline__ unsigned compare(const typename SLeg<LEG>::Acc (&acc)[128], unsigned r0, unsigned c0, unsigned smid,
                                            const SparseArgs& a, unsigned long long* efold) {
    constexpr unsigned N = SLeg<LEG>::N;
    unsigned m = 0;
#pragma unroll
    for (int q = 0; q < 32; ++q) {
        const int j = 32 * C + q;
        const unsigned row = r0 + 8u * ((j >> 1) & 1), col = 8u * (j >> 2) + c0 + (j & 1);
        const int e = __ldg(a.expect + row * N + col);
        *efold += (unsigned long long)canon<LEG>(expected_bits<LEG>(e)) * (2u * (row * N + col) + 1u);
        if (!value_equal<LEG>(value_bits<LEG>(acc, j), e)) m |= 1u << q;
    }
    if (__ballot_sync(0xffffffffu, m != 0)) record<LEG, C>(acc, m, r0, c0, smid, a);
    return __popc(m);
}

// Instruction s of an iteration: selector s % 2 for the forms that take two.
template <unsigned LEG, unsigned S>
__device__ __forceinline__ void sp_step(typename SLeg<LEG>::Acc (&acc)[128], unsigned long long da, unsigned long long db,
                                        unsigned meta) {
    constexpr int scale = S != 0;
    if constexpr (LEG == CRO_SPARSE_LEG_S8) wgmma_sp_s8(acc, da, db, meta, scale);
    else if constexpr (LEG == CRO_SPARSE_LEG_E4M3) wgmma_sp_e4m3(acc, da, db, meta, scale);
    else if constexpr (LEG == CRO_SPARSE_LEG_E5M2) wgmma_sp_e5m2(acc, da, db, meta, scale);
    else if constexpr (LEG == CRO_SPARSE_LEG_BF16 && S % 2 == 0) wgmma_sp_bf16_0(acc, da, db, meta, scale);
    else if constexpr (LEG == CRO_SPARSE_LEG_BF16) wgmma_sp_bf16_1(acc, da, db, meta, scale);
    else if constexpr (LEG == CRO_SPARSE_LEG_F16 && S % 2 == 0) wgmma_sp_f16_0(acc, da, db, meta, scale);
    else if constexpr (LEG == CRO_SPARSE_LEG_F16) wgmma_sp_f16_1(acc, da, db, meta, scale);
    else if constexpr (S % 2 == 0) wgmma_sp_tf32_0(acc, da, db, meta, scale);
    else wgmma_sp_tf32_1(acc, da, db, meta, scale);
}

template <unsigned LEG, unsigned S>
__device__ __forceinline__ void sp_steps(typename SLeg<LEG>::Acc (&acc)[128], unsigned long long da, unsigned long long db,
                                         const unsigned (&meta)[8]) {
    if constexpr (S < SLeg<LEG>::kSteps) {
        // one instruction reads 32 bytes of K of A (2 core matrices, +256 bytes) and 64 of B (4, +512): >> 4 in a descriptor
        sp_step<LEG, S>(acc, da + 16u * S, db + 32u * S, meta[S]);
        sp_steps<LEG, S + 1>(acc, da, db, meta);
    }
}

// Applies (and, applied again, takes back) a thread's substitution `sub` (sparse_kernel's s_sub) to its registers.
__device__ __forceinline__ void substitute(unsigned (&meta)[8], unsigned sub) {
    const unsigned flip = sub ? (sub & 0xFu) << (4 * ((sub >> 4) & 7u)) : 0u;
#pragma unroll
    for (unsigned s = 0; s < 8; ++s) meta[s] ^= s == ((sub >> 8) & 7u) ? flip : 0u;
}

template <unsigned LEG>
__global__ void __launch_bounds__(kSparseThreads, 1) sparse_kernel(const SparseArgs a) {
    using L = SLeg<LEG>;
    using Acc = typename L::Acc;
    constexpr unsigned M = L::M, N = L::N, K = L::K, KC = L::KC, ELEM = L::kElem;
    extern __shared__ __align__(128) unsigned char sp_smem[];
    __shared__ unsigned long long s_mism, s_fold_mism, s_fold, s_t0;
    __shared__ long long s_k0;
    __shared__ unsigned s_sub[kSparseThreads];   // each thread's substitution: 0, or 1 << 16 | instruction << 8 |
                                                 // nibble << 4 | (old code ^ new code)
    unsigned char* const sA = sp_smem;                          // compressed A, M x KC
    unsigned char* const sB = sp_smem + (size_t)M * KC * ELEM;  // B^T, N x K
    const unsigned tid = threadIdx.x;
    if (tid == 0) s_mism = s_fold_mism = s_fold = 0;

    // operands (include/croprobe.h): compressed A[m][c] is byte m * KC + c, B[k][n] byte M * KC + k * N + n
    for (unsigned w = tid; w < (M * KC + K * N) / 8; w += kSparseThreads) {
        const unsigned long long v = pattern_word(a.seed, w);
#pragma unroll
        for (unsigned b = 0; b < 8; ++b) {
            const unsigned e = 8 * w + b, byte = (unsigned)(v >> (8 * b)) & 0xFFu;
            int x = L::kInt ? (int)(signed char)byte : (int)(byte & 7u) - 4;
            if (e < M * KC) {
                x = L::kInt ? (x ? x : 1) : x + (x >= 0);     // a kept value is never 0
                store_operand<LEG>(sA + kmajor_off<ELEM, KC>(e / KC, e % KC), x);
            } else {
                store_operand<LEG>(sB + kmajor_off<ELEM, K>((e - M * KC) % N, (e - M * KC) / N), x);
            }
        }
    }
    asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");

    unsigned smid, nsmid;
    asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
    asm volatile("mov.u32 %0, %%nsmid;" : "=r"(nsmid));
    const unsigned wg = tid >> 7, warp = tid >> 5, lane = tid & 31u, q = lane & 3u;
    const unsigned r0 = 64u * wg + 16u * (warp & 3u) + (lane >> 2), c0 = 2u * q;
    const Injection inj = resolve_injection(a, r0, smid);

    // this thread's metadata register of each instruction, and the substitution it makes if it holds that nibble.  In
    // the 16- and 32-bit forms only the threads with q / 2 == selector supply the register; the other pair holds every
    // nibble advanced to the next legal pair, so an instruction that read the wrong pair would compute a wrong answer
    // (a selector fault fails a clean call), and a substitution is made only where the register is read.
    unsigned meta[L::kSteps];
    unsigned sub = 0;
    const bool sub_here = a.meta && (a.meta_sm < 0 || (unsigned)a.meta_sm == smid);
#pragma unroll
    for (unsigned s = 0; s < L::kSteps; ++s) {
        const bool supplies = ELEM == 1 || (q >> 1) == (s & 1u);
        unsigned reg = 0, hit_n = 8, hit_code = 0;
#pragma unroll
        for (unsigned n = 0; n < 8; ++n) {
            const unsigned row = ELEM == 1 ? r0 + 8u * (q & 1u) : r0 + 8u * (n >> 2);
            const unsigned g = ELEM == 1 ? 16u * s + 8u * (q >> 1) + n : 8u * s + 4u * (q & 1u) + (n & 3u);
            const unsigned p = pair_of<LEG>(a.seed, row, g);
            reg |= ((L::kCodes >> (4 * (supplies ? p : (p + 1) % L::P))) & 0xFu) << (4 * n);
            if (supplies && sub_here && row == a.meta_row && g == a.meta_group) {
                hit_n = n;
                hit_code = (L::kCodes >> (4 * ((p + 1) % L::P))) & 0xFu;      // the next legal pair
            }
        }
        meta[s] = reg;
        if (hit_n < 8) sub = 1u << 16 | s << 8 | hit_n << 4 | (((reg >> (4 * hit_n)) & 0xFu) ^ hit_code);
    }
    s_sub[tid] = sub;
    __syncthreads();

    Acc acc[128];
#pragma unroll
    for (int j = 0; j < 128; ++j) acc[j] = 0;
    const unsigned long long da = wgmma_desc(smem_u32(sA) + wg * 64u * KC * ELEM, 8u * KC * ELEM);
    const unsigned long long db = wgmma_desc(smem_u32(sB), 8u * K * ELEM);
    const unsigned w0 = 2u * (r0 * N + c0) + 1u;                   // value j's weight 2e + 1 is w0 + a constant
    unsigned long long run = 0;
    if (tid == 0) {                             // only thread 0's window is published: kept out of the registers
        s_t0 = globaltimer_ns();
        s_k0 = clock64();
    }
    for (unsigned it = 0; it < a.iterations; ++it) {
        // test only: the substitution goes in before the fence and out after the wait (nothing touches a register
        // between the instructions)
        if (a.meta && it == a.meta_iter) substitute(meta, s_sub[tid]);
        asm volatile("wgmma.fence.sync.aligned;\n" ::: "memory");
        sp_steps<LEG, 0>(acc, da, db, meta);
        asm volatile("wgmma.commit_group.sync.aligned;\n" ::: "memory");
        asm volatile("wgmma.wait_group.sync.aligned 0;\n" ::: "memory");
        if (a.meta && it == a.meta_iter) substitute(meta, s_sub[tid]);
#pragma unroll
        for (int j = 0; j < 128; ++j) {
            if constexpr (L::kInt) asm volatile("" : "+r"(acc[j])::"memory");
            else asm volatile("" : "+f"(acc[j])::"memory");
        }
        if (it == inj.iter) {                                        // test only: one compare on the clean path
#pragma unroll
            for (int j = 0; j < 128; ++j) {
                const unsigned col = 8u * (j >> 2) + c0 + (j & 1);
                if (((inj.rows >> ((j >> 1) & 1)) & 1u) && (a.inj_col < 0 || (unsigned)a.inj_col == col))
                    inject<LEG>(acc, j, (unsigned)a.inj_mask);
            }
        }
        __syncwarp();
        unsigned long long f = 0;
#pragma unroll
        for (int j = 0; j < 128; ++j)
            f += (unsigned long long)canon<LEG>(value_bits<LEG>(acc, j)) * (w0 + 2u * (8u * N * ((j >> 1) & 1) + 8u * (j >> 2) + (j & 1)));
        run += f;
    }
    const long long k1 = clock64();
    const unsigned long long t1 = globaltimer_ns();

    unsigned long long efold = 0;
    unsigned mism = compare<LEG, 0>(acc, r0, c0, smid, a, &efold);
    mism += compare<LEG, 1>(acc, r0, c0, smid, a, &efold);
    mism += compare<LEG, 2>(acc, r0, c0, smid, a, &efold);
    mism += compare<LEG, 3>(acc, r0, c0, smid, a, &efold);
    const unsigned fold_bad = run != (unsigned long long)a.iterations * efold ? 1u : 0u;
    publish_cta<CRO_SPARSE_MAX_SMS>(a, mism, fold_bad, run, s_t0, t1, s_k0, k1, smid, nsmid, s_mism, s_fold_mism, s_fold);
}

template <unsigned LEG>
cudaError_t launch_leg(const SparseArgs& a, int grid, cudaStream_t st) {
    constexpr size_t smem = SLeg<LEG>::kSmem;
    cudaError_t e = cudaFuncSetAttribute(sparse_kernel<LEG>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    sparse_kernel<LEG><<<grid, kSparseThreads, smem, st>>>(a);
    return cudaGetLastError();
}

}  // namespace

cudaError_t launch_sparse(unsigned leg, const SparseArgs& a, int grid, cudaStream_t st) {
    if (grid < 1) return cudaErrorInvalidValue;
    switch (leg) {
        case CRO_SPARSE_LEG_S8: return launch_leg<CRO_SPARSE_LEG_S8>(a, grid, st);
        case CRO_SPARSE_LEG_E4M3: return launch_leg<CRO_SPARSE_LEG_E4M3>(a, grid, st);
        case CRO_SPARSE_LEG_E5M2: return launch_leg<CRO_SPARSE_LEG_E5M2>(a, grid, st);
        case CRO_SPARSE_LEG_BF16: return launch_leg<CRO_SPARSE_LEG_BF16>(a, grid, st);
        case CRO_SPARSE_LEG_F16: return launch_leg<CRO_SPARSE_LEG_F16>(a, grid, st);
        case CRO_SPARSE_LEG_TF32: return launch_leg<CRO_SPARSE_LEG_TF32>(a, grid, st);
        default: return cudaErrorInvalidValue;
    }
}

}  // namespace cro
