// precision_kernels.cu — the precision probe's kernels (cro_probe_precision): every SM computes its leg's answer tile
// D = A * B `iterations` times from operands it generates into its own shared memory, and checks every value for
// IEEE equality with the exact answer (include/croprobe.h, "SM precision").  One template per leg:
//   F64          mma.sync m16n8k16 .f64 (DMMA), 8 warps of 16 rows, chained over K with the accumulator zeroed per
//                iteration
//   DFMA         the same 32-value fragment computed by DFMA chains on the CUDA cores
//   TF32, F16,   wgmma.mma_async m64n256 (HGMMA / QGMMA), each of the two warpgroups owning 64 rows, chained over K
//   F16ACC, E5M2 with scale-d = 0 on the first instruction of every iteration (F16ACC: 64 f16x2 accumulators)
//   HFMA2        the F16ACC fragment computed by HFMA2 chains, f16 accumulators, (col, col + 1) packed
// The wgmma legs keep their operands in the canonical K-major no-swizzle layout (kmajor_off, sm_tile.cuh); B is held
// transposed (N rows of K).  The F64 legs keep A and B^T row-major with rows of K + 4 doubles, so that the eight rows
// a fragment load touches fall on distinct banks.
// After each iteration every thread adds sum_j canon(value_j) * (2e_j + 1) to a running fold (e_j = row * N + col); at
// the end it compares the fold with iterations * the fold of the expected values, and the last answer element by
// element with the expected tile (global memory, L2-resident, shared by all CTAs).  Mismatches are recorded with the
// compute probe's idiom (warp_claim).
#include <cuda_fp16.h>
#include <cuda_fp8.h>

#include <type_traits>

#include "precision_kernels.cuh"
#include "sm_tile.cuh"
#include "warp_claim.cuh"

namespace cro {

namespace {

template <unsigned LEG> struct PLeg {
    static constexpr bool kF64 = LEG == CRO_PRECISION_LEG_F64 || LEG == CRO_PRECISION_LEG_DFMA;   // the F64 fragment
    static constexpr bool kTensor = LEG != CRO_PRECISION_LEG_DFMA && LEG != CRO_PRECISION_LEG_HFMA2;
    static constexpr bool kHalf = LEG == CRO_PRECISION_LEG_F16ACC || LEG == CRO_PRECISION_LEG_HFMA2;   // f16 accumulators
    static constexpr unsigned M = CRO_PRECISION_M;
    static constexpr unsigned N = kF64 ? CRO_PRECISION_F64_N : CRO_PRECISION_N;
    static constexpr unsigned K = kF64 ? CRO_PRECISION_F64_K : LEG == CRO_PRECISION_LEG_TF32 ? CRO_PRECISION_TF32_K : CRO_PRECISION_K;
    static constexpr unsigned kElem = kF64 ? 8 : LEG == CRO_PRECISION_LEG_TF32 ? 4 : LEG == CRO_PRECISION_LEG_E5M2 ? 1 : 2;
    static constexpr unsigned kLd = K + 4;                  // F64 legs: doubles per shared-memory row
    static constexpr unsigned kVals = kF64 ? 32 : 128;      // values per thread
    static constexpr unsigned kRegs = kHalf ? 64 : kVals;   // accumulator registers per thread
    static constexpr unsigned kBits = kF64 ? 64 : kHalf ? 16 : 32;
    static constexpr size_t kSmem = kF64 ? (size_t)(M + N) * kLd * 8 : (size_t)(M + N) * K * kElem;
    using Acc = typename std::conditional<kF64, double, typename std::conditional<kHalf, unsigned, float>::type>::type;
    using Bits = typename std::conditional<kF64, unsigned long long, unsigned>::type;
};
static_assert(PLeg<CRO_PRECISION_LEG_F64>::kSmem <= 227 * 1024 && PLeg<CRO_PRECISION_LEG_TF32>::kSmem <= 227 * 1024 &&
                  PLeg<CRO_PRECISION_LEG_F16>::kSmem <= 227 * 1024,
              "one CTA's operands fit an H100 SM's shared memory");

SM_TILE_WGMMA(wgmma_tf32, float, 128, "+f", "m64n256k8.f32.tf32.tf32", ", 1, 1")
SM_TILE_WGMMA(wgmma_f16, float, 128, "+f", "m64n256k16.f32.f16.f16", ", 1, 1, 0, 0")
SM_TILE_WGMMA(wgmma_e5m2, float, 128, "+f", "m64n256k32.f32.e5m2.e5m2", ", 1, 1")
SM_TILE_WGMMA(wgmma_f16acc, unsigned, 64, "+r", "m64n256k16.f16.f16.f16", ", 1, 1, 0, 0")

// d += a * b for one 16 x 8 x 16 tile of the F64 leg (DMMA).
__device__ __forceinline__ void dmma(double* d, const double (&a)[8], const double (&b)[4]) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0, %1, %2, %3}, {%4, %5, %6, %7, %8, %9, %10, %11}, "
                 "{%12, %13, %14, %15}, {%0, %1, %2, %3};\n"
                 : "+d"(d[0]), "+d"(d[1]), "+d"(d[2]), "+d"(d[3])
                 : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]), "d"(b[0]),
                   "d"(b[1]), "d"(b[2]), "d"(b[3]));
}

__device__ __forceinline__ unsigned hfma2(unsigned a, unsigned b, unsigned c) {
    unsigned d;
    asm volatile("fma.rn.f16x2 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
}

// The operand value v as each leg's element type.
template <unsigned LEG>
__device__ __forceinline__ void store_operand(unsigned char* p, int v) {
    if constexpr (PLeg<LEG>::kF64) *reinterpret_cast<double*>(p) = (double)v;
    else if constexpr (LEG == CRO_PRECISION_LEG_TF32) *reinterpret_cast<float*>(p) = (float)v;
    else if constexpr (LEG == CRO_PRECISION_LEG_E5M2) *p = (unsigned char)__nv_cvt_float_to_fp8((float)v, __NV_SATFINITE, __NV_E5M2);
    else *reinterpret_cast<__half*>(p) = __int2half_rn(v);
}

// Raw bits of value j (zero-extended), canon (-0 taken as 0), the expected value's bits, IEEE equality, injection.
template <unsigned LEG>
__device__ __forceinline__ typename PLeg<LEG>::Bits value_bits(const typename PLeg<LEG>::Acc (&acc)[PLeg<LEG>::kRegs], int j) {
    if constexpr (PLeg<LEG>::kF64) return (unsigned long long)__double_as_longlong(acc[j]);
    else if constexpr (PLeg<LEG>::kHalf) return (acc[j >> 1] >> (16 * (j & 1))) & 0xFFFFu;
    else return __float_as_uint(acc[j]);
}
template <unsigned LEG>
__device__ __forceinline__ typename PLeg<LEG>::Bits canon(typename PLeg<LEG>::Bits bits) {
    return bits == (typename PLeg<LEG>::Bits)1 << (PLeg<LEG>::kBits - 1) ? 0 : bits;
}
template <unsigned LEG>
__device__ __forceinline__ typename PLeg<LEG>::Bits expected_bits(long long e) {
    if constexpr (PLeg<LEG>::kF64) return (unsigned long long)__double_as_longlong((double)e);
    else if constexpr (PLeg<LEG>::kHalf) return __half_as_ushort(__int2half_rn((int)e));
    else return __float_as_uint((float)e);
}
template <unsigned LEG>
__device__ __forceinline__ bool ieee_equal(typename PLeg<LEG>::Bits bits, long long e) {
    if constexpr (PLeg<LEG>::kF64) return __longlong_as_double((long long)bits) == (double)e;
    else if constexpr (PLeg<LEG>::kHalf) return __half2float(__ushort_as_half((unsigned short)bits)) == (float)e;   // exact widening
    else return __uint_as_float((unsigned)bits) == (float)e;
}
template <unsigned LEG>
__device__ __forceinline__ void inject(typename PLeg<LEG>::Acc (&acc)[PLeg<LEG>::kRegs], int j, unsigned long long mask) {
    if constexpr (PLeg<LEG>::kF64) acc[j] = __longlong_as_double(__double_as_longlong(acc[j]) ^ (long long)mask);
    else if constexpr (PLeg<LEG>::kHalf) acc[j >> 1] ^= ((unsigned)mask & 0xFFFFu) << (16 * (j & 1));
    else acc[j] = __uint_as_float(__float_as_uint(acc[j]) ^ (unsigned)mask);
}

// Records the warp's mismatching values of chunk C (values 32 C .. 32 C + 31; bit q of m: value 32 C + q).  The whole
// warp calls this (some lane has m != 0).
template <unsigned LEG, int C>
__device__ __forceinline__ void record(const typename PLeg<LEG>::Acc (&acc)[PLeg<LEG>::kRegs], unsigned m, unsigned r0,
                                       unsigned c0, unsigned smid, const PrecisionArgs& a) {
    constexpr unsigned N = PLeg<LEG>::N;
    unsigned long long base = warp_claim(__popc(m), a.claims, CRO_PRECISION_RECORDS, [](unsigned) {});
#pragma unroll
    for (int q = 0; q < 32; ++q) {
        const int j = 32 * C + q;
        if (!((m >> q) & 1u)) continue;
        if (base < CRO_PRECISION_RECORDS) {
            const unsigned row = r0 + 8u * ((j >> 1) & 1), col = 8u * (j >> 2) + c0 + (j & 1);
            a.rec[base] = cro_precision_fault{LEG, smid, row, col, __ldg(a.expect + row * N + col), value_bits<LEG>(acc, j)};
        }
        ++base;
    }
}

template <unsigned LEG, int C>
__device__ __forceinline__ unsigned compare(const typename PLeg<LEG>::Acc (&acc)[PLeg<LEG>::kRegs], unsigned r0, unsigned c0,
                                            unsigned smid, const PrecisionArgs& a, unsigned long long* efold) {
    constexpr unsigned N = PLeg<LEG>::N;
    unsigned m = 0;
#pragma unroll
    for (int q = 0; q < 32; ++q) {
        const int j = 32 * C + q;
        const unsigned row = r0 + 8u * ((j >> 1) & 1), col = 8u * (j >> 2) + c0 + (j & 1);
        const long long e = __ldg(a.expect + row * N + col);
        *efold += (unsigned long long)canon<LEG>(expected_bits<LEG>(e)) * (2u * (row * N + col) + 1u);
        if (!ieee_equal<LEG>(value_bits<LEG>(acc, j), e)) m |= 1u << q;
    }
    if (__ballot_sync(0xffffffffu, m != 0)) record<LEG, C>(acc, m, r0, c0, smid, a);
    return __popc(m);
}

template <unsigned LEG>
__global__ void __launch_bounds__(kPrecisionThreads, 1) precision_kernel(const PrecisionArgs a) {
    using L = PLeg<LEG>;
    using Acc = typename L::Acc;
    constexpr unsigned M = L::M, N = L::N, K = L::K, ELEM = L::kElem, LD = L::kLd;
    extern __shared__ __align__(128) unsigned char prec_smem[];
    __shared__ unsigned long long s_mism, s_fold_mism, s_fold;
    unsigned char* const sA = prec_smem;
    unsigned char* const sB = prec_smem + (L::kF64 ? (size_t)M * LD * 8 : (size_t)M * K * ELEM);
    const unsigned tid = threadIdx.x;
    if (tid == 0) s_mism = s_fold_mism = s_fold = 0;

    // operands (include/croprobe.h): A[m][k] is element m * K + k, B[k][n] element M * K + k * N + n
    auto place = [&](unsigned e, int v) {
        const unsigned m = e < M * K ? e / K : (e - M * K) % N, k = e < M * K ? e % K : (e - M * K) / N;
        unsigned char* base = e < M * K ? sA : sB;
        if constexpr (L::kF64) store_operand<LEG>(base + ((size_t)m * LD + k) * 8, v);
        else store_operand<LEG>(base + kmajor_off<ELEM, K>(m, k), v);
    };
    if constexpr (L::kF64) {
        for (unsigned e = tid; e < M * K + K * N; e += kPrecisionThreads)       // wide: 20 low bits, sign-extended
            place(e, (int)((long long)(pattern_word(a.seed, e) << 44) >> 44));
    } else {
        for (unsigned w = tid; w < (M * K + K * N) / 8; w += kPrecisionThreads) {
            const unsigned long long v = pattern_word(a.seed, w);
#pragma unroll
            for (unsigned b = 0; b < 8; ++b) {
                const unsigned byte = (unsigned)(v >> (8 * b)) & 0xFFu;
                place(8 * w + b, L::kHalf ? (int)(byte & 3u) - 2 : (int)(byte & 7u) - 4);
            }
        }
    }
    if constexpr (L::kTensor && !L::kF64) asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");
    __syncthreads();

    unsigned smid, nsmid;
    asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
    asm volatile("mov.u32 %0, %%nsmid;" : "=r"(nsmid));
    const unsigned wg = tid >> 7, warp = tid >> 5, lane = tid & 31u;
    const unsigned r0 = (L::kF64 ? 16u * warp : 64u * wg + 16u * (warp & 3u)) + (lane >> 2), c0 = 2u * (lane & 3u);
    const Injection inj = resolve_injection(a, r0, smid);

    Acc acc[L::kRegs];
#pragma unroll
    for (int j = 0; j < (int)L::kRegs; ++j) acc[j] = 0;
    const unsigned w0 = 2u * (r0 * N + c0) + 1u;                   // value j's weight 2e + 1 is w0 + a constant
    unsigned long long run = 0;
    const unsigned long long t0 = globaltimer_ns();
    const long long k0 = clock64();
    for (unsigned it = 0; it < a.iterations; ++it) {
        if constexpr (LEG == CRO_PRECISION_LEG_F64) {
            const double* A = reinterpret_cast<const double*>(sA);
            const double* B = reinterpret_cast<const double*>(sB);     // B^T: row n holds B[.][n]
            const unsigned g = lane >> 2, t = lane & 3u;
#pragma unroll
            for (int j = 0; j < 32; ++j) acc[j] = 0;
#pragma unroll 1
            for (unsigned kb = 0; kb < K; kb += 16) {
                double fa[8];
#pragma unroll
                for (int i = 0; i < 8; ++i) fa[i] = A[(r0 + 8u * (i & 1)) * LD + kb + t + 4u * (i >> 1)];
#pragma unroll
                for (int nt = 0; nt < 8; ++nt) {
                    double fb[4];
#pragma unroll
                    for (int i = 0; i < 4; ++i) fb[i] = B[(8u * nt + g) * LD + kb + t + 4u * i];
                    dmma(acc + 4 * nt, fa, fb);
                }
            }
        } else if constexpr (LEG == CRO_PRECISION_LEG_DFMA) {
            const double* A = reinterpret_cast<const double*>(sA);
            const double* B = reinterpret_cast<const double*>(sB);
#pragma unroll
            for (int j = 0; j < 32; ++j) acc[j] = 0;
#pragma unroll 1
            for (unsigned k = 0; k < K; k += 2) {
                const double2 p = *reinterpret_cast<const double2*>(A + r0 * LD + k);
                const double2 q = *reinterpret_cast<const double2*>(A + (r0 + 8) * LD + k);
#pragma unroll
                for (int nt = 0; nt < 8; ++nt) {
                    const double2 u = *reinterpret_cast<const double2*>(B + (8u * nt + c0) * LD + k);
                    const double2 v = *reinterpret_cast<const double2*>(B + (8u * nt + c0 + 1) * LD + k);
                    acc[4 * nt] = fma(p.x, u.x, acc[4 * nt]);
                    acc[4 * nt + 1] = fma(p.x, v.x, acc[4 * nt + 1]);
                    acc[4 * nt + 2] = fma(q.x, u.x, acc[4 * nt + 2]);
                    acc[4 * nt + 3] = fma(q.x, v.x, acc[4 * nt + 3]);
                    acc[4 * nt] = fma(p.y, u.y, acc[4 * nt]);
                    acc[4 * nt + 1] = fma(p.y, v.y, acc[4 * nt + 1]);
                    acc[4 * nt + 2] = fma(q.y, u.y, acc[4 * nt + 2]);
                    acc[4 * nt + 3] = fma(q.y, v.y, acc[4 * nt + 3]);
                }
            }
        } else if constexpr (LEG == CRO_PRECISION_LEG_HFMA2) {
#pragma unroll
            for (int j = 0; j < 64; ++j) acc[j] = 0;
#pragma unroll 1
            for (unsigned kc = 0; kc < K; kc += 8) {                 // 8 halves: one 16-byte core-matrix row
                const uint4 x0 = *reinterpret_cast<const uint4*>(sA + kmajor_off<2, K>(r0, kc));
                const uint4 x1 = *reinterpret_cast<const uint4*>(sA + kmajor_off<2, K>(r0 + 8, kc));
                const unsigned a0[4] = {x0.x, x0.y, x0.z, x0.w}, a1[4] = {x1.x, x1.y, x1.z, x1.w};
#pragma unroll
                for (int g = 0; g < 32; ++g) {
                    const uint4 y0 = *reinterpret_cast<const uint4*>(sB + kmajor_off<2, K>(8u * g + c0, kc));
                    const uint4 y1 = *reinterpret_cast<const uint4*>(sB + kmajor_off<2, K>(8u * g + c0 + 1, kc));
                    const unsigned b0[4] = {y0.x, y0.y, y0.z, y0.w}, b1[4] = {y1.x, y1.y, y1.z, y1.w};
#pragma unroll
                    for (int k = 0; k < 8; ++k) {
                        const unsigned lo = (k & 1) ? 0x3232u : 0x1010u;                 // half k of A, broadcast
                        const unsigned p = __byte_perm(a0[k >> 1], 0, lo), q = __byte_perm(a1[k >> 1], 0, lo);
                        const unsigned u = __byte_perm(b0[k >> 1], b1[k >> 1], (k & 1) ? 0x7632u : 0x5410u);   // (col, col + 1)
                        acc[2 * g] = hfma2(p, u, acc[2 * g]);
                        acc[2 * g + 1] = hfma2(q, u, acc[2 * g + 1]);
                    }
                }
            }
        } else {
            constexpr unsigned SBO = 8u * K * ELEM;
            const unsigned long long da = wgmma_desc(smem_u32(sA) + wg * 64u * K * ELEM, SBO);
            const unsigned long long db = wgmma_desc(smem_u32(sB), SBO);
            asm volatile("wgmma.fence.sync.aligned;\n" ::: "memory");
#pragma unroll
            for (unsigned s = 0; s < K * ELEM / 32; ++s) {            // 32 bytes of K per instruction: +256 bytes, >> 4
                if constexpr (LEG == CRO_PRECISION_LEG_TF32) wgmma_tf32(acc, da + 16u * s, db + 16u * s, s != 0);
                else if constexpr (LEG == CRO_PRECISION_LEG_F16) wgmma_f16(acc, da + 16u * s, db + 16u * s, s != 0);
                else if constexpr (LEG == CRO_PRECISION_LEG_F16ACC) wgmma_f16acc(acc, da + 16u * s, db + 16u * s, s != 0);
                else wgmma_e5m2(acc, da + 16u * s, db + 16u * s, s != 0);
            }
            asm volatile("wgmma.commit_group.sync.aligned;\n" ::: "memory");
            asm volatile("wgmma.wait_group.sync.aligned 0;\n" ::: "memory");
#pragma unroll
            for (int j = 0; j < (int)L::kRegs; ++j) {
                if constexpr (L::kHalf) asm volatile("" : "+r"(acc[j])::"memory");
                else asm volatile("" : "+f"(acc[j])::"memory");
            }
        }
        if (it == inj.iter) {                                        // test only: one compare on the clean path
#pragma unroll
            for (int j = 0; j < (int)L::kVals; ++j) {
                const unsigned col = 8u * (j >> 2) + c0 + (j & 1);
                if (((inj.rows >> ((j >> 1) & 1)) & 1u) && (a.inj_col < 0 || (unsigned)a.inj_col == col)) inject<LEG>(acc, j, a.inj_mask);
            }
        }
        __syncwarp();
        unsigned long long f = 0;
#pragma unroll
        for (int j = 0; j < (int)L::kVals; ++j)
            f += (unsigned long long)canon<LEG>(value_bits<LEG>(acc, j)) * (w0 + 2u * (8u * N * ((j >> 1) & 1) + 8u * (j >> 2) + (j & 1)));
        run += f;
    }
    const long long k1 = clock64();
    const unsigned long long t1 = globaltimer_ns();

    unsigned long long efold = 0;
    unsigned mism = compare<LEG, 0>(acc, r0, c0, smid, a, &efold);
    if constexpr (L::kVals == 128) {
        mism += compare<LEG, 1>(acc, r0, c0, smid, a, &efold);
        mism += compare<LEG, 2>(acc, r0, c0, smid, a, &efold);
        mism += compare<LEG, 3>(acc, r0, c0, smid, a, &efold);
    }
    const unsigned fold_bad = run != (unsigned long long)a.iterations * efold ? 1u : 0u;
    publish_cta<CRO_PRECISION_MAX_SMS>(a, mism, fold_bad, run, t0, t1, k0, k1, smid, nsmid, s_mism, s_fold_mism, s_fold);
}

template <unsigned LEG>
cudaError_t launch_leg(const PrecisionArgs& a, int grid, cudaStream_t st) {
    constexpr size_t smem = PLeg<LEG>::kSmem;
    cudaError_t e = cudaFuncSetAttribute(precision_kernel<LEG>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    precision_kernel<LEG><<<grid, kPrecisionThreads, smem, st>>>(a);
    return cudaGetLastError();
}

}  // namespace

cudaError_t launch_precision(unsigned leg, const PrecisionArgs& a, int grid, cudaStream_t st) {
    if (grid < 1) return cudaErrorInvalidValue;
    switch (leg) {
        case CRO_PRECISION_LEG_F64: return launch_leg<CRO_PRECISION_LEG_F64>(a, grid, st);
        case CRO_PRECISION_LEG_DFMA: return launch_leg<CRO_PRECISION_LEG_DFMA>(a, grid, st);
        case CRO_PRECISION_LEG_TF32: return launch_leg<CRO_PRECISION_LEG_TF32>(a, grid, st);
        case CRO_PRECISION_LEG_F16: return launch_leg<CRO_PRECISION_LEG_F16>(a, grid, st);
        case CRO_PRECISION_LEG_F16ACC: return launch_leg<CRO_PRECISION_LEG_F16ACC>(a, grid, st);
        case CRO_PRECISION_LEG_E5M2: return launch_leg<CRO_PRECISION_LEG_E5M2>(a, grid, st);
        case CRO_PRECISION_LEG_HFMA2: return launch_leg<CRO_PRECISION_LEG_HFMA2>(a, grid, st);
        default: return cudaErrorInvalidValue;
    }
}

}  // namespace cro
