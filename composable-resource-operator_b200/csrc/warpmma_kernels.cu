// warpmma_kernels.cu — the warp-MMA probe's kernels (cro_probe_warpmma): every SM computes its leg's answer tile
// D = A * B `iterations` times with warp-synchronous mma.sync, every operand fragment loaded by ldmatrix from operands
// it generates into its own shared memory, and checks every value against the exact answer (include/croprobe.h, "SM
// warp-MMA").  One template per leg:
//   S8       mma.sync m16n8k32 .s32.s8.s8 (IMMA.16832.S8.S8), B^T by ldmatrix.x4
//   F16      mma.sync m16n8k16 .f32.f16.f16.f32 (HMMA.16816.F32), B by ldmatrix.x4.trans
//   BF16     mma.sync m16n8k16 .f32.bf16.bf16.f32 (HMMA.16816.F32.BF16), B by ldmatrix.x4.trans
//   TF32     mma.sync m16n8k8 .f32.tf32.tf32.f32 (HMMA.1688.F32.TF32), B^T by ldmatrix.x4
//   F16ACC   mma.sync m16n8k16 .f16.f16.f16.f16 (HMMA.16816.F16), B by ldmatrix.x4.trans, 64 f16x2 accumulators
//   MOVE     the source tile through ldmatrix, movmatrix.trans, stmatrix.trans, ldmatrix.trans, stmatrix, ldmatrix
// Warp w owns rows 16w .. 16w + 15 across all 32 n-tiles of 8 columns.  Each k-step of an arithmetic leg takes one
// ldmatrix.x4 of A (16 rows x 32 bytes of K) and one ldmatrix.x4 of B per two n-tiles; the k-step loop stays rolled so
// that the 128 accumulators, the A fragment and a B fragment fit the 255 registers without a spill.  Every row of
// every operand is padded by 16 bytes, so the eight row addresses of one 8 x 8 load fall on distinct bank groups.
// After each iteration every thread adds sum_j canon(value_j) * (2e_j + 1) to a running fold (e_j = row * N + col); at
// the end it compares the fold with iterations * the fold of the expected values, and the last answer element by
// element with the expected tile (global memory, L2-resident, shared by all CTAs), recording mismatches with the
// compute probe's idiom (warp_claim).
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <type_traits>

#include "sm_tile.cuh"
#include "warp_claim.cuh"
#include "warpmma_kernels.cuh"

namespace cro {

namespace {

template <unsigned LEG> struct WLeg {
    static constexpr bool kMove = LEG == CRO_WARPMMA_LEG_MOVE;
    static constexpr bool kInt = LEG == CRO_WARPMMA_LEG_S8;
    static constexpr bool kHalf = LEG == CRO_WARPMMA_LEG_F16ACC || kMove;      // 16-bit values, two per register
    static constexpr bool kTransB = LEG == CRO_WARPMMA_LEG_F16 || LEG == CRO_WARPMMA_LEG_BF16 || LEG == CRO_WARPMMA_LEG_F16ACC;
    static constexpr unsigned M = CRO_WARPMMA_M, N = CRO_WARPMMA_N;
    static constexpr unsigned K = LEG == CRO_WARPMMA_LEG_TF32 ? CRO_WARPMMA_TF32_K : CRO_WARPMMA_K;
    static constexpr unsigned kElem = LEG == CRO_WARPMMA_LEG_S8 ? 1 : LEG == CRO_WARPMMA_LEG_TF32 ? 4 : 2;
    static constexpr unsigned kLd = (kMove ? N * 2 : K * kElem) + 16;   // bytes per row: A, B^T, the MOVE tiles
    static constexpr unsigned kLdB = kTransB ? N * 2 + 16 : kLd;         // ... of B (B [k][n] or B^T [n][k])
    static constexpr unsigned kBRows = kTransB ? K : N;
    static constexpr unsigned kRegs = kHalf ? 64 : 128;                 // value registers per thread
    static constexpr size_t kSmem = kMove ? (size_t)3 * M * kLd : (size_t)M * kLd + (size_t)kBRows * kLdB;
    using Acc = typename std::conditional<kHalf, unsigned, typename std::conditional<kInt, int, float>::type>::type;
};
static_assert(WLeg<CRO_WARPMMA_LEG_F16>::kSmem == 198 * 1024 && WLeg<CRO_WARPMMA_LEG_TF32>::kSmem == 198 * 1024 &&
                  WLeg<CRO_WARPMMA_LEG_MOVE>::kSmem == 198 * 1024 && WLeg<CRO_WARPMMA_LEG_S8>::kSmem <= 198 * 1024,
              "every leg's operands fit the 227 KiB of shared memory an H100 CTA can have");
static_assert(WLeg<CRO_WARPMMA_LEG_F16>::kLd % 128 == 16 && WLeg<CRO_WARPMMA_LEG_S8>::kLd % 128 == 16,
              "a padded row starts one 16-byte bank group after the row above it");

// Fragment moves: lane l supplies the address of row l % 8 of 8 x 8 matrix l / 8; register i holds matrix i.
__device__ __forceinline__ void ldsm_x4(unsigned addr, unsigned (&r)[4]) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];\n"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr) : "memory");
}
__device__ __forceinline__ void ldsm_x4_trans(unsigned addr, unsigned (&r)[4]) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];\n"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr) : "memory");
}
__device__ __forceinline__ void stsm_x4(unsigned addr, const unsigned (&r)[4]) {
    asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};\n"
                 :: "r"(addr), "r"(r[0]), "r"(r[1]), "r"(r[2]), "r"(r[3]) : "memory");
}
__device__ __forceinline__ void stsm_x4_trans(unsigned addr, const unsigned (&r)[4]) {
    asm volatile("stmatrix.sync.aligned.m8n8.x4.trans.shared.b16 [%0], {%1, %2, %3, %4};\n"
                 :: "r"(addr), "r"(r[0]), "r"(r[1]), "r"(r[2]), "r"(r[3]) : "memory");
}
__device__ __forceinline__ unsigned movm_trans(unsigned x) {
    unsigned d;
    asm volatile("movmatrix.sync.aligned.m8n8.trans.b16 %0, %1;\n" : "=r"(d) : "r"(x));
    return d;
}

// d += a * b for one 16 x 8 tile of the leg: d is the n-tile's accumulators (4 registers, F16ACC 2).
template <unsigned LEG>
__device__ __forceinline__ void mma(typename WLeg<LEG>::Acc* d, const unsigned (&a)[4], unsigned b0, unsigned b1) {
    if constexpr (LEG == CRO_WARPMMA_LEG_S8)
        asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.s8.s8.s32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
                     "{%0, %1, %2, %3};\n"
                     : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
    else if constexpr (LEG == CRO_WARPMMA_LEG_F16)
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
                     "{%0, %1, %2, %3};\n"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
    else if constexpr (LEG == CRO_WARPMMA_LEG_BF16)
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
                     "{%0, %1, %2, %3};\n"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
    else if constexpr (LEG == CRO_WARPMMA_LEG_TF32)
        asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
                     "{%0, %1, %2, %3};\n"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
    else
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f16.f16.f16.f16 {%0, %1}, {%2, %3, %4, %5}, {%6, %7}, {%0, %1};\n"
                     : "+r"(d[0]), "+r"(d[1])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// The operand value v as each arithmetic leg's element type.
template <unsigned LEG>
__device__ __forceinline__ void store_operand(unsigned char* p, int v) {
    if constexpr (LEG == CRO_WARPMMA_LEG_S8) *reinterpret_cast<signed char*>(p) = (signed char)v;
    else if constexpr (LEG == CRO_WARPMMA_LEG_BF16) *reinterpret_cast<__nv_bfloat16*>(p) = __float2bfloat16_rn((float)v);
    else if constexpr (LEG == CRO_WARPMMA_LEG_TF32) *reinterpret_cast<float*>(p) = (float)v;
    else *reinterpret_cast<__half*>(p) = __int2half_rn(v);
}

// Raw bits of value j, canon (the f32 and f16 legs take -0 as 0), the expected value's bits, the compare, injection.
template <unsigned LEG>
__device__ __forceinline__ unsigned value_bits(const typename WLeg<LEG>::Acc (&acc)[WLeg<LEG>::kRegs], int j) {
    if constexpr (WLeg<LEG>::kHalf) return (acc[j >> 1] >> (16 * (j & 1))) & 0xFFFFu;
    else if constexpr (WLeg<LEG>::kInt) return (unsigned)acc[j];
    else return __float_as_uint(acc[j]);
}
template <unsigned LEG>
__device__ __forceinline__ unsigned canon(unsigned bits) {
    if constexpr (WLeg<LEG>::kInt || WLeg<LEG>::kMove) return bits;
    else return bits == (WLeg<LEG>::kHalf ? 0x8000u : 0x80000000u) ? 0u : bits;
}
template <unsigned LEG>
__device__ __forceinline__ unsigned expected_bits(int e) {
    if constexpr (WLeg<LEG>::kMove) return (unsigned)e & 0xFFFFu;
    else if constexpr (WLeg<LEG>::kInt) return (unsigned)e;
    else if constexpr (WLeg<LEG>::kHalf) return __half_as_ushort(__int2half_rn(e));
    else return __float_as_uint((float)e);
}
template <unsigned LEG>
__device__ __forceinline__ bool value_equal(unsigned bits, int e) {
    if constexpr (WLeg<LEG>::kMove) return bits == (unsigned)e;
    else if constexpr (WLeg<LEG>::kInt) return (int)bits == e;
    else if constexpr (WLeg<LEG>::kHalf) return __half2float(__ushort_as_half((unsigned short)bits)) == (float)e;   // exact widening
    else return __uint_as_float(bits) == (float)e;
}
template <unsigned LEG>
__device__ __forceinline__ void inject(typename WLeg<LEG>::Acc (&acc)[WLeg<LEG>::kRegs], int j, unsigned long long mask) {
    if constexpr (WLeg<LEG>::kHalf) acc[j >> 1] ^= ((unsigned)mask & 0xFFFFu) << (16 * (j & 1));
    else if constexpr (WLeg<LEG>::kInt) acc[j] = (int)((unsigned)acc[j] ^ (unsigned)mask);
    else acc[j] = __uint_as_float(__float_as_uint(acc[j]) ^ (unsigned)mask);
}

// Records the warp's mismatching values of chunk C (values 32 C .. 32 C + 31; bit q of m: value 32 C + q).  The whole
// warp calls this (some lane has m != 0).
template <unsigned LEG, int C>
__device__ __forceinline__ void record(const typename WLeg<LEG>::Acc (&acc)[WLeg<LEG>::kRegs], unsigned m, unsigned r0,
                                       unsigned c0, unsigned smid, const WarpMmaArgs& a) {
    constexpr unsigned N = WLeg<LEG>::N;
    unsigned long long base = warp_claim(__popc(m), a.claims, CRO_WARPMMA_RECORDS, [](unsigned) {});
#pragma unroll
    for (int q = 0; q < 32; ++q) {
        const int j = 32 * C + q;
        if (!((m >> q) & 1u)) continue;
        if (base < CRO_WARPMMA_RECORDS) {
            const unsigned row = r0 + 8u * ((j >> 1) & 1), col = 8u * (j >> 2) + c0 + (j & 1);
            a.rec[base] = cro_warpmma_fault{LEG, smid, row, col, __ldg(a.expect + row * N + col), value_bits<LEG>(acc, j)};
        }
        ++base;
    }
}

template <unsigned LEG, int C>
__device__ __forceinline__ unsigned compare(const typename WLeg<LEG>::Acc (&acc)[WLeg<LEG>::kRegs], unsigned r0, unsigned c0,
                                            unsigned smid, const WarpMmaArgs& a, unsigned long long* efold) {
    constexpr unsigned N = WLeg<LEG>::N;
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

template <unsigned LEG>
__global__ void __launch_bounds__(kWarpMmaThreads, 1) warpmma_kernel(const WarpMmaArgs a) {
    using L = WLeg<LEG>;
    using Acc = typename L::Acc;
    constexpr unsigned M = L::M, N = L::N, K = L::K, ELEM = L::kElem, LD = L::kLd, LDB = L::kLdB;
    extern __shared__ __align__(128) unsigned char wm_smem[];
    __shared__ unsigned long long s_mism, s_fold_mism, s_fold, s_t0;
    __shared__ long long s_k0;
    unsigned char* const sA = wm_smem;                         // A [m][k]; MOVE: the source tile S
    unsigned char* const sB = wm_smem + (size_t)M * LD;        // B [k][n] or B^T [n][k]; MOVE: T, then U
    const unsigned tid = threadIdx.x;
    if (tid == 0) s_mism = s_fold_mism = s_fold = 0;

    if constexpr (L::kMove) {
        // S[r][c] is halfword e % 4 of pattern_word(seed, e / 4), e = r * N + c: one word fills four columns
        for (unsigned w = tid; w < M * N / 4; w += kWarpMmaThreads) {
            const unsigned long long v = pattern_word(a.seed, w);
            *reinterpret_cast<uint2*>(sA + (4 * w / N) * LD + (4 * w % N) * 2) = make_uint2((unsigned)v, (unsigned)(v >> 32));
        }
    } else {
        // operands (include/croprobe.h): A[m][k] is element m * K + k, B[k][n] element M * K + k * N + n
        for (unsigned w = tid; w < (M * K + K * N) / 8; w += kWarpMmaThreads) {
            const unsigned long long v = pattern_word(a.seed, w);
#pragma unroll
            for (unsigned b = 0; b < 8; ++b) {
                const unsigned e = 8 * w + b, byte = (unsigned)(v >> (8 * b)) & 0xFFu;
                const int x = L::kInt ? (int)(signed char)byte : L::kHalf ? (int)(byte & 3u) - 2 : (int)(byte & 7u) - 4;
                if (e < M * K) {
                    store_operand<LEG>(sA + (e / K) * LD + (e % K) * ELEM, x);
                } else {
                    const unsigned k = (e - M * K) / N, n = (e - M * K) % N;
                    store_operand<LEG>(sB + (L::kTransB ? k * LDB + n * 2 : n * LD + k * ELEM), x);
                }
            }
        }
    }
    __syncthreads();

    unsigned smid, nsmid;
    asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
    asm volatile("mov.u32 %0, %%nsmid;" : "=r"(nsmid));
    const unsigned warp = tid >> 5, lane = tid & 31u;
    const unsigned r0 = 16u * warp + (lane >> 2), c0 = 2u * (lane & 3u);
    const Injection inj = resolve_injection(a, r0, smid);
    // the row and 16-byte K half whose address this lane supplies to an .x4 load of its warp's band (A, S, T, U)
    const unsigned lrow = 16u * warp + (lane & 7u) + 8u * ((lane >> 3) & 1u), lhalf = lane >> 4;
    const unsigned aLane = smem_u32(sA) + lrow * LD + 16u * lhalf;

    Acc acc[L::kRegs];
#pragma unroll
    for (int j = 0; j < (int)L::kRegs; ++j) acc[j] = 0;
    const unsigned w0 = 2u * (r0 * N + c0) + 1u;                   // value j's weight 2e + 1 is w0 + a constant
    unsigned long long run = 0;
    if (tid == 0) {                             // only thread 0's window is published: kept out of the registers
        s_t0 = globaltimer_ns();
        s_k0 = clock64();
    }
    if constexpr (L::kMove) {
        const unsigned tLane = aLane + M * LD, uLane = aLane + 2u * M * LD;
        const unsigned m16 = (unsigned)a.inj_mask & 0xFFFFu;
        for (unsigned it = 0; it < a.iterations; ++it) {
            const bool inj_now = it == inj.iter;
            __syncwarp();
#pragma unroll
            for (unsigned st = 0; st < N / 16; ++st) {              // the warp's 16 x 16 sub-tiles, 32 bytes apart
                unsigned r[4];
                ldsm_x4(aLane + 32u * st, r);
#pragma unroll
                for (int i = 0; i < 4; ++i) r[i] = movm_trans(r[i]);
                stsm_x4_trans(tLane + 32u * st, r);                 // T's blocks are S's
                __syncwarp();
                ldsm_x4_trans(tLane + 32u * st, r);
#pragma unroll
                for (unsigned i = 0; i < 4; ++i) {                  // test only: register 4 st + i holds values 8 st + 2i, + 1
                    const unsigned col = 8u * (2u * st + (i >> 1)) + c0;
                    const bool row_hit = inj_now && ((inj.rows >> (i & 1u)) & 1u);
                    r[i] ^= (row_hit && (a.inj_col < 0 || (unsigned)a.inj_col == col) ? m16 : 0u) |
                            (row_hit && (a.inj_col < 0 || (unsigned)a.inj_col == col + 1) ? m16 << 16 : 0u);
                }
                stsm_x4(uLane + 32u * st, r);                       // U holds each block transposed
                __syncwarp();
                ldsm_x4(uLane + 32u * st, r);
#pragma unroll
                for (unsigned i = 0; i < 4; ++i) acc[4 * st + i] = r[i];
            }
            unsigned long long f = 0;
#pragma unroll
            for (int j = 0; j < 128; ++j)
                f += (unsigned long long)canon<LEG>(value_bits<LEG>(acc, j)) * (w0 + 2u * (8u * N * ((j >> 1) & 1) + 8u * (j >> 2) + (j & 1)));
            run += f;
        }
    } else {
        // B: lane l supplies row l % 8 of matrix l / 8; for B [k][n] (.trans) matrices 0, 1 are k 0-7, 8-15 of n-tile 2p
        // and 2, 3 those of n-tile 2p + 1; for B^T [n][k] matrices 0, 1 are K halves 0, 1 of n-tile 2p, 2, 3 of 2p + 1
        const unsigned bLane = L::kTransB ? smem_u32(sB) + ((lane & 7u) + 8u * ((lane >> 3) & 1u)) * LDB + 16u * lhalf
                                          : smem_u32(sB) + ((lane & 7u) + 8u * lhalf) * LD + 16u * ((lane >> 3) & 1u);
        // test only: the substitution this lane makes, resolved once: in iteration addr_iter, the A load of instruction
        // addr_step reads row lrow ^ 1 (addr_delta bytes away) for the half this lane supplies
        const bool sub = a.addr && (a.addr_sm < 0 || (unsigned)a.addr_sm == smid) && lrow == a.addr_row &&
                         (a.addr_kstep & 1u) == lhalf;
        const unsigned addr_step = sub ? a.addr_kstep >> 1 : ~0u;
        const unsigned addr_delta = (lrow & 1u) ? 0u - LD : LD;
        for (unsigned it = 0; it < a.iterations; ++it) {
#pragma unroll
            for (int j = 0; j < (int)L::kRegs; ++j) acc[j] = 0;
            const unsigned qs = it == a.addr_iter ? addr_step : ~0u;
#pragma unroll 1
            for (unsigned s = 0; s < K * ELEM / 32; ++s) {           // one mma.sync per n-tile: 32 bytes of K
                unsigned fa[4];
                ldsm_x4(aLane + 32u * s + (s == qs ? addr_delta : 0u), fa);
                const unsigned bs = L::kTransB ? bLane + 16u * LDB * s : bLane + 32u * s;
#pragma unroll
                for (unsigned p = 0; p < N / 16; ++p) {
                    unsigned fb[4];
                    if constexpr (L::kTransB) ldsm_x4_trans(bs + 32u * p, fb);
                    else ldsm_x4(bs + 16u * LD * p, fb);
                    mma<LEG>(acc + (L::kHalf ? 4 : 8) * p, fa, fb[0], fb[1]);
                    mma<LEG>(acc + (L::kHalf ? 4 : 8) * p + (L::kHalf ? 2 : 4), fa, fb[2], fb[3]);
                }
            }
            if (it == inj.iter) {                                        // test only: one compare on the clean path
#pragma unroll
                for (int j = 0; j < 128; ++j) {
                    const unsigned col = 8u * (j >> 2) + c0 + (j & 1);
                    if (((inj.rows >> ((j >> 1) & 1)) & 1u) && (a.inj_col < 0 || (unsigned)a.inj_col == col)) inject<LEG>(acc, j, a.inj_mask);
                }
            }
            __syncwarp();
            unsigned long long f = 0;
#pragma unroll
            for (int j = 0; j < 128; ++j)
                f += (unsigned long long)canon<LEG>(value_bits<LEG>(acc, j)) * (w0 + 2u * (8u * N * ((j >> 1) & 1) + 8u * (j >> 2) + (j & 1)));
            run += f;
        }
    }
    const long long k1 = clock64();
    const unsigned long long t1 = globaltimer_ns();

    unsigned long long efold = 0;
    unsigned mism = compare<LEG, 0>(acc, r0, c0, smid, a, &efold);
    mism += compare<LEG, 1>(acc, r0, c0, smid, a, &efold);
    mism += compare<LEG, 2>(acc, r0, c0, smid, a, &efold);
    mism += compare<LEG, 3>(acc, r0, c0, smid, a, &efold);
    const unsigned fold_bad = run != (unsigned long long)a.iterations * efold ? 1u : 0u;
    publish_cta<CRO_WARPMMA_MAX_SMS>(a, mism, fold_bad, run, s_t0, t1, s_k0, k1, smid, nsmid, s_mism, s_fold_mism, s_fold);
}

template <unsigned LEG>
cudaError_t launch_leg(const WarpMmaArgs& a, int grid, cudaStream_t st) {
    constexpr size_t smem = WLeg<LEG>::kSmem;
    cudaError_t e = cudaFuncSetAttribute(warpmma_kernel<LEG>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    warpmma_kernel<LEG><<<grid, kWarpMmaThreads, smem, st>>>(a);
    return cudaGetLastError();
}

}  // namespace

cudaError_t launch_warpmma(unsigned leg, const WarpMmaArgs& a, int grid, cudaStream_t st) {
    if (grid < 1) return cudaErrorInvalidValue;
    switch (leg) {
        case CRO_WARPMMA_LEG_S8: return launch_leg<CRO_WARPMMA_LEG_S8>(a, grid, st);
        case CRO_WARPMMA_LEG_F16: return launch_leg<CRO_WARPMMA_LEG_F16>(a, grid, st);
        case CRO_WARPMMA_LEG_BF16: return launch_leg<CRO_WARPMMA_LEG_BF16>(a, grid, st);
        case CRO_WARPMMA_LEG_TF32: return launch_leg<CRO_WARPMMA_LEG_TF32>(a, grid, st);
        case CRO_WARPMMA_LEG_F16ACC: return launch_leg<CRO_WARPMMA_LEG_F16ACC>(a, grid, st);
        case CRO_WARPMMA_LEG_MOVE: return launch_leg<CRO_WARPMMA_LEG_MOVE>(a, grid, st);
        default: return cudaErrorInvalidValue;
    }
}

}  // namespace cro
