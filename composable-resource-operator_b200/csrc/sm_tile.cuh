// sm_tile.cuh — what the per-SM arithmetic kernels share (the compute probe's, kernels.cu, and the precision probe's,
// precision_kernels.cu): the PTX helpers, the K-major operand layout and its wgmma descriptor, the wgmma wrappers, the
// injection each thread resolves once, and the CTA epilogue that publishes a ComputeCta.  kernels.cu's sweep kernels
// use the same timer and shared-address helpers.
#pragma once
#include "kernels.cuh"

namespace cro {

__device__ __forceinline__ unsigned long long globaltimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return (uint32_t)__cvta_generic_to_shared(p);
}

// Byte offset of element (row, k) of a K-major operand with K elements of ELEM bytes per row: core matrices of 8 rows
// x 16 bytes (128 contiguous bytes, row r at +16 r), the core matrices along K of one 8-row group side by side
// (leading byte offset 128), 8-row groups 8 * K * ELEM bytes apart (stride byte offset).
template <unsigned ELEM, unsigned K>
__device__ __forceinline__ unsigned kmajor_off(unsigned row, unsigned k) {
    const unsigned kb = k * ELEM;
    return (row >> 3) * (8u * K * ELEM) + (kb >> 4) * 128u + (row & 7u) * 16u + (kb & 15u);
}

// wgmma shared-memory descriptor, no swizzle: start address, leading byte offset 128, stride byte offset sbo.
__device__ __forceinline__ unsigned long long wgmma_desc(unsigned addr, unsigned sbo) {
    return (unsigned long long)((addr & 0x3FFFFu) >> 4) | ((unsigned long long)(128u >> 4) << 16) |
           ((unsigned long long)(sbo >> 4) << 32);
}

// The accumulator operands of a wgmma with 128 or 64 registers per thread: the instruction's register list followed
// by its descriptor and scale-d operands (SM_TILE_ACC*), the index of the scale-d input (SM_TILE_SCALE*), and the
// output bindings d[0 ..] under constraint c (SM_TILE_OUT*).
#define SM_TILE_ACC128                                                                                                   \
    "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "      \
    "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, "  \
    "%47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, "  \
    "%70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, "  \
    "%93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, "    \
    "%113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p"
#define SM_TILE_ACC64                                                                                                    \
    "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "      \
    "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, "  \
    "%47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p"
#define SM_TILE_SCALE128 "%130"
#define SM_TILE_SCALE64 "%66"
#define SM_TILE_D8(c, b) c(d[b]), c(d[b + 1]), c(d[b + 2]), c(d[b + 3]), c(d[b + 4]), c(d[b + 5]), c(d[b + 6]), c(d[b + 7])
#define SM_TILE_D64(c, b) SM_TILE_D8(c, b), SM_TILE_D8(c, b + 8), SM_TILE_D8(c, b + 16), SM_TILE_D8(c, b + 24),           \
                          SM_TILE_D8(c, b + 32), SM_TILE_D8(c, b + 40), SM_TILE_D8(c, b + 48), SM_TILE_D8(c, b + 56)
#define SM_TILE_OUT128(c) SM_TILE_D64(c, 0), SM_TILE_D64(c, 64)
#define SM_TILE_OUT64(c) SM_TILE_D64(c, 0)

// name(d, da, db, scale_d): one wgmma.mma_async `shape` on N accumulators of type Acc bound as c ("+r" or "+f"), scale-d
// off when scale_d is 0.  `tail` is the rest of the instruction after the predicate, leading comma included ("" when it
// takes no scale or transpose immediates).
#define SM_TILE_WGMMA(name, Acc, N, c, shape, tail)                                                                      \
    __device__ __forceinline__ void name(Acc (&d)[N], unsigned long long da, unsigned long long db, int scale_d) {       \
        asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, " SM_TILE_SCALE##N ", 0;\nwgmma.mma_async.sync.aligned." shape     \
                     " " SM_TILE_ACC##N tail ";\n}\n"                                                                   \
                     : SM_TILE_OUT##N(c)                                                                                \
                     : "l"(da), "l"(db), "r"(scale_d));                                                                 \
    }

// The injection of a launch (a.inj_*), resolved once by the thread owning rows r0 and r0 + 8 of SM smid: which of its
// rows it covers (bit 0: r0, bit 1: r0 + 8) and the iteration after which it injects (all ones: none).  `a` is taken by
// value, as the kernel's own parameter is: taken by reference, the resolve compiles to other (branching) code.
struct Injection {
    unsigned rows, iter;
};
template <class Args>
__device__ __forceinline__ Injection resolve_injection(const Args a, unsigned r0, unsigned smid) {
    const unsigned rowsel = (a.inj_row < 0) ? 3u : ((unsigned)a.inj_row == r0 ? 1u : (unsigned)a.inj_row == r0 + 8 ? 2u : 0u);
    return Injection{rowsel, (a.inj_mask && rowsel && (a.inj_sm < 0 || (unsigned)a.inj_sm == smid)) ? a.inj_iter : ~0u};
}

// The end of a per-SM arithmetic kernel, called by every thread: each warp's mismatches (mism per thread) and threads
// whose running fold is wrong (fold_bad) are counted into the CTA's shared tallies and every fold (run) summed; thread
// 0 then ORs the SM's bit into a.sm_bits (SM ids below MAX_SMS) and publishes the CTA's ComputeCta, stamp a.stamp.
template <unsigned MAX_SMS, class Args>
__device__ __forceinline__ void publish_cta(const Args& a, unsigned mism, unsigned fold_bad, unsigned long long run,
                                            unsigned long long t0, unsigned long long t1, long long k0, long long k1,
                                            unsigned smid, unsigned nsmid, unsigned long long& s_mism,
                                            unsigned long long& s_fold_mism, unsigned long long& s_fold) {
    const unsigned wm = __reduce_add_sync(0xffffffffu, mism), wf = __reduce_add_sync(0xffffffffu, fold_bad);
    if ((threadIdx.x & 31u) == 0 && (wm | wf)) {
        atomicAdd(&s_mism, (unsigned long long)wm);
        atomicAdd(&s_fold_mism, (unsigned long long)wf);
    }
    atomicAdd(&s_fold, run);
    __syncthreads();
    if (threadIdx.x == 0) {
        if (smid < MAX_SMS) atomicOr(a.sm_bits + (smid >> 6), 1ull << (smid & 63u));
        ComputeCta& o = a.cta[blockIdx.x];
        o.t0 = t0;
        o.t1 = t1;
        o.cycles = (unsigned long long)(k1 - k0);
        o.mismatches = s_mism;
        o.fold_mismatches = s_fold_mism;
        o.fold = s_fold;
        o.smid = smid;
        o.nsmid = nsmid;
        o.stamp = a.stamp;
    }
}

}  // namespace cro
