// alu_kernels.cu — the ALU probe's kernels (cro_probe_alu): one instantiation and one launch per leg, one CTA of 8
// warps per SM.  The device computes no operand and no expected value: each thread loads its record of the host's
// table, runs exactly one instruction form on it in asm volatile and compares the result with the loaded one.  Every
// form has its own loop over its rows, so each form's instruction sits once in the iteration loop, where
// tests/test_alu_abi.py finds it in the SASS.  The report path is lane_tally.cuh.
#include <utility>

#include "alu_kernels.cuh"
#include "lane_tally.cuh"

namespace cro {

namespace {

typedef unsigned long long u64;
constexpr unsigned kT = CRO_ALU_THREADS;
// More than half of an SM's shared memory, so no second CTA of any kernel shares the SM.
constexpr size_t kSmemBytes = 160u << 10;

struct Tally : LaneCounts<cro_alu_fault, CRO_ALU_THREAD_RECORDS> {
    unsigned leg, smid, warp, lane;
};

__device__ __forceinline__ unsigned lo(u64 x) { return (unsigned)x; }
__device__ __forceinline__ float f32(u64 x) { return __uint_as_float((unsigned)x); }
__device__ __forceinline__ double f64(u64 x) { return __longlong_as_double((long long)x); }
__device__ __forceinline__ u64 bits(float x) { return __float_as_uint(x); }
__device__ __forceinline__ u64 bits(double x) { return (u64)__double_as_longlong(x); }

#define A1(ins) asm volatile(ins " %0, %1;" : "=r"(d) : "r"(a))
#define A2(ins) asm volatile(ins " %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b))
#define A3(ins) asm volatile(ins " %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c))
#define S64(ins) asm volatile(ins " %0, %1, %2;" : "=l"(q) : "l"(x[0]), "r"(b))
#define SETP(cmp) asm volatile("{ .reg .pred p; setp." cmp " p, %1, %2; selp.b32 %0, %3, %4, p; }" : "=r"(d) : "r"(a), "r"(b), "r"(c), "r"(e))
#define PAIR(first, second) asm volatile("{ .reg .b32 t; " first " t, %1, %2; " second " %0, t, %3; }" : "=r"(d) : "r"(a), "r"(b), "r"(c))

// ---- LOGIC ----
template <unsigned F>
__device__ __forceinline__ void form_logic(const u64 (&x)[4], u64 (&g)[3]) {
    const unsigned a = lo(x[0]), b = lo(x[1]), c = lo(x[2]);
    unsigned d = 0;
    if constexpr (F < 256) asm volatile("lop3.b32 %0, %1, %2, %3, %4;" : "=r"(d) : "r"(a), "r"(b), "r"(c), "n"(F));
    else if constexpr (F == alu::kBmskClamp) A2("bmsk.clamp.b32");
    else if constexpr (F == alu::kBmskWrap) A2("bmsk.wrap.b32");
    else if constexpr (F == alu::kBrev) A1("brev.b32");
    else if constexpr (F == alu::kPopc32) A1("popc.b32");
    else if constexpr (F == alu::kPopc64) asm volatile("popc.b64 %0, %1;" : "=r"(d) : "l"(x[0]));
    else if constexpr (F == alu::kBfindU) A1("bfind.u32");
    else if constexpr (F == alu::kBfindS) A1("bfind.s32");
    else if constexpr (F == alu::kBfindShU) A1("bfind.shiftamt.u32");
    else if constexpr (F == alu::kBfindShS) A1("bfind.shiftamt.s32");
    else if constexpr (F == alu::kSzextClampU) A2("szext.clamp.u32");
    else if constexpr (F == alu::kSzextClampS) A2("szext.clamp.s32");
    else if constexpr (F == alu::kSzextWrapU) A2("szext.wrap.u32");
    else A2("szext.wrap.s32");
    g[0] = d;
}

// ---- SHIFT ----
template <unsigned F>
__device__ __forceinline__ void form_shift(const u64 (&x)[4], u64 (&g)[3]) {
    using namespace alu;
    const unsigned a = lo(x[0]), b = lo(x[1]), c = lo(x[2]);
    unsigned d = 0;
    u64 q = 0;
    if constexpr (F == kShfLWrap) A3("shf.l.wrap.b32");
    else if constexpr (F == kShfLClamp) A3("shf.l.clamp.b32");
    else if constexpr (F == kShfRWrap) A3("shf.r.wrap.b32");
    else if constexpr (F == kShfRClamp) A3("shf.r.clamp.b32");
    else if constexpr (F == kShl32) A2("shl.b32");
    else if constexpr (F == kShrB32) A2("shr.b32");
    else if constexpr (F == kShrU32) A2("shr.u32");
    else if constexpr (F == kShrS32) A2("shr.s32");
    else if constexpr (F == kShl64) S64("shl.b64");
    else if constexpr (F == kShrB64) S64("shr.b64");
    else if constexpr (F == kShrU64) S64("shr.u64");
    else if constexpr (F == kShrS64) S64("shr.s64");
    else if constexpr (F == kPrmt) A3("prmt.b32");
    else if constexpr (F == kPrmtF4e) A3("prmt.b32.f4e");
    else if constexpr (F == kPrmtB4e) A3("prmt.b32.b4e");
    else if constexpr (F == kPrmtRc8) A3("prmt.b32.rc8");
    else if constexpr (F == kPrmtEcl) A3("prmt.b32.ecl");
    else if constexpr (F == kPrmtEcr) A3("prmt.b32.ecr");
    else A3("prmt.b32.rc16");
    g[0] = (F >= kShl64 && F <= kShrS64) ? q : (u64)d;
}

// ---- IADD ----
template <unsigned F>
__device__ __forceinline__ void form_iadd(const u64 (&x)[4], u64 (&g)[3]) {
    using namespace alu;
    const unsigned a = lo(x[0]), b = lo(x[1]), c = lo(x[2]), e = lo(x[3]);
    unsigned d = 0;
    if constexpr (F == kAdd64 || F == kSub64) {
        unsigned r0, r1, r2;
        if constexpr (F == kAdd64)
            asm volatile("add.cc.u32 %0, %3, %5; addc.cc.u32 %1, %4, %6; addc.u32 %2, 0, 0;"
                         : "=r"(r0), "=r"(r1), "=r"(r2) : "r"(lo(x[0])), "r"(lo(x[0] >> 32)), "r"(lo(x[1])), "r"(lo(x[1] >> 32)));
        else
            asm volatile("sub.cc.u32 %0, %3, %5; subc.cc.u32 %1, %4, %6; subc.u32 %2, 0, 0;"
                         : "=r"(r0), "=r"(r1), "=r"(r2) : "r"(lo(x[0])), "r"(lo(x[0] >> 32)), "r"(lo(x[1])), "r"(lo(x[1] >> 32)));
        g[0] = ((u64)r1 << 32) | r0;
        g[1] = r2;
        return;
    } else if constexpr (F == kAdd128 || F == kSub128) {
        unsigned r[5];
        if constexpr (F == kAdd128)
            asm volatile("add.cc.u32 %0, %5, %9; addc.cc.u32 %1, %6, %10; addc.cc.u32 %2, %7, %11; addc.cc.u32 %3, %8, %12; addc.u32 %4, 0, 0;"
                         : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]), "=r"(r[4])
                         : "r"(lo(x[0])), "r"(lo(x[0] >> 32)), "r"(lo(x[1])), "r"(lo(x[1] >> 32)), "r"(lo(x[2])), "r"(lo(x[2] >> 32)),
                           "r"(lo(x[3])), "r"(lo(x[3] >> 32)));
        else
            asm volatile("sub.cc.u32 %0, %5, %9; subc.cc.u32 %1, %6, %10; subc.cc.u32 %2, %7, %11; subc.cc.u32 %3, %8, %12; subc.u32 %4, 0, 0;"
                         : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]), "=r"(r[4])
                         : "r"(lo(x[0])), "r"(lo(x[0] >> 32)), "r"(lo(x[1])), "r"(lo(x[1] >> 32)), "r"(lo(x[2])), "r"(lo(x[2] >> 32)),
                           "r"(lo(x[3])), "r"(lo(x[3] >> 32)));
        g[0] = ((u64)r[1] << 32) | r[0];
        g[1] = ((u64)r[3] << 32) | r[2];
        g[2] = r[4];
        return;
    } else if constexpr (F == kSetp0 + 0) SETP("eq.s32");
    else if constexpr (F == kSetp0 + 1) SETP("ne.s32");
    else if constexpr (F == kSetp0 + 2) SETP("lt.s32");
    else if constexpr (F == kSetp0 + 3) SETP("le.s32");
    else if constexpr (F == kSetp0 + 4) SETP("gt.s32");
    else if constexpr (F == kSetp0 + 5) SETP("ge.s32");
    else if constexpr (F == kSetp0 + 6) SETP("lo.u32");
    else if constexpr (F == kSetp0 + 7) SETP("ls.u32");
    else if constexpr (F == kSetp0 + 8) SETP("hi.u32");
    else if constexpr (F == kSetp0 + 9) SETP("hs.u32");
    else if constexpr (F == kMinMax0 + 0) A2("min.u32");
    else if constexpr (F == kMinMax0 + 1) A2("max.u32");
    else if constexpr (F == kMinMax0 + 2) A2("min.s32");
    else if constexpr (F == kMinMax0 + 3) A2("max.s32");
    else if constexpr (F == kMinMax0 + 4) A2("min.relu.s32");
    else if constexpr (F == kMinMax0 + 5) A2("max.relu.s32");
    else if constexpr (F == kMinMax0 + 6) A2("min.u16x2");
    else if constexpr (F == kMinMax0 + 7) A2("max.u16x2");
    else if constexpr (F == kMinMax0 + 8) A2("min.s16x2");
    else if constexpr (F == kMinMax0 + 9) A2("max.s16x2");
    else if constexpr (F == kMinMax0 + 10) A2("min.relu.s16x2");
    else if constexpr (F == kMinMax0 + 11) A2("max.relu.s16x2");
    else if constexpr (F == kDpx0 + 0) PAIR("max.s32", "max.s32");
    else if constexpr (F == kDpx0 + 1) PAIR("min.s32", "min.s32");
    else if constexpr (F == kDpx0 + 2) PAIR("max.u32", "max.u32");
    else if constexpr (F == kDpx0 + 3) PAIR("min.u32", "min.u32");
    else if constexpr (F == kDpx0 + 4) PAIR("max.s32", "max.relu.s32");
    else if constexpr (F == kDpx0 + 5) PAIR("min.s32", "min.relu.s32");
    else if constexpr (F == kDpx0 + 6) PAIR("max.s16x2", "max.s16x2");
    else if constexpr (F == kDpx0 + 7) PAIR("min.s16x2", "min.s16x2");
    else if constexpr (F == kDpx0 + 8) PAIR("max.u16x2", "max.u16x2");
    else if constexpr (F == kDpx0 + 9) PAIR("min.u16x2", "min.u16x2");
    else if constexpr (F == kDpx0 + 10) PAIR("max.s16x2", "max.relu.s16x2");
    else if constexpr (F == kDpx0 + 11) PAIR("min.s16x2", "min.relu.s16x2");
    else if constexpr (F == kDpx0 + 12) PAIR("add.s32", "max.s32");
    else if constexpr (F == kDpx0 + 13) PAIR("add.s32", "min.s32");
    else if constexpr (F == kDpx0 + 14) PAIR("add.u32", "max.u32");
    else if constexpr (F == kDpx0 + 15) PAIR("add.u32", "min.u32");
    else if constexpr (F == kDpx0 + 16) PAIR("add.s32", "max.relu.s32");
    else if constexpr (F == kDpx0 + 17) PAIR("add.s32", "min.relu.s32");
    else if constexpr (F == kDpx0 + 18) PAIR("add.s16x2", "max.s16x2");
    else if constexpr (F == kDpx0 + 19) PAIR("add.s16x2", "min.s16x2");
    else if constexpr (F == kDpx0 + 20) PAIR("add.u16x2", "max.u16x2");
    else if constexpr (F == kDpx0 + 21) PAIR("add.u16x2", "min.u16x2");
    else if constexpr (F == kSadU) A3("sad.u32");
    else A3("sad.s32");
    g[0] = d;
}

// ---- IMUL ----
template <unsigned F>
__device__ __forceinline__ void form_imul(const u64 (&x)[4], u64 (&g)[3]) {
    using namespace alu;
    const unsigned a = lo(x[0]), b = lo(x[1]), c = lo(x[2]), e = lo(x[3]);
    unsigned d = 0;
    u64 q = 0;
    if constexpr (F == kMulLoS) A2("mul.lo.s32");
    else if constexpr (F == kMulLoU) A2("mul.lo.u32");
    else if constexpr (F == kMulHiS) A2("mul.hi.s32");
    else if constexpr (F == kMulHiU) A2("mul.hi.u32");
    else if constexpr (F == kMulWideS) asm volatile("mul.wide.s32 %0, %1, %2;" : "=l"(q) : "r"(a), "r"(b));
    else if constexpr (F == kMulWideU) asm volatile("mul.wide.u32 %0, %1, %2;" : "=l"(q) : "r"(a), "r"(b));
    else if constexpr (F == kMadLo) A3("mad.lo.u32");
    else if constexpr (F == kMadHiU) A3("mad.hi.u32");
    else if constexpr (F == kMadHiS) A3("mad.hi.s32");
    else if constexpr (F == kMadccLoHi) {
        unsigned r0, r1, r2;
        asm volatile("mad.lo.cc.u32 %0, %3, %4, %5; madc.hi.cc.u32 %1, %3, %4, %6; addc.u32 %2, 0, 0;"
                     : "=r"(r0), "=r"(r1), "=r"(r2) : "r"(a), "r"(b), "r"(c), "r"(e));
        g[0] = ((u64)r1 << 32) | r0;
        g[1] = r2;
        return;
    } else if constexpr (F == kMadccLoHiS) {
        unsigned r0, r1;
        asm volatile("mad.lo.cc.u32 %0, %2, %3, %4; madc.hi.s32 %1, %2, %3, %5;" : "=r"(r0), "=r"(r1) : "r"(a), "r"(b), "r"(c), "r"(e));
        q = ((u64)r1 << 32) | r0;
    } else if constexpr (F == kMadccHiLo) {
        unsigned r0, r1;
        asm volatile("mad.hi.cc.u32 %0, %2, %3, %4; madc.lo.u32 %1, %2, %3, %5;" : "=r"(r0), "=r"(r1) : "r"(a), "r"(b), "r"(c), "r"(e));
        q = ((u64)r1 << 32) | r0;
    } else if constexpr (F == kMulLo64) asm volatile("mul.lo.u64 %0, %1, %2;" : "=l"(q) : "l"(x[0]), "l"(x[1]));
    else if constexpr (F == kDp4a0 + 0) A3("dp4a.u32.u32");
    else if constexpr (F == kDp4a0 + 1) A3("dp4a.u32.s32");
    else if constexpr (F == kDp4a0 + 2) A3("dp4a.s32.u32");
    else if constexpr (F == kDp4a0 + 3) A3("dp4a.s32.s32");
    else if constexpr (F == kDp2aLo0 + 0) A3("dp2a.lo.u32.u32");
    else if constexpr (F == kDp2aLo0 + 1) A3("dp2a.lo.u32.s32");
    else if constexpr (F == kDp2aLo0 + 2) A3("dp2a.lo.s32.u32");
    else if constexpr (F == kDp2aLo0 + 3) A3("dp2a.lo.s32.s32");
    else if constexpr (F == kDp2aHi0 + 0) A3("dp2a.hi.u32.u32");
    else if constexpr (F == kDp2aHi0 + 1) A3("dp2a.hi.u32.s32");
    else if constexpr (F == kDp2aHi0 + 2) A3("dp2a.hi.s32.u32");
    else A3("dp2a.hi.s32.s32");
    constexpr bool wide = F == kMulWideS || F == kMulWideU || F == kMadccLoHiS || F == kMadccHiLo || F == kMulLo64;
    g[0] = wide ? q : (u64)d;
}

// ---- FLOAT ----
#define F2(ins) asm volatile(ins " %0, %1, %2;" : "=f"(r) : "f"(fa), "f"(fb))
#define F3(ins) asm volatile(ins " %0, %1, %2, %3;" : "=f"(r) : "f"(fa), "f"(fb), "f"(fc))
#define D2(ins) asm volatile(ins " %0, %1, %2;" : "=d"(s) : "d"(da), "d"(db))
#define D3(ins) asm volatile(ins " %0, %1, %2, %3;" : "=d"(s) : "d"(da), "d"(db), "d"(dc))
#define FSETP(cmp) asm volatile("{ .reg .pred p; setp." cmp ".f32 p, %1, %2; selp.u32 %0, 1, 0, p; }" : "=r"(d) : "f"(fa), "f"(fb))

template <unsigned F>
__device__ __forceinline__ void form_float(const u64 (&x)[4], u64 (&g)[3]) {
    using namespace alu;
    const float fa = f32(x[0]), fb = f32(x[1]), fc = f32(x[2]);
    const double da = f64(x[0]), db = f64(x[1]), dc = f64(x[2]);
    float r = 0.f;
    double s = 0.;
    unsigned d = 0;
    if constexpr (F == 0) F2("add.rn.f32");
    else if constexpr (F == 1) F2("add.rz.f32");
    else if constexpr (F == 2) F2("add.rm.f32");
    else if constexpr (F == 3) F2("add.rp.f32");
    else if constexpr (F == 4) F2("sub.rn.f32");
    else if constexpr (F == 5) F2("sub.rz.f32");
    else if constexpr (F == 6) F2("sub.rm.f32");
    else if constexpr (F == 7) F2("sub.rp.f32");
    else if constexpr (F == 8) F2("mul.rn.f32");
    else if constexpr (F == 9) F2("mul.rz.f32");
    else if constexpr (F == 10) F2("mul.rm.f32");
    else if constexpr (F == 11) F2("mul.rp.f32");
    else if constexpr (F == 12) F3("fma.rn.f32");
    else if constexpr (F == 13) F3("fma.rz.f32");
    else if constexpr (F == 14) F3("fma.rm.f32");
    else if constexpr (F == 15) F3("fma.rp.f32");
    else if constexpr (F == 16) D2("add.rz.f64");
    else if constexpr (F == 17) D2("add.rm.f64");
    else if constexpr (F == 18) D2("add.rp.f64");
    else if constexpr (F == 19) D2("mul.rz.f64");
    else if constexpr (F == 20) D2("mul.rm.f64");
    else if constexpr (F == 21) D2("mul.rp.f64");
    else if constexpr (F == 22) D3("fma.rz.f64");
    else if constexpr (F == 23) D3("fma.rm.f64");
    else if constexpr (F == 24) D3("fma.rp.f64");
    else if constexpr (F == kFMin) F2("min.f32");
    else if constexpr (F == kFMax) F2("max.f32");
    else if constexpr (F == kFMinNaN) F2("min.NaN.f32");
    else if constexpr (F == kFMaxNaN) F2("max.NaN.f32");
    else if constexpr (F == kFMinXs) F2("min.xorsign.abs.f32");
    else if constexpr (F == kFMaxXs) F2("max.xorsign.abs.f32");
    else if constexpr (F == kFSetp0 + 0) FSETP("eq");
    else if constexpr (F == kFSetp0 + 1) FSETP("ne");
    else if constexpr (F == kFSetp0 + 2) FSETP("lt");
    else if constexpr (F == kFSetp0 + 3) FSETP("le");
    else if constexpr (F == kFSetp0 + 4) FSETP("gt");
    else if constexpr (F == kFSetp0 + 5) FSETP("ge");
    else if constexpr (F == kFSetp0 + 6) FSETP("equ");
    else if constexpr (F == kFSetp0 + 7) FSETP("neu");
    else if constexpr (F == kFSetp0 + 8) FSETP("ltu");
    else if constexpr (F == kFSetp0 + 9) FSETP("leu");
    else if constexpr (F == kFSetp0 + 10) FSETP("gtu");
    else if constexpr (F == kFSetp0 + 11) FSETP("geu");
    else if constexpr (F == kFSetp0 + 12) FSETP("num");
    else FSETP("nan");
    g[0] = F >= kF64_0 && F < kFMin ? bits(s) : F >= kFSetp0 ? (u64)d : bits(r);
}

template <unsigned LEG, unsigned F>
__device__ __forceinline__ void form(const u64 (&x)[4], u64 (&g)[3]) {
    if constexpr (LEG == CRO_ALU_LEG_LOGIC) form_logic<F>(x, g);
    if constexpr (LEG == CRO_ALU_LEG_SHIFT) form_shift<F>(x, g);
    if constexpr (LEG == CRO_ALU_LEG_IADD) form_iadd<F>(x, g);
    if constexpr (LEG == CRO_ALU_LEG_IMUL) form_imul<F>(x, g);
    if constexpr (LEG == CRO_ALU_LEG_FLOAT) form_float<F>(x, g);
}

// What one iteration needs beyond the tally: the thread's first record, the op injected in this iteration (~0u: none)
// and the mask per operand word.
struct Iter {
    const cro_alu_record* p;
    unsigned it, inj_op;
    bool lastit;
    u64 m[4];
};

// Every row of form F: load, run, compare.
template <unsigned LEG, unsigned F>
__device__ __forceinline__ void rows(Tally& T, const Iter& I) {
    constexpr unsigned R = alu::kRows[LEG];
#pragma unroll 1
    for (unsigned row = 0; row < R; ++row) {
        const unsigned op = F * R + row;
        const cro_alu_record* p = I.p + (size_t)op * kT;
        const ulonglong2 i01 = __ldg(reinterpret_cast<const ulonglong2*>(p->in));
        const ulonglong2 i23 = __ldg(reinterpret_cast<const ulonglong2*>(p->in + 2));
        const ulonglong2 o01 = __ldg(reinterpret_cast<const ulonglong2*>(p->out));
        const u64 o2 = __ldg(p->out + 2);
        u64 x[4] = {i01.x, i01.y, i23.x, i23.y};
        if (op == I.inj_op) {
            x[0] ^= I.m[0];
            x[1] ^= I.m[1];
            x[2] ^= I.m[2];
            x[3] ^= I.m[3];
        }
        u64 g[3] = {0, 0, 0};
        form<LEG, F>(x, g);
        if ((g[0] != o01.x) | (g[1] != o01.y) | (g[2] != o2))
            T.miss(I.lastit, [&] {
                return cro_alu_fault{T.leg, op, I.it, T.smid, T.warp, T.lane, {0u, 0u}, {i01.x, i01.y, i23.x, i23.y}, {o01.x, o01.y, o2},
                                     {g[0], g[1], g[2]}};
            });
        if (I.lastit) T.fold(op, g[0] + 2 * g[1] + 4 * g[2]);
    }
}

template <unsigned LEG, size_t... F>
__device__ __forceinline__ void every_form(Tally& T, const Iter& I, std::index_sequence<F...>) {
    (rows<LEG, (unsigned)F>(T, I), ...);
}

template <unsigned LEG>
__global__ void __launch_bounds__(kT, 1) alu_kernel(const AluArgs a) {
    unsigned smid, nsmid;
    asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
    asm volatile("mov.u32 %0, %%nsmid;" : "=r"(nsmid));
    const unsigned t = threadIdx.x, w = t >> 5, l = t & 31u;
    const size_t me = (size_t)blockIdx.x * kT + t;
    const bool inj = a.inj_mask && (a.inj_sm < 0 || (unsigned)a.inj_sm == smid) && (a.inj_warp < 0 || (unsigned)a.inj_warp == w) &&
                     (a.inj_lane < 0 || (unsigned)a.inj_lane == l);
    Tally T;
    T.rec = a.rec + me * CRO_ALU_THREAD_RECORDS;
    T.leg = LEG;
    T.smid = smid;
    T.warp = w;
    T.lane = l;
    Iter I;
    I.p = a.table + t;
    for (unsigned k = 0; k < 4; ++k) I.m[k] = a.inj_operand == k ? a.inj_mask : 0ull;
    const unsigned long long t0 = lane_timer_ns();
    const long long k0 = clock64();
#pragma unroll 1
    for (unsigned it = 0; it < a.iterations; ++it) {
        I.it = it;
        I.lastit = it + 1 == a.iterations;
        I.inj_op = inj && it == a.inj_iter ? a.inj_op : ~0u;
        every_form<LEG>(T, I, std::make_index_sequence<alu::kForms[LEG]>{});
    }
    const long long k1 = clock64();
    const unsigned long long t1 = lane_timer_ns();
    T.publish(a.thr[me], a.cta, a.stamp, t0, t1, k0, k1, smid, nsmid);
}

template <unsigned LEG>
cudaError_t plan_leg() {
    return cudaFuncSetAttribute(alu_kernel<LEG>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBytes);
}

}  // namespace

cudaError_t alu_plan(int device, unsigned leg) {
    int optin = 0;
    cudaError_t e = cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device);
    if (e) return e;
    if ((size_t)optin < kSmemBytes) return cudaErrorInvalidConfiguration;
    switch (leg) {
        case CRO_ALU_LEG_LOGIC: return plan_leg<CRO_ALU_LEG_LOGIC>();
        case CRO_ALU_LEG_SHIFT: return plan_leg<CRO_ALU_LEG_SHIFT>();
        case CRO_ALU_LEG_IADD: return plan_leg<CRO_ALU_LEG_IADD>();
        case CRO_ALU_LEG_IMUL: return plan_leg<CRO_ALU_LEG_IMUL>();
        default: return plan_leg<CRO_ALU_LEG_FLOAT>();
    }
}

cudaError_t launch_alu(unsigned leg, const AluArgs& a, int grid, cudaStream_t st) {
    switch (leg) {
        case CRO_ALU_LEG_LOGIC: alu_kernel<CRO_ALU_LEG_LOGIC><<<grid, kT, kSmemBytes, st>>>(a); break;
        case CRO_ALU_LEG_SHIFT: alu_kernel<CRO_ALU_LEG_SHIFT><<<grid, kT, kSmemBytes, st>>>(a); break;
        case CRO_ALU_LEG_IADD: alu_kernel<CRO_ALU_LEG_IADD><<<grid, kT, kSmemBytes, st>>>(a); break;
        case CRO_ALU_LEG_IMUL: alu_kernel<CRO_ALU_LEG_IMUL><<<grid, kT, kSmemBytes, st>>>(a); break;
        default: alu_kernel<CRO_ALU_LEG_FLOAT><<<grid, kT, kSmemBytes, st>>>(a); break;
    }
    return cudaGetLastError();
}

}  // namespace cro
