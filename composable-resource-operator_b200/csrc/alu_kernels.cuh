// alu_kernels.cuh — the ALU probe's shape (cro_probe_alu): each leg's forms and rows, shared by the kernels
// (alu_kernels.cu), which run one instruction form per op on the operands the host's table gives them, and the host
// (alu_probe.cu), which builds that table.  oracle/alu.py restates every form from the PTX ISA.
#pragma once
#include "kernels.cuh"

namespace cro {

struct AluArgs {
    const cro_alu_record* table;        // the leg's records: op * CRO_ALU_THREADS + thread
    cro_alu_cta* cta;                   // grid entries
    cro_alu_thread* thr;                // grid * CRO_ALU_THREADS entries, by block then thread
    cro_alu_fault* rec;                 // CRO_ALU_THREAD_RECORDS per thread entry
    unsigned long long stamp;
    unsigned iterations;
    int inj_sm, inj_warp, inj_lane;     // -1: every SM / warp / lane
    unsigned inj_op, inj_iter, inj_operand;
    unsigned long long inj_mask;        // 0: nothing is injected in this launch (or not in this leg)
};
// Sets the leg's dynamic shared memory request; cudaErrorInvalidConfiguration when the device cannot hold it.
cudaError_t alu_plan(int device, unsigned leg);
cudaError_t launch_alu(unsigned leg, const AluArgs& a, int grid, cudaStream_t);

namespace alu {

// Forms and rows per leg: op = form * rows + row.
constexpr unsigned kForms[CRO_ALU_LEGS] = {269, 19, 50, 25, 45};
constexpr unsigned kRows[CRO_ALU_LEGS] = {2, 4, 4, 4, 8};
constexpr unsigned kOps[CRO_ALU_LEGS] = {CRO_ALU_LOGIC_OPS, CRO_ALU_SHIFT_OPS, CRO_ALU_IADD_OPS, CRO_ALU_IMUL_OPS, CRO_ALU_FLOAT_OPS};
static_assert(kForms[0] * kRows[0] == kOps[0] && kForms[1] * kRows[1] == kOps[1] && kForms[2] * kRows[2] == kOps[2] &&
                  kForms[3] * kRows[3] == kOps[3] && kForms[4] * kRows[4] == kOps[4],
              "ops = forms x rows");

// LOGIC: forms 0 .. 255 lop3.b32 at LUT = form, then:
enum { kBmskClamp = 256, kBmskWrap, kBrev, kPopc32, kPopc64, kBfindU, kBfindS, kBfindShU, kBfindShS, kSzextClampU, kSzextClampS,
       kSzextWrapU, kSzextWrapS };
// SHIFT
enum { kShfLWrap, kShfLClamp, kShfRWrap, kShfRClamp, kShl32, kShrB32, kShrU32, kShrS32, kShl64, kShrB64, kShrU64, kShrS64, kPrmt,
       kPrmtF4e, kPrmtB4e, kPrmtRc8, kPrmtEcl, kPrmtEcr, kPrmtRc16 };
// IADD: carry chains; setp (eq ne lt le gt ge .s32, lo ls hi hs .u32) feeding selp; min / max; the DPX pairs; sad
enum { kAdd64, kAdd128, kSub64, kSub128, kSetp0 = 4, kMinMax0 = 14, kDpx0 = 26, kSadU = 48, kSadS = 49 };
// min / max from kMinMax0: min.u32 max.u32 min.s32 max.s32 min.relu.s32 max.relu.s32 min.u16x2 max.u16x2 min.s16x2
// max.s16x2 min.relu.s16x2 max.relu.s16x2.  DPX from kDpx0: max(max(a,b),c) and min(min(a,b),c) in .s32 .u32
// .relu.s32 .s16x2 .u16x2 .relu.s16x2 (12), then max(a+b,c) and min(a+b,c) in .s32 .u32 .relu.s32 .s16x2 .u16x2 (10).
// IMUL
enum { kMulLoS, kMulLoU, kMulHiS, kMulHiU, kMulWideS, kMulWideU, kMadLo, kMadHiU, kMadHiS, kMadccLoHi, kMadccLoHiS, kMadccHiLo,
       kMulLo64, kDp4a0, kDp2aLo0 = 17, kDp2aHi0 = 21 };
// FLOAT: 0 .. 15 f32 {add, sub, mul, fma} x {rn, rz, rm, rp} (4 op + mode); 16 .. 24 f64 {add, mul, fma} x {rz, rm, rp};
// then min max min.NaN max.NaN min.xorsign.abs max.xorsign.abs .f32; then setp.f32 at eq ne lt le gt ge equ neu ltu
// leu gtu geu num nan.
enum { kF64_0 = 16, kFMin = 25, kFMax, kFMinNaN, kFMaxNaN, kFMinXs, kFMaxXs, kFSetp0 = 31 };

}  // namespace alu
}  // namespace cro
