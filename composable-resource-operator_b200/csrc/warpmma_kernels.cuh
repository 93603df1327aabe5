// warpmma_kernels.cuh — launch wrapper of the warp-MMA probe's kernels (cro_probe_warpmma, warpmma_kernels.cu).  Kept
// out of kernels.cuh so that kernels.cu, whose SASS tests/golden/kernel_sass.json records, does not see it.
#pragma once
#include "kernels.cuh"

namespace cro {

// One launch of leg `leg` (CRO_WARPMMA_LEG_*) runs `grid` CTAs of kWarpMmaThreads, one per SM.  Each CTA generates
// the call's operands (MOVE: the source tile) into its shared memory, computes the answer tile `iterations` times with
// mma.sync from ldmatrix fragments (MOVE: moves the tile through ldmatrix, movmatrix and stmatrix), folds every
// iteration and compares the last one element by element with *expect (the leg's M x N int32 answer, row-major).  It
// publishes one ComputeCta (stamp last written = the call number), ORs its %smid into sm_bits and records its
// mismatching elements while the record buffer has room (*claims counts the slots claimed, possibly past the end).
struct WarpMmaArgs {
    const int* expect;
    ComputeCta* cta;                            // grid entries
    unsigned long long* sm_bits;                // CRO_WARPMMA_MAX_SMS / 64 words
    cro_warpmma_fault* rec;                     // CRO_WARPMMA_RECORDS entries
    unsigned long long* claims;
    unsigned long long seed, stamp;
    unsigned iterations;
    int inj_sm, inj_row, inj_col;               // -1: every SM / row / column
    unsigned inj_iter;
    unsigned long long inj_mask;                // 0: nothing is injected in this launch
    unsigned addr;                              // 0: no fragment-address substitution in this launch
    int addr_sm;                                // -1: every SM
    unsigned addr_iter, addr_row, addr_kstep;
};
constexpr int kWarpMmaThreads = 256;
cudaError_t launch_warpmma(unsigned leg, const WarpMmaArgs& a, int grid, cudaStream_t);

}  // namespace cro
