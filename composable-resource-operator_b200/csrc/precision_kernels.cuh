// precision_kernels.cuh — launch wrapper of the precision probe's kernels (cro_probe_precision, precision_kernels.cu).
// Kept out of kernels.cuh so that kernels.cu, whose SASS tests/golden/kernel_sass.json records, does not see it.
#pragma once
#include "kernels.cuh"

namespace cro {

// One launch of leg `leg` (CRO_PRECISION_LEG_*) runs `grid` CTAs of kPrecisionThreads, one per SM.  Each CTA generates
// the call's operands into its shared memory, computes the answer tile `iterations` times, folds every iteration and
// compares the last one element by element with *expect (the leg's M x N int64 answer, row-major).  It publishes one
// ComputeCta (stamp last written = the call number), ORs its %smid into sm_bits and records its mismatching elements
// while the record buffer has room (*claims counts the slots claimed, possibly past the end).
struct PrecisionArgs {
    const long long* expect;
    ComputeCta* cta;                            // grid entries
    unsigned long long* sm_bits;                // CRO_PRECISION_MAX_SMS / 64 words
    cro_precision_fault* rec;                   // CRO_PRECISION_RECORDS entries
    unsigned long long* claims;
    unsigned long long seed, stamp;
    unsigned iterations;
    int inj_sm, inj_row, inj_col;               // -1: every SM / row / column
    unsigned inj_iter;
    unsigned long long inj_mask;                // 0: nothing is injected in this launch
};
constexpr int kPrecisionThreads = 256;
cudaError_t launch_precision(unsigned leg, const PrecisionArgs& a, int grid, cudaStream_t);

}  // namespace cro
