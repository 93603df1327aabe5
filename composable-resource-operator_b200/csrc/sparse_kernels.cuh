// sparse_kernels.cuh — launch wrapper of the sparse probe's kernels (cro_probe_sparse, sparse_kernels.cu).  Kept out of
// kernels.cuh so that kernels.cu, whose SASS tests/golden/kernel_sass.json records, does not see it.
#pragma once
#include "kernels.cuh"

namespace cro {

// One launch of leg `leg` (CRO_SPARSE_LEG_*) runs `grid` CTAs of kSparseThreads, one per SM.  Each CTA generates the
// call's compressed A, B and metadata into its shared memory and registers, computes the answer tile `iterations`
// times with wgmma.mma_async.sp, folds every iteration and compares the last one element by element with *expect (the
// leg's M x N int32 answer, row-major).  It publishes one ComputeCta (stamp last written = the call number), ORs its
// %smid into sm_bits and records its mismatching elements while the record buffer has room (*claims counts the slots
// claimed, possibly past the end).
struct SparseArgs {
    const int* expect;
    ComputeCta* cta;                            // grid entries
    unsigned long long* sm_bits;                // CRO_SPARSE_MAX_SMS / 64 words
    cro_sparse_fault* rec;                      // CRO_SPARSE_RECORDS entries
    unsigned long long* claims;
    unsigned long long seed, stamp;
    unsigned iterations;
    int inj_sm, inj_row, inj_col;               // -1: every SM / row / column
    unsigned inj_iter;
    unsigned long long inj_mask;                // 0: nothing is injected in this launch
    unsigned meta;                              // 0: no metadata substitution in this launch
    int meta_sm;                                // -1: every SM
    unsigned meta_iter, meta_row, meta_group;
};
constexpr int kSparseThreads = 256;
cudaError_t launch_sparse(unsigned leg, const SparseArgs& a, int grid, cudaStream_t);

}  // namespace cro
