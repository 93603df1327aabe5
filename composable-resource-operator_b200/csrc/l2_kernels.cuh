// l2_kernels.cuh — launch wrappers of the L2 probe's kernels (cro_probe_l2, l2_kernels.cu).  Kept out of kernels.cuh
// so that kernels.cu, whose SASS tests/golden/kernel_sass.json records, does not see them.
#pragma once
#include "kernels.cuh"

namespace cro {

constexpr int kL2Threads = 1024;                                   // one 16-byte vector per thread per block
constexpr unsigned kL2BlockWords = CRO_L2_BLOCK_BYTES / 8;
static_assert(CRO_L2_BLOCK_BYTES == 16u * kL2Threads, "a block is one vector per thread");

// What each march CTA publishes per launch (stamp last = the call number; all ones: armed, the CTA did not publish).
struct L2Cta {
    unsigned long long stamp;
    unsigned long long t0, t1;                  // %globaltimer around the CTA's work
    unsigned long long count;                   // compares that failed
    unsigned long long fx, fs, fw;              // M5: fold of the words read, by global word index
    unsigned smid, nsmid;
};
static_assert(sizeof(L2Cta) == 64, "per-CTA record");

struct L2Args {
    ulonglong2* buf;                            // W bytes: blocks * kL2BlockWords words
    L2Cta* cta;                                 // [iteration * 6 + element][G]
    cro_l2_fault* rec;                          // CRO_L2_RECORDS entries
    unsigned long long* claims;
    unsigned long long seed, stamp;
    unsigned blocks, G, delta;
    int inj_sm, inj_element;                    // -1: every SM / every reading element
    unsigned inj_iter;
    long long inj_word;                         // -1: every word
    unsigned long long inj_mask;                // 0: nothing is injected
};
// Element el (0 .. 5) of iteration it: CTA j handles the blocks b with (b + el * delta) mod G == j.
// dyn: the dynamic shared memory l2_plan set, which no launch uses but which keeps two CTAs off one SM.
cudaError_t launch_l2_march(const L2Args& a, unsigned el, unsigned it, size_t dyn, cudaStream_t);
cudaError_t l2_plan(int device, size_t* dyn);
// Discards every 128-byte line of the march's buffer from the L2 (discard.global.L2): the call's last launch.
cudaError_t launch_l2_release(const void* buf, unsigned long long bytes, int grid, cudaStream_t);

struct L2AtomicArgs {
    unsigned long long *a1_sum, *a1_xor;        // a1 counters each
    unsigned* a2_ctr;                           // a2 counters, 32 words (128 bytes) apart
    unsigned* tickets;                          // [a2 counter][32 * G]
    unsigned char* present;                     // [a2 counter][32 * G], zeroed by the host
    unsigned char *a1_bad, *a2_bad;             // per counter: 1 when it failed (plain stores)
    unsigned long long* a1_partial;             // per A1 checker CTA: failed counters (armed all ones by the host)
    unsigned long long* a2_partial;             // per A2 checker CTA: {holes, failed counters}
    unsigned long long seed;
    unsigned a1, a2, G;
    int inj_leg;
    unsigned long long inj_counter, inj_mask;
};
// A1's kernel (G CTAs of red.add / red.xor) and A2's (G CTAs of atom.add tickets), and their checkers, which use no
// atomic: one thread per A1 counter, one warp per A2 counter.
cudaError_t launch_l2_a1(const L2AtomicArgs& a, cudaStream_t);
cudaError_t launch_l2_a1_check(const L2AtomicArgs& a, cudaStream_t);
cudaError_t launch_l2_a2(const L2AtomicArgs& a, cudaStream_t);
cudaError_t launch_l2_a2_check(const L2AtomicArgs& a, cudaStream_t);
inline unsigned l2_a1_check_ctas(unsigned a1) { return (a1 + kL2Threads - 1) / kL2Threads; }
inline unsigned l2_a2_check_ctas(unsigned a2) { return (a2 + kL2Threads / 32 - 1) / (kL2Threads / 32); }

}  // namespace cro
