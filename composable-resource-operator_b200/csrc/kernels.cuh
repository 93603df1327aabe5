// kernels.cuh — launch wrappers for the sm_90a probe kernels.
//
// No reference counterpart: the reference's post-attach check is a UUID string
// match (internal/utils/gpus.go:54-86); these kernels are the strong check that
// takes its slot (SURVEY.md §2b).  All arithmetic is 64-bit integer; results
// are bit-exact against the CPU restatement the tests hold (see tests/).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include <string>

#include "../../include/croprobe.h"
#include "env.hpp"

namespace cro {

// Per-sweep result slot in device memory, written by the last CTA to finish.
// The checksum of a sweep over words w[0..n) is the triple
//   x = XOR of all words,  s = wrapping sum,  w = wrapping sum of w[i] * (2i + 1)
// (the third component makes the position of every word matter: swapped or
// misplaced tiles change it, which XOR and sum alone cannot see).
struct SweepOut {
    unsigned long long x;
    unsigned long long s;
    unsigned long long w;
    unsigned long long t0;      // min %globaltimer at CTA start (ns)
    unsigned long long t1;      // max %globaltimer at CTA end   (ns)
    unsigned long long stamp;   // nonce of the probe whose kernel wrote the slot (a stale slot is a failure)
    unsigned long long n_words; // words the sweep covered
    unsigned long long mismatches;  // a comparing read: words that differ from the pattern (exact); 0 from a read that
                                    // only folds; not written by the fill, the copies and the closed form
};
static_assert(sizeof(SweepOut) == 64 && sizeof(SweepOut) == sizeof(cro_sweep_slot), "SweepOut is one 64-byte slot");
static_assert(offsetof(SweepOut, t0) == offsetof(cro_sweep_slot, t0) && offsetof(SweepOut, stamp) == offsetof(cro_sweep_slot, stamp) &&
                  offsetof(SweepOut, n_words) == offsetof(cro_sweep_slot, n_words) &&
                  offsetof(SweepOut, mismatches) == offsetof(cro_sweep_slot, mismatches),
              "SweepOut is the cro_sweep_slot of include/croprobe.h");

// What a probe's kernels read from device memory instead of taking as launch
// parameters, so that ONE captured CUDA graph serves every probe: the host
// refreshes these 16 bytes (a memcpy node at the head of the graph).
struct ProbeParams {
    unsigned long long seed;    // effective pattern seed of this probe (device seed + nonce * kNonceStride)
    unsigned long long nonce;   // probe number on this device, starts at 0
};
constexpr unsigned long long kNonceStride = 0xD1B54A32D192ED03ull;   // odd: distinct nonces give distinct seeds

// Scratch a kernel needs for its reduction.  Kernels that may run CONCURRENTLY
// on one device (main stream vs the closed-form generator on the side stream)
// each own one.
struct SweepScratch {
    ulonglong4*  partials;     // one (xor, sum, wsum, -) per CTA, >= max grid
    unsigned int* counter;     // self-resetting "CTAs done" ticket
    unsigned long long* tmin;  // per-sweep timers, reset by the last CTA
    unsigned long long* tmax;
    unsigned long long* tile_ctr;  // dynamic tile counter of the TMA kernels, reset by the last CTA
};

struct LaunchCfg {
    int grid;
    int block;
    size_t smem;
};

// Pattern word i of a region: splitmix64 step of state (seed + i).
__host__ __device__ __forceinline__ unsigned long long pattern_word(unsigned long long seed,
                                                                     unsigned long long i) {
    unsigned long long z = seed + i + 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

enum : unsigned { READ_LDG = 1, READ_TMA = 2, READ_LDG256 = 3, COPY_LDG = 1, COPY_TMA = 2, COPY_TMA_FUSED = 3 };

// One-time per-device setup (smem carve-outs, occupancy → persistent grid size).
struct KernelPlan {
    LaunchCfg fill, read_ldg, read_ldg256, read_tma, copy_ldg, copy_tma, copy_fused, expect, locate;
    int link_grid;                 // default grid of the host link probe's SM legs
    int sm_count;
    // tuning knobs, from the owning context's validated snapshot (see env.hpp)
    unsigned read_tile, read_stages, read_chunk, read_dyn;
    unsigned copy_tile, copy_stages, copy_chunk, copy_dyn;
    unsigned fused_tile, fused_stages, fused_chunk, fused_threads;
};
// A ring (tile * stages) that does not fit the device next to the kernel's static shared memory, or that leaves no
// room for one CTA per SM, is refused: *why gets the knob's refusal sentence and the call returns cudaErrorInvalidValue.
cudaError_t plan_kernels(int device, const env::Values& knobs, KernelPlan* plan, std::string* why);

// Seed and stamp of a launch: `pp` (device pointer) when non-null — the captured graph's kernels read the 16 bytes
// the host refreshed — else the immediate `imm`.
struct Params {
    ProbeParams imm;
    const ProbeParams* pp;
};
// invert: write the bitwise complement of the pattern (the fault locator's second retest pass; the probe never does).
cudaError_t launch_fill(const KernelPlan&, void* base, uint64_t bytes, const Params&,
                        const SweepScratch&, SweepOut* out, cudaStream_t, bool invert = false);
// compare: every word is also compared with pattern_word(seed, i), i counted from `base`, and out->mismatches gets the
// exact count of words that differ (the probe's reads: a fold alone misses multi-word faults that cancel in it, see
// DESIGN.md §3).  Without it the read only folds and writes 0 there (a peer's pattern, the single timed sweeps).
cudaError_t launch_read(const KernelPlan&, unsigned variant, const void* base, uint64_t bytes,
                        const Params&, const SweepScratch&, SweepOut* out, cudaStream_t, bool compare);
// Every variant publishes *out when out is non-null: the %globaltimer window, the stamp and n_words = bytes / 8.
// COPY_TMA_FUSED also folds every tile it moves (checksum of the SOURCE stream as read) into it and needs out; the
// plain variants fold nothing and write a zero checksum, like the fill.
cudaError_t launch_copy(const KernelPlan&, unsigned variant, void* dst, const void* src, uint64_t bytes,
                        const Params&, const SweepScratch&, SweepOut* out, cudaStream_t);
cudaError_t launch_expected(const KernelPlan&, uint64_t bytes, const Params&,
                            const SweepScratch&, SweepOut* out, cudaStream_t);
// word ^= mask for the words [first, first + count) of base: the test hooks' software faults.
cudaError_t launch_xor_words(void* base, uint64_t first, uint64_t count, uint64_t mask, cudaStream_t);

// Fault locator (cro_locate_faults).  One compare pass over one half: every word is checked against
// pattern_word(seed, i) ^ invert (i counted from the half's start, as the probe's copies keep it), the half is folded
// into *out like a read sweep, and every mismatch is counted into the pass's LocateCounters and bitmap, and recorded
// while the pass's record buffer has room.
constexpr unsigned kLocateRecords = CRO_LOCATE_RECORDS;
constexpr unsigned kLocateGranuleShift = 21;               // 2 MiB granules of the region
struct LocateRecord {
    unsigned long long word, expected, actual;             // word: region index (half B starts at S / 8)
};
struct LocateCounters {
    unsigned long long mismatches;                          // exact
    unsigned long long claims;                              // record slots claimed (may run past kLocateRecords)
    unsigned long long bits[64];                            // mismatching words with bit b flipped
};
struct LocateBufs {
    LocateCounters* ctr;
    LocateRecord* rec;                                      // kLocateRecords entries
    unsigned long long* granules;                           // bit g: granule g of the region holds a mismatch
};
cudaError_t launch_locate(const KernelPlan&, const void* half, uint64_t bytes, uint64_t word0, uint64_t seed,
                          uint64_t invert, const LocateBufs&, const SweepScratch&, SweepOut* out, cudaStream_t);
// word = (word & and_mask) | or_mask over region words [first, first + count): the locator's test hook.
cudaError_t launch_force_words(void* base, uint64_t first, uint64_t count, uint64_t and_mask, uint64_t or_mask,
                               int sm_count, cudaStream_t);

// Host link probe (cro_probe_host_link): one launch streams over mapped pinned host memory with two roles, each a
// number of warps of every CTA (0 warps: the role is off).  The read role folds its buffer like a read sweep and
// compares every word with pattern_word(seed, i), i the buffer's own word index, counting and recording mismatches as
// the locator does (LocateBufs, word0 = 0, no granule above L); the write role stores pattern_word(seed, i).  Each role
// publishes its own SweepOut: %globaltimer window, stamp, n_words, and the fold (read) or a zero checksum (write).
constexpr int kLinkWarps = 8;                               // warps per role and CTA
struct LinkRole {
    void* buf;                                              // device address of the mapped host buffer
    uint64_t bytes;                                         // multiple of 16
    uint64_t seed;
    SweepScratch sc;                                        // the role's own reduction scratch (grid entries)
    SweepOut* out;
    unsigned warps;                                         // 0 or kLinkWarps
};
cudaError_t launch_link_stream(const LinkRole& rd, const LinkRole& wr, const LocateBufs& lb, int grid, uint64_t stamp,
                               cudaStream_t);

// SM compute probe (cro_probe_compute): one launch of leg `leg` (CRO_COMPUTE_LEG_*) runs `grid` CTAs of 256 threads,
// one per SM.  Each CTA generates the call's operands into its shared memory, computes the answer tile `iterations`
// times, folds every iteration and compares the last one element by element with *expect (M x N int32, row-major).
// It publishes one ComputeCta (stamp last written = the call number), ORs its %smid into sm_bits and records its
// mismatching elements while the record buffer has room (*claims counts the slots claimed, possibly past the end).
struct ComputeCta {
    unsigned long long stamp;                   // the call number; all ones (armed) = the CTA did not publish
    unsigned long long t0, t1;                  // %globaltimer around the iterations
    unsigned long long cycles;                  // %clock64 around the iterations
    unsigned long long mismatches;              // elements of the last iteration that differ
    unsigned long long fold_mismatches;         // threads whose running fold differs
    unsigned long long fold;                    // every thread's running fold, summed
    unsigned smid, nsmid;
};
static_assert(sizeof(ComputeCta) == 64, "one 64-byte record per CTA");
struct ComputeArgs {
    const int* expect;
    ComputeCta* cta;                            // grid entries
    unsigned long long* sm_bits;                // CRO_COMPUTE_MAX_SMS / 64 words
    cro_compute_fault* rec;                     // CRO_COMPUTE_RECORDS entries
    unsigned long long* claims;
    unsigned long long seed, stamp;
    unsigned iterations;
    int inj_sm, inj_row, inj_col;               // -1: every SM / row / column
    unsigned inj_iter, inj_mask;                // inj_mask 0: nothing is injected in this launch
};
constexpr int kComputeThreads = 256;            // two warpgroups of 64 rows each
cudaError_t launch_compute(unsigned leg, const ComputeArgs& a, int grid, cudaStream_t);

// SRAM probe (cro_probe_sram, sram_kernels.cu).  Local leg: `grid` CTAs of kSramThreads, each marching its own
// n_words of dynamic shared memory (March C-, include/croprobe.h).  Network leg: clusters of `cluster` CTAs, rank r
// with seed + r * kNonceStride.  Each CTA publishes one SramCta (stamp last = the call number) and records its
// mismatching words while the leg's record buffer has room (*claims counts the slots claimed, possibly past the end).
struct SramCta {
    unsigned long long stamp;                   // the call number; all ones (armed) = the CTA did not publish
    unsigned long long t0, t1;                  // %globaltimer around the iterations
    unsigned long long cycles;                  // %clock64 around the iterations
    unsigned long long count[CRO_SRAM_ELEMENTS];  // compares that failed, per element
    unsigned long long last;                    // ... of them in the last iteration
    unsigned long long fold_x, fold_s, fold_w;  // local: M5 fold over every iteration
    unsigned smid, nsmid, rank, block;          // rank in the cluster (0 for the local leg), blockIdx.x
};
static_assert(sizeof(SramCta) == 128, "per-CTA record");
struct SramRecord {
    unsigned element, iteration, smid;          // smid: the CTA whose compare failed
    unsigned peer_block;                        // network: blockIdx.x of the owner (D1) or the writer (D3)
    unsigned round, word;                       // round: the launch's round number, to resolve peer_block
    unsigned long long expected, actual;
};
static_assert(sizeof(SramRecord) == 40, "word record");
struct SramArgs {
    SramCta* cta;                               // grid entries
    SramRecord* rec;                            // CRO_SRAM_RECORDS entries
    unsigned long long* claims;
    unsigned long long seed, stamp;
    unsigned n_words;                           // a multiple of 32 (the march loops stay warp-uniform)
    unsigned iterations;
    unsigned round;
    int inj_sm, inj_word;                       // -1: every SM / word
    unsigned inj_element, inj_iter;
    unsigned long long inj_mask;                // 0: nothing is injected in this launch
};
constexpr int kSramThreads = 1024;
// The words each CTA marches on the current device: its opt-in shared memory per block less the kernels' static
// shared memory, rounded down to 32 words.  Sets both kernels' dynamic shared memory to that and the carve-out to
// the most shared memory.
cudaError_t sram_plan(int device, unsigned* n_words);
cudaError_t launch_sram_smem(const SramArgs& a, int grid, cudaStream_t);
cudaError_t launch_sram_dsmem(const SramArgs& a, int grid, unsigned cluster, cudaStream_t);
// Clusters of `cluster` CTAs the device can hold at once with the leg's shared memory (0: none fits).
cudaError_t sram_max_clusters(unsigned cluster, unsigned n_words, int* clusters);

// Register-file probe (cro_probe_regfile, regfile_kernels.cu): `grid` CTAs of CRO_REGFILE_THREADS, one per SM, each
// holding CRO_REGFILE_SLOTS pattern words per thread in registers (include/croprobe.h).  Each CTA publishes one
// cro_regfile_cta (stamp last = the call number) and records its mismatching slots while the record buffer has room
// (*claims counts the slots claimed, possibly past the end).
struct RegfileArgs {
    cro_regfile_cta* cta;                       // grid entries
    cro_regfile_fault* rec;                     // CRO_REGFILE_RECORDS entries
    unsigned long long* claims;
    unsigned long long seed, stamp;             // seed: iteration 0's; iteration i adds i * kNonceStride
    unsigned iterations;
    int inj_sm, inj_warp, inj_lane, inj_slot;   // -1: every SM / warp / lane / slot
    unsigned inj_element, inj_iter;
    unsigned inj_mask;                          // 0: nothing is injected in this launch
};
// Sets the kernel's dynamic shared memory (the source words) and carve-out; *fa gets its attributes (numRegs).
// cudaErrorInvalidConfiguration when the device's opt-in shared memory per block cannot hold the source.
cudaError_t regfile_plan(int device, cudaFuncAttributes* fa);
cudaError_t launch_regfile(const RegfileArgs& a, int grid, cudaStream_t);

// Pointer chase for NVLink latency: warp j of the one CTA follows `hops` dependent ld.relaxed.sys loads through
// table[j] (one 8-byte slot per 128-byte line, peer-resident); out[2j] = final index, out[2j+1] = %globaltimer ns.
struct ChaseArgs {
    const unsigned long long* table[CRO_MAX_DEVICES];
    unsigned start[CRO_MAX_DEVICES];
    unsigned n;           // tables to chase concurrently (one warp each)
    unsigned hops;
};
cudaError_t launch_chase(const ChaseArgs& a, unsigned long long* out, cudaStream_t);
// The chase output before the chase: every word all 0xFF bytes.  No chase ends there (a table has 65536 slots), so a
// row the chase did not walk fails the end check at any hop count.
constexpr unsigned long long kChaseArmed = ~0ull;
constexpr size_t kChaseOutWords = 2 * CRO_MAX_DEVICES;
cudaError_t arm_chase_out(unsigned long long* out, cudaStream_t);

// Slot map of one device's SweepOut array (d_out): include/croprobe.h's, which the test hooks share.
constexpr int kSlotFill = CRO_SLOT_FILL;
constexpr int kSlotSweep0 = CRO_SLOT_SWEEP0;          // copies first, then reads: 1 .. 1 + C + R
constexpr int kMaxSweepsEach = CRO_MAX_SWEEPS_EACH;
constexpr int kSlotExpect = CRO_SLOT_EXPECT;          // closed form of the whole region
constexpr int kSlotPrefix = CRO_SLOT_PREFIX;          // closed form of the first p2p_bytes (what peers must read)
constexpr int kSlotP2P0 = CRO_SLOT_P2P0;              // per peer j: 64 + 3j + {0 read, 1 push, 2 receiver re-read}
constexpr int kSlotScratch = CRO_SLOT_SCRATCH;        // single-sweep entry points
constexpr int kSlotCount = CRO_SLOT_COUNT;
static_assert(kSlotSweep0 + 2 * kMaxSweepsEach <= kSlotExpect && kSlotPrefix + 1 == kSlotP2P0, "slot map");

// The probe's verdict, computed on the device: fills *out (the all-gather send buffer) from the template
// (identity, staged at init), the sweep slots and the closed form.  One CTA.
struct FinalizeArgs {
    const cro_probe_result* tmpl;
    cro_probe_result* out;
    const SweepOut* slots;
    const ProbeParams* pp;
    unsigned long long sweep_bytes;
    unsigned read_sweeps, copy_sweeps;
    unsigned read_variant, copy_variant;
    unsigned fused;          // copy sweeps carry a checksum of their source stream
};
// The arguments of one probe's finalize: `cv` is the resolved copy variant, C the copy sweeps actually run (a probe
// without copies reports copy variant 0).
inline FinalizeArgs finalize_args(const cro_probe_result* tmpl, cro_probe_result* out, const SweepOut* slots,
                                  const ProbeParams* pp, unsigned long long sweep_bytes, unsigned R, unsigned C,
                                  unsigned rv, unsigned cv) {
    FinalizeArgs fa{};
    fa.tmpl = tmpl;
    fa.out = out;
    fa.slots = slots;
    fa.pp = pp;
    fa.sweep_bytes = sweep_bytes;
    fa.read_sweeps = R;
    fa.copy_sweeps = C;
    fa.read_variant = rv;
    fa.copy_variant = C ? cv : 0;
    fa.fused = (cv == COPY_TMA_FUSED) ? 1u : 0u;
    return fa;
}
cudaError_t launch_finalize(const FinalizeArgs& a, cudaStream_t);

// NVLink part of the verdict: folds the per-peer slots of this device (and the peers' slots it must agree with)
// into out->p2p_* and out->status.  One CTA.
struct P2PFinalizeArgs {
    cro_probe_result* out;
    const SweepOut* slots;                        // this device's
    const SweepOut* peer_slots[CRO_MAX_DEVICES];  // peer j's slot array (peer-mapped), null = no such peer
    const unsigned long long* chase_out;          // [2j] end index, [2j+1] ns, indexed by peer
    unsigned chase_expect[CRO_MAX_DEVICES];       // where the chase into peer j must end
    unsigned n;                                   // devices managed
    unsigned self;
    unsigned hops;
    unsigned have_push;
    unsigned push_folded;                         // the push kernel carries a checksum of its source (COPY_TMA_FUSED)
    unsigned long long p2p_bytes;
    unsigned long long stamp;                     // nonce every p2p slot this device wrote must carry
    unsigned long long peer_stamp[CRO_MAX_DEVICES];   // ... and the nonce of peer j's closed-form slot
};
cudaError_t launch_p2p_finalize(const P2PFinalizeArgs& a, cudaStream_t);

}  // namespace cro
