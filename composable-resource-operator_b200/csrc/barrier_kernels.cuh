// barrier_kernels.cuh — the barrier probe's shape (cro_probe_barrier): the kernels' arguments and shared-memory map,
// shared by the kernels (barrier_kernels.cu), which run each row of the host's table, and the host (barrier_probe.cu),
// which builds that table.  oracle/barrier.py restates the table and every check.
#pragma once
#include "kernels.cuh"

namespace cro {

struct BarrierArgs {
    const cro_barrier_row* rows;        // the leg's rows
    const unsigned long long* words;    // the leg's words: (row * CRO_BARRIER_THREADS + thread) * 2 + j
    cro_barrier_cta* cta;               // grid entries
    cro_barrier_thread* thr;            // grid * CRO_BARRIER_THREADS entries, by block then thread
    cro_barrier_fault* rec;             // CRO_BARRIER_THREAD_RECORDS per thread entry
    unsigned long long stamp;
    unsigned iterations;
    int inj_sm, inj_warp, inj_lane;     // -1: every SM / warp / lane
    unsigned inj_op, inj_iter;
    unsigned long long inj_mask;        // 0: nothing is injected in this launch (or not in this leg)
};
// Sets the leg's dynamic shared memory request; cudaErrorInvalidConfiguration when the device cannot hold it.
cudaError_t barrier_plan(int device, unsigned leg);
// The CLUSTER leg's grid: as many clusters of `cluster` CTAs as the device holds at once, times cluster.
cudaError_t barrier_cluster_grid(unsigned cluster, int* grid);
cudaError_t launch_barrier(unsigned leg, const BarrierArgs& a, int grid, unsigned cluster, cudaStream_t);

namespace barrier {

constexpr unsigned kOps[CRO_BARRIER_LEGS] = {CRO_BARRIER_BAR_OPS, CRO_BARRIER_MBAR_OPS, CRO_BARRIER_CLUSTER_OPS};
constexpr unsigned kCbarRows = 2;       // CLUSTER rows 0 .. 1 are CBAR, then one row per async form
constexpr unsigned kTicketSlots = 512;

// Shared-memory byte offsets (of the 160 KiB each CTA asks for).
constexpr unsigned kSlotOff = 0;                                    // BAR producer words: u32 per thread
constexpr unsigned kTicketOff = 1024;                               // MBAR ticket slots: u32 x kTicketSlots
constexpr unsigned kMbarOff = 3072;                                 // MBAR's mbarrier
constexpr unsigned kSmidOff = 3080;                                 // CLUSTER: the CTA's %smid
constexpr unsigned kClusterMbarOff = 3136;                          // CLUSTER: one mbarrier per row
constexpr unsigned kCbarOff = 4096;                                 // CLUSTER CBAR rows: u32 per thread, 1 KiB per row
constexpr unsigned kRecvOff = 8192;                                 // CLUSTER async rows: 16 bytes per thread, 4 KiB per row

}  // namespace barrier
}  // namespace cro
