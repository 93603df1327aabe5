// lane_tally.cuh — the device half of the per-thread report path the cross-lane and ALU probes share
// (xlane_kernels.cu, alu_kernels.cu; the host half is lane_report.hpp).  Each thread counts its failed compares, keeps
// its first kR records in its own slots, folds its last iteration's results and publishes them with plain stores;
// thread 0 publishes the CTA's window.  No ballot, shuffle, shared tally or atomic: nothing here uses the units those
// probes check.
#pragma once

namespace cro {

__device__ __forceinline__ unsigned long long lane_timer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

template <class Fault, unsigned kR>
struct LaneCounts {
    unsigned long long count = 0, last = 0, fx = 0, fs = 0, fw = 0;
    Fault* rec;
    // A failed compare: make() is the record, kept while the thread has a slot left.
    template <class Make>
    __device__ __forceinline__ void miss(bool lastit, Make make) {
        if (count < kR) rec[count] = make();
        ++count;
        last += lastit ? 1u : 0u;
    }
    __device__ __forceinline__ void fold(unsigned op, unsigned long long v) {
        fx ^= v;
        fs += v;
        fw += v * (2ull * op + 1ull);
    }
    // The thread's entry, then (thread 0) the CTA's: each stamped last, after a fence.
    template <class Thread, class Cta>
    __device__ __forceinline__ void publish(Thread& o, Cta* cta, unsigned long long stamp, unsigned long long t0, unsigned long long t1,
                                            long long k0, long long k1, unsigned smid, unsigned nsmid) const {
        o.count = count;
        o.last = last;
        o.fold_x = fx;
        o.fold_s = fs;
        o.fold_w = fw;
        __threadfence();
        o.stamp = stamp;
        if (threadIdx.x == 0) {
            Cta& c = cta[blockIdx.x];
            c.t0 = t0;
            c.t1 = t1;
            c.cycles = (unsigned long long)(k1 - k0);
            c.smid = smid;
            c.nsmid = nsmid;
            c.block = blockIdx.x;
            c.reserved = 0;
            __threadfence();
            c.stamp = stamp;
        }
    }
};

}  // namespace cro
