// warp_claim.cuh — the warp-aggregated claim of record slots that every word- or element-checking kernel shares (the
// locator, the link probe, the compute probe and the SRAM probe).
#pragma once

namespace cro {

// Slots for the records of a warp: lane l writes n_lane records.  Lane 0 first runs lane0(n_warp) with the warp's
// total, then claims that many slots with one atomic on *claims, while *claims is still below cap (so the claim count
// may run past cap but stops growing soon after).  Returns this lane's first slot, its later records taking the slots
// after it; a slot >= cap is not written.  The whole warp calls this.
template <class Lane0>
__device__ __forceinline__ unsigned long long warp_claim(unsigned n_lane, unsigned long long* claims, unsigned long long cap,
                                                         Lane0 lane0) {
    const unsigned lane = threadIdx.x & 31u;
    const unsigned n_warp = __reduce_add_sync(0xffffffffu, n_lane);
    unsigned incl = n_lane;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= (unsigned)o) incl += t;
    }
    unsigned long long base = cap;
    if (lane == 0) {
        lane0(n_warp);
        if (*reinterpret_cast<volatile unsigned long long*>(claims) < cap) base = atomicAdd(claims, (unsigned long long)n_warp);
    }
    return __shfl_sync(0xffffffffu, base, 0) + (incl - n_lane);
}

}  // namespace cro
