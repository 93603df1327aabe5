// barrier_kernels.cu — the barrier probe's kernels (cro_probe_barrier): one instantiation and one launch per leg, one
// CTA of 8 warps per SM (the CLUSTER leg: clusters of 2, 4 or 8 such CTAs).  The device computes no expected value:
// each row's barrier ids, counts, participants, held-back thread and expected results come from the host's table.
// Each form's instructions sit once in the iteration loop, where tests/test_barrier_abi.py finds them in the SASS.
// Every mbarrier wait is bounded by %globaltimer and no branch depends on a compared value, so a failed check cannot
// desynchronise the CTA; bar.sync, bar.red and barrier.cluster.wait cannot be bounded.  The report path is
// lane_tally.cuh: plain stores, no barrier, vote or atomic.
#include "barrier_kernels.cuh"
#include "lane_tally.cuh"

namespace cro {

namespace {

typedef unsigned long long u64;
constexpr unsigned kT = CRO_BARRIER_THREADS;
// More than half of an SM's shared memory, so no second CTA of any kernel shares the SM.
constexpr size_t kSmemBytes = 160u << 10;

struct Tally : LaneCounts<cro_barrier_fault, CRO_BARRIER_THREAD_RECORDS> {
    unsigned leg, smid, warp, lane;
};

// What one iteration needs beyond the tally: the row injected in this iteration (~0u: none) and its mask.
struct Iter {
    unsigned it, inj_op;
    bool lastit;
    u64 mask;
};

// One check: the mask XORed in when the row is injected, a record when the value differs, and (last iteration,
// `fold`) the value folded.
__device__ __forceinline__ void check(Tally& T, const Iter& I, unsigned op, unsigned kind, unsigned bar, unsigned phase, unsigned slot,
                                      unsigned peer, u64 expected, u64 got, bool fold = true) {
    const u64 v = got ^ (op == I.inj_op ? I.mask : 0ull);
    if (v != expected)
        T.miss(I.lastit, [&] {
            return cro_barrier_fault{T.leg, op, I.it, T.smid, T.warp, T.lane, kind, bar, phase, slot, peer, 0u, expected, v};
        });
    if (I.lastit && fold) T.fold(op, v);
}

// ---- named barriers ----
__device__ __forceinline__ void bar_sync(unsigned id, unsigned n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }
__device__ __forceinline__ void bar_arrive(unsigned id, unsigned n) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(n) : "memory"); }
__device__ __forceinline__ unsigned bar_popc(unsigned id, unsigned n, unsigned p) {
    unsigned d;
    asm volatile("{ .reg .pred q; setp.ne.u32 q, %3, 0; bar.red.popc.u32 %0, %1, %2, q; }" : "=r"(d) : "r"(id), "r"(n), "r"(p) : "memory");
    return d;
}
__device__ __forceinline__ unsigned bar_and(unsigned id, unsigned n, unsigned p) {
    unsigned d;
    asm volatile("{ .reg .pred q, r; setp.ne.u32 q, %3, 0; bar.red.and.pred r, %1, %2, q; selp.u32 %0, 1, 0, r; }"
                 : "=r"(d) : "r"(id), "r"(n), "r"(p) : "memory");
    return d;
}
__device__ __forceinline__ unsigned bar_or(unsigned id, unsigned n, unsigned p) {
    unsigned d;
    asm volatile("{ .reg .pred q, r; setp.ne.u32 q, %3, 0; bar.red.or.pred r, %1, %2, q; selp.u32 %0, 1, 0, r; }"
                 : "=r"(d) : "r"(id), "r"(n), "r"(p) : "memory");
    return d;
}
__device__ __forceinline__ void st_shared(unsigned addr, unsigned v) { asm volatile("st.shared.u32 [%0], %1;" ::"r"(addr), "r"(v) : "memory"); }
__device__ __forceinline__ unsigned ld_shared(unsigned addr) {
    unsigned v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
    return v;
}
__device__ __forceinline__ void st_shared4(unsigned addr, unsigned a, unsigned b, unsigned c, unsigned d) {
    asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
__device__ __forceinline__ u64 ld_shared64(unsigned addr) {
    u64 v;
    asm volatile("ld.shared.u64 %0, [%1];" : "=l"(v) : "r"(addr) : "memory");
    return v;
}
__device__ __forceinline__ void st_shared64(unsigned addr, u64 v) { asm volatile("st.shared.u64 [%0], %1;" ::"r"(addr), "l"(v) : "memory"); }

// ---- mbarrier (the SYNCS unit) ----
__device__ __forceinline__ void mb_init(unsigned mb, unsigned n) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(mb), "r"(n) : "memory"); }
__device__ __forceinline__ void mb_inval(unsigned mb) { asm volatile("mbarrier.inval.shared::cta.b64 [%0];" ::"r"(mb) : "memory"); }
__device__ __forceinline__ void mb_arrive(unsigned mb) {
    asm volatile("{ .reg .b64 s; mbarrier.arrive.shared::cta.b64 s, [%0]; }" ::"r"(mb) : "memory");
}
__device__ __forceinline__ void mb_arrive_n(unsigned mb, unsigned n) {
    asm volatile("{ .reg .b64 s; mbarrier.arrive.shared::cta.b64 s, [%0], %1; }" ::"r"(mb), "r"(n) : "memory");
}
__device__ __forceinline__ void mb_arrive_drop(unsigned mb) {
    asm volatile("{ .reg .b64 s; mbarrier.arrive_drop.shared::cta.b64 s, [%0]; }" ::"r"(mb) : "memory");
}
// The pending count of the phase as the arrive found it: the state is opaque, read only through pending_count.
__device__ __forceinline__ unsigned mb_ticket(unsigned mb) {
    unsigned n;
    asm volatile("{ .reg .b64 s; mbarrier.arrive.noComplete.shared::cta.b64 s, [%1], 1; mbarrier.pending_count.b64 %0, s; }"
                 : "=r"(n) : "r"(mb) : "memory");
    return n;
}
__device__ __forceinline__ void mb_arrive_tx(unsigned mb, unsigned bytes) {
    asm volatile("{ .reg .b64 s; mbarrier.arrive.expect_tx.shared::cta.b64 s, [%0], %1; }" ::"r"(mb), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mb_complete_tx(unsigned mb, unsigned bytes) {
    asm volatile("mbarrier.complete_tx.shared::cta.b64 [%0], %1;" ::"r"(mb), "r"(bytes) : "memory");
}
__device__ __forceinline__ unsigned mb_test(unsigned mb, unsigned par) {
    unsigned d;
    asm volatile("{ .reg .pred p; mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                 : "=r"(d) : "r"(mb), "r"(par) : "memory");
    return d;
}
// try_wait.parity until the phase completes or CRO_BARRIER_WAIT_NS have been spent waiting; *out: the budget ran out.
// %globaltimer is wall time, and a time-sliced GPU can stop the CTA between two reads for longer than the budget, so
// each step counts at most kWaitStepNs: a stopped CTA does not run out its budget, and a wait that never completes
// still ends, after at least CRO_BARRIER_WAIT_NS / kWaitStepNs steps.
constexpr u64 kWaitStepNs = 1000000;
template <bool kCluster>
__device__ __forceinline__ unsigned mb_wait(unsigned mb, unsigned par, bool* out) {
    u64 prev = lane_timer_ns(), spent = 0;
    unsigned d;
    do {
        if constexpr (kCluster)
            asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                         : "=r"(d) : "r"(mb), "r"(par) : "memory");
        else
            asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                         : "=r"(d) : "r"(mb), "r"(par) : "memory");
        const u64 now = lane_timer_ns();
        spent += now - prev < kWaitStepNs ? now - prev : kWaitStepNs;
        prev = now;
    } while (!d && spent < CRO_BARRIER_WAIT_NS);
    *out = !d;
    return d;
}

// ---- cluster ----
__device__ __forceinline__ void cluster_sync() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ unsigned mapa(unsigned addr, unsigned rank) {
    unsigned r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank));
    return r;
}
__device__ __forceinline__ unsigned ld_cluster(unsigned addr) {
    unsigned v;
    asm volatile("ld.shared::cluster.u32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
    return v;
}
__device__ __forceinline__ unsigned ctarank(unsigned addr) {
    unsigned r;
    asm volatile("getctarank.shared::cluster.u32 %0, %1;" : "=r"(r) : "r"(addr));
    return r;
}

#define ST_ASYNC(ty, ...) asm volatile("st.async.shared::cluster.mbarrier::complete_tx::bytes" ty " [%0], " __VA_ARGS__)
#define RED_ASYNC(op, v)                                                                                                         \
    asm volatile("red.async.relaxed.cluster.shared::cluster.mbarrier::complete_tx::bytes" op " [%0], %1, [%2];" ::"r"(dst), v, \
                 "r"(mbn)                                                                                                        \
                 : "memory")

__device__ __forceinline__ void send(unsigned form, unsigned dst, unsigned mbn, u64 w0, u64 w1) {
    const unsigned a = (unsigned)w0, b = (unsigned)(w0 >> 32), c = (unsigned)w1, d = (unsigned)(w1 >> 32);
    switch (form) {
        case CRO_BARRIER_FORM_ST_B32: ST_ASYNC(".b32", "%1, [%2];" ::"r"(dst), "r"(a), "r"(mbn) : "memory"); break;
        case CRO_BARRIER_FORM_ST_B64: ST_ASYNC(".b64", "%1, [%2];" ::"r"(dst), "l"(w0), "r"(mbn) : "memory"); break;
        case CRO_BARRIER_FORM_ST_V2: ST_ASYNC(".v2.b32", "{%1, %2}, [%3];" ::"r"(dst), "r"(a), "r"(b), "r"(mbn) : "memory"); break;
        case CRO_BARRIER_FORM_ST_V4:
            ST_ASYNC(".v4.b32", "{%1, %2, %3, %4}, [%5];" ::"r"(dst), "r"(a), "r"(b), "r"(c), "r"(d), "r"(mbn) : "memory");
            break;
        case CRO_BARRIER_FORM_RED_ADD: RED_ASYNC(".add.u32", "r"(a)); break;
        case CRO_BARRIER_FORM_RED_ADD64: RED_ASYNC(".add.u64", "l"(w0)); break;
        case CRO_BARRIER_FORM_RED_MIN: RED_ASYNC(".min.u32", "r"(a)); break;
        case CRO_BARRIER_FORM_RED_MAX: RED_ASYNC(".max.u32", "r"(a)); break;
        case CRO_BARRIER_FORM_RED_MINS: RED_ASYNC(".min.s32", "r"(a)); break;
        case CRO_BARRIER_FORM_RED_MAXS: RED_ASYNC(".max.s32", "r"(a)); break;
        case CRO_BARRIER_FORM_RED_AND: RED_ASYNC(".and.b32", "r"(a)); break;
        case CRO_BARRIER_FORM_RED_OR: RED_ASYNC(".or.b32", "r"(a)); break;
        case CRO_BARRIER_FORM_RED_XOR: RED_ASYNC(".xor.b32", "r"(a)); break;
        case CRO_BARRIER_FORM_RED_INC: RED_ASYNC(".inc.u32", "r"(a)); break;
        default: RED_ASYNC(".dec.u32", "r"(a)); break;
    }
}

__device__ __forceinline__ u64 word(const BarrierArgs& a, unsigned row, unsigned t, unsigned j) {
    return __ldg(a.words + ((size_t)row * kT + t) * 2 + j);
}

// ---- BAR: every row, then a whole-CTA bar.sync on another id before the next row reuses any participant ----
__device__ __forceinline__ void bar_row(Tally& T, const Iter& I, const BarrierArgs& a, unsigned op, unsigned base) {
    const cro_barrier_row& R = a.rows[op];
    const unsigned form = __ldg(&R.form), id = __ldg(&R.bar), n = __ldg(&R.count), warps = __ldg(&R.warps), prod = __ldg(&R.producers);
    const unsigned t = threadIdx.x, w = t >> 5, sep = id ^ 1u;
    const bool part = warps >> w & 1u, producer = prod >> w & 1u;
    if (form == CRO_BARRIER_FORM_ARRIVE) {
        if (producer) {
            st_shared(base + barrier::kSlotOff + 4 * t, (unsigned)word(a, op, t, 0));
            bar_arrive(id, n);
        } else if (part) {
            bar_sync(id, n);
#pragma unroll 1
            for (unsigned p = 0; p < kT; ++p)
                if (prod >> (p >> 5) & 1u)
                    check(T, I, op, CRO_BARRIER_KIND_EARLY, id, 0, p, T.smid, word(a, op, p, 0), ld_shared(base + barrier::kSlotOff + 4 * p));
        }
        bar_sync(sep, kT);
        if (producer) st_shared(base + barrier::kSlotOff + 4 * t, 0u);
        return;
    }
    if (part) {
        const unsigned p = __ldg(&R.pred[w]) >> (t & 31) & 1u;
        const unsigned d = form == CRO_BARRIER_FORM_POPC ? bar_popc(id, n, p) : form == CRO_BARRIER_FORM_AND ? bar_and(id, n, p) : bar_or(id, n, p);
        check(T, I, op, CRO_BARRIER_KIND_VALUE, id, 0, 0, T.smid, __ldg(&R.expect), d);
    }
    bar_sync(sep, kT);
}

// ---- MBAR: a fresh mbarrier per row, K phases, one arrival or byte piece held back per phase ----
__device__ __forceinline__ void mbar_row(Tally& T, const Iter& I, const BarrierArgs& a, unsigned op, unsigned base) {
    const cro_barrier_row& R = a.rows[op];
    const unsigned form = __ldg(&R.form), warps = __ldg(&R.warps), phases = __ldg(&R.phases), held = __ldg(&R.held),
                   arriver = __ldg(&R.arriver), total = (unsigned)__ldg(&R.expect);
    const unsigned t = threadIdx.x, w = t >> 5, mb = base + barrier::kMbarOff;
    const bool part = warps >> w & 1u;
    const unsigned mine = (unsigned)word(a, op, t, 0);   // COUNT: arrivals; TX: bytes; DROP: 1 = drops
    if (t == 0) mb_init(mb, __ldg(&R.count));
    bar_sync(0, kT);
#pragma unroll 1
    for (unsigned j = 0; j < phases; ++j) {
        const unsigned par = j & 1u;
        unsigned ticket = 0;
        if (form == CRO_BARRIER_FORM_TICKET && part) {
            ticket = mb_ticket(mb);
            st_shared(base + barrier::kTicketOff + 4 * ((ticket - 2u) & (barrier::kTicketSlots - 1)), t);
        } else if (form == CRO_BARRIER_FORM_COUNT && part && t != held) {
            mb_arrive_n(mb, mine);
        } else if (form == CRO_BARRIER_FORM_DROP && part && t != held && (j == 0 || !mine)) {
            if (j == 0 && mine) mb_arrive_drop(mb);
            else mb_arrive(mb);
        } else if (form == CRO_BARRIER_FORM_TX) {
            if (t == arriver) mb_arrive_tx(mb, total);
            if (part && t != held) mb_complete_tx(mb, mine);
        }
        bar_sync(0, kT);
        if (form == CRO_BARRIER_FORM_TICKET && part) {
            const unsigned n = __ldg(&R.count) - 1u;       // tickets N+1 .. 2 of the N participants
            check(T, I, op, CRO_BARRIER_KIND_TICKET, form, j, 0, T.smid, 1, ticket - 2u < n ? 1u : 0u);
            check(T, I, op, CRO_BARRIER_KIND_TICKET, form, j, 1, T.smid, t,
                  ld_shared(base + barrier::kTicketOff + 4 * ((ticket - 2u) & (barrier::kTicketSlots - 1))));
        }
        check(T, I, op, CRO_BARRIER_KIND_EARLY, form, j, 2, T.smid, 0, mb_test(mb, par));
        check(T, I, op, CRO_BARRIER_KIND_VALUE, form, j, 3, T.smid, 1, mb_test(mb, par ^ 1u));
        bar_sync(0, kT);
        if (t == held) {
            if (form == CRO_BARRIER_FORM_COUNT) mb_arrive_n(mb, mine);
            else if (form == CRO_BARRIER_FORM_TX) mb_complete_tx(mb, mine);
            else mb_arrive(mb);
        }
        bool out;
        const unsigned done = mb_wait<false>(mb, par, &out);
        check(T, I, op, out ? CRO_BARRIER_KIND_TIMEOUT : CRO_BARRIER_KIND_VALUE, form, j, 4, T.smid, 1, done);
    }
    bar_sync(0, kT);
    if (t == 0) mb_inval(mb);
}

// ---- CLUSTER ----
struct Peers {
    unsigned rank, next, next_smid, prev_smid;
};

__device__ __forceinline__ void cluster_row(Tally& T, const Iter& I, const BarrierArgs& a, unsigned op, unsigned base, const Peers& P,
                                            unsigned par) {
    const cro_barrier_row& R = a.rows[op];
    const unsigned form = __ldg(&R.form), t = threadIdx.x;
    if (form == CRO_BARRIER_FORM_CBAR) {
        const unsigned mine = base + barrier::kCbarOff + op * 1024u + 4 * t;
        const unsigned w0 = (unsigned)word(a, op, t, 0);
        st_shared(mine, w0);
        cluster_sync();
        const unsigned there = mapa(mine, P.next);
        check(T, I, op, CRO_BARRIER_KIND_EARLY, form, 0, 0, P.next_smid, w0, ld_cluster(there));
        check(T, I, op, CRO_BARRIER_KIND_VALUE, form, 0, 1, P.next_smid, __ldg(&R.next_rank[P.rank]), ctarank(there), false);
        cluster_sync();
        st_shared(mine, 0u);
        return;
    }
    const bool red = form >= CRO_BARRIER_FORM_RED_ADD, wide = form == CRO_BARRIER_FORM_RED_ADD64;
    const unsigned slots = __ldg(&R.arriver), recv = base + barrier::kRecvOff + (op - barrier::kCbarRows) * 4096u;
    const unsigned mb = base + barrier::kClusterMbarOff + 8 * op;
    if (!red) st_shared4(recv + 16 * t, 0, 0, 0, 0);
    else if (t < slots) st_shared64(recv + 8 * t, __ldg(&R.slot_init[t]));
    if (t == 0) mb_arrive_tx(mb, __ldg(&R.count));
    cluster_sync();
    const u64 w0 = word(a, op, t, 0), w1 = word(a, op, t, 1);
    send(form, mapa(red ? recv + 8 * (t % slots) : recv + 16 * t, P.next), mapa(mb, P.next), w0, w1);
    bool out;
    const unsigned done = mb_wait<true>(mb, par, &out);
    check(T, I, op, out ? CRO_BARRIER_KIND_TIMEOUT : CRO_BARRIER_KIND_VALUE, form, 0, 2, P.prev_smid, 1, done);
    if (!red) {
        check(T, I, op, CRO_BARRIER_KIND_VALUE, form, 0, 0, P.prev_smid, w0, ld_shared64(recv + 16 * t));
        check(T, I, op, CRO_BARRIER_KIND_VALUE, form, 0, 1, P.prev_smid, w1, ld_shared64(recv + 16 * t + 8));
    } else if (t < slots) {
        const u64 v = ld_shared64(recv + 8 * t);
        check(T, I, op, CRO_BARRIER_KIND_VALUE, form, 0, 0, P.prev_smid, __ldg(&R.slot_expect[t]), wide ? v : v & 0xFFFFFFFFull);
    }
}

template <unsigned LEG>
__global__ void __launch_bounds__(kT, 1) barrier_kernel(const BarrierArgs a) {
    extern __shared__ __align__(16) unsigned char barrier_smem[];
    unsigned smid, nsmid;
    asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
    asm volatile("mov.u32 %0, %%nsmid;" : "=r"(nsmid));
    const unsigned t = threadIdx.x, w = t >> 5, l = t & 31u;
    const unsigned base = (unsigned)__cvta_generic_to_shared(barrier_smem);
    const size_t me = (size_t)blockIdx.x * kT + t;
    const bool inj = a.inj_mask && (a.inj_sm < 0 || (unsigned)a.inj_sm == smid) && (a.inj_warp < 0 || (unsigned)a.inj_warp == w) &&
                     (a.inj_lane < 0 || (unsigned)a.inj_lane == l);
    Tally T;
    T.rec = a.rec + me * CRO_BARRIER_THREAD_RECORDS;
    T.leg = LEG;
    T.smid = smid;
    T.warp = w;
    T.lane = l;
    Iter I;
    I.mask = a.inj_mask;
    Peers P{};
    constexpr unsigned kRows = barrier::kOps[LEG];
    if constexpr (LEG == CRO_BARRIER_LEG_BAR) {
        st_shared(base + barrier::kSlotOff + 4 * t, 0u);
        bar_sync(0, kT);
    } else if constexpr (LEG == CRO_BARRIER_LEG_CLUSTER) {
        unsigned size;
        asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(P.rank));
        asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(size));
        P.next = P.rank + 1 == size ? 0u : P.rank + 1;
        const unsigned prev = P.rank == 0 ? size - 1 : P.rank - 1;
        if (t == 0) {
            st_shared(base + barrier::kSmidOff, smid);
            for (unsigned op = barrier::kCbarRows; op < CRO_BARRIER_CLUSTER_OPS; ++op) mb_init(base + barrier::kClusterMbarOff + 8 * op, 1);
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        }
        cluster_sync();
        P.next_smid = ld_cluster(mapa(base + barrier::kSmidOff, P.next));
        P.prev_smid = ld_cluster(mapa(base + barrier::kSmidOff, prev));
    }
    const unsigned long long t0 = lane_timer_ns();
    const long long k0 = clock64();
#pragma unroll 1
    for (unsigned it = 0; it < a.iterations; ++it) {
        I.it = it;
        I.lastit = it + 1 == a.iterations;
        I.inj_op = inj && it == a.inj_iter ? a.inj_op : ~0u;
#pragma unroll 1
        for (unsigned op = 0; op < kRows; ++op) {
            if constexpr (LEG == CRO_BARRIER_LEG_BAR) bar_row(T, I, a, op, base);
            else if constexpr (LEG == CRO_BARRIER_LEG_MBAR) mbar_row(T, I, a, op, base);
            else cluster_row(T, I, a, op, base, P, it & 1u);
        }
    }
    const long long k1 = clock64();
    const unsigned long long t1 = lane_timer_ns();
    // No CTA of a cluster leaves while a peer may still read its shared memory or send into it.
    if constexpr (LEG == CRO_BARRIER_LEG_CLUSTER) cluster_sync();
    T.publish(a.thr[me], a.cta, a.stamp, t0, t1, k0, k1, smid, nsmid);
}

template <unsigned LEG>
cudaError_t plan_leg() {
    return cudaFuncSetAttribute(barrier_kernel<LEG>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBytes);
}

cudaLaunchConfig_t cluster_config(int grid, unsigned cluster, cudaStream_t st, cudaLaunchAttribute* attr) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)grid);
    cfg.blockDim = dim3(kT);
    cfg.dynamicSmemBytes = kSmemBytes;
    cfg.stream = st;
    attr->id = cudaLaunchAttributeClusterDimension;
    attr->val.clusterDim.x = cluster;
    attr->val.clusterDim.y = 1;
    attr->val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cfg;
}

}  // namespace

cudaError_t barrier_plan(int device, unsigned leg) {
    int optin = 0;
    cudaError_t e = cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device);
    if (e) return e;
    if ((size_t)optin < kSmemBytes) return cudaErrorInvalidConfiguration;
    switch (leg) {
        case CRO_BARRIER_LEG_BAR: return plan_leg<CRO_BARRIER_LEG_BAR>();
        case CRO_BARRIER_LEG_MBAR: return plan_leg<CRO_BARRIER_LEG_MBAR>();
        default: return plan_leg<CRO_BARRIER_LEG_CLUSTER>();
    }
}

cudaError_t barrier_cluster_grid(unsigned cluster, int* grid) {
    cudaLaunchAttribute attr;
    const cudaLaunchConfig_t cfg = cluster_config((int)cluster, cluster, nullptr, &attr);
    int clusters = 0;
    const cudaError_t e = cudaOccupancyMaxActiveClusters(&clusters, barrier_kernel<CRO_BARRIER_LEG_CLUSTER>, &cfg);
    *grid = clusters * (int)cluster;
    return e;
}

cudaError_t launch_barrier(unsigned leg, const BarrierArgs& a, int grid, unsigned cluster, cudaStream_t st) {
    switch (leg) {
        case CRO_BARRIER_LEG_BAR: barrier_kernel<CRO_BARRIER_LEG_BAR><<<grid, kT, kSmemBytes, st>>>(a); break;
        case CRO_BARRIER_LEG_MBAR: barrier_kernel<CRO_BARRIER_LEG_MBAR><<<grid, kT, kSmemBytes, st>>>(a); break;
        default: {
            cudaLaunchAttribute attr;
            const cudaLaunchConfig_t cfg = cluster_config(grid, cluster, st, &attr);
            return cudaLaunchKernelEx(&cfg, barrier_kernel<CRO_BARRIER_LEG_CLUSTER>, a);
        }
    }
    return cudaGetLastError();
}

}  // namespace cro
