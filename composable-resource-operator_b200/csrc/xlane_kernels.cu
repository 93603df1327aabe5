// xlane_kernels.cu — the cross-lane probe's kernels (cro_probe_xlane): one instantiation and one launch per leg, one
// CTA of 8 warps per SM, each lane checking every op of its leg against the answer it computes from the iteration's
// seed (xlane_kernels.cuh).
//
// The report path uses none of the units under test: each thread counts its mismatches, keeps its first
// CRO_XLANE_THREAD_RECORDS records in its own slots, folds the last iteration's results and publishes them with plain
// stores; thread 0 publishes the CTA's window.  No ballot gate, warp-aggregated claim, shared tally or global atomic:
// tests/test_xlane_abi.py checks on the SASS that an instantiation issues only its own leg's cross-lane forms.
#include "lane_tally.cuh"
#include "xlane_kernels.cuh"

namespace cro {

namespace {

using xlane::u64;
constexpr unsigned kT = CRO_XLANE_THREADS;
constexpr unsigned kR = CRO_XLANE_THREAD_RECORDS;
// More than half of an SM's shared memory, so no second CTA of any kernel shares the SM.
constexpr size_t kSmemBytes = 160u << 10;
constexpr unsigned kArenaWords = 1024;                  // ATOMS: 8-byte words, then 512 presence bytes
constexpr unsigned kCasTries = 512;                     // more than any group's size: a correct unit never runs out

// What a thread accumulates for its own entry.
struct Tally : LaneCounts<cro_xlane_fault, kR> {
    unsigned leg, smid, warp, lane;
    __device__ __forceinline__ void check(unsigned it, bool lastit, unsigned op, unsigned peer, u64 e, u64 got) {
        if (got != e) miss(lastit, [&] { return cro_xlane_fault{leg, op, it, smid, warp, lane, peer, 0u, e, got}; });
        if (lastit) fold(op, got);
    }
};

// ---- SHFL ----
__device__ __forceinline__ u64 shfl(unsigned mode, unsigned x, unsigned b, unsigned c) {
    unsigned d, p;
    switch (mode) {
        case xlane::kShflUp:
            asm volatile("{ .reg .pred q; shfl.sync.up.b32 %0|q, %2, %3, %4, 0xffffffff; selp.u32 %1, 1, 0, q; }"
                         : "=r"(d), "=r"(p) : "r"(x), "r"(b), "r"(c));
            break;
        case xlane::kShflDown:
            asm volatile("{ .reg .pred q; shfl.sync.down.b32 %0|q, %2, %3, %4, 0xffffffff; selp.u32 %1, 1, 0, q; }"
                         : "=r"(d), "=r"(p) : "r"(x), "r"(b), "r"(c));
            break;
        case xlane::kShflBfly:
            asm volatile("{ .reg .pred q; shfl.sync.bfly.b32 %0|q, %2, %3, %4, 0xffffffff; selp.u32 %1, 1, 0, q; }"
                         : "=r"(d), "=r"(p) : "r"(x), "r"(b), "r"(c));
            break;
        default:
            asm volatile("{ .reg .pred q; shfl.sync.idx.b32 %0|q, %2, %3, %4, 0xffffffff; selp.u32 %1, 1, 0, q; }"
                         : "=r"(d), "=r"(p) : "r"(x), "r"(b), "r"(c));
            break;
    }
    return d | ((u64)p << 32);
}

__device__ __forceinline__ void leg_shfl(Tally& T, u64 seed, unsigned it, bool lastit, unsigned w, unsigned l, unsigned inj_op,
                                         u64 m) {
#pragma unroll 1
    for (unsigned op = 0; op < CRO_XLANE_SHFL_OPS; ++op) {
        const xlane::Shfl s = xlane::shfl_op(op, l);
        const unsigned x = xlane::shfl_operand(seed, op, w, l) ^ (op == inj_op ? (unsigned)m : 0u);
        const u64 got = shfl(s.mode, x, s.b, s.c);
        bool p;
        const unsigned j = xlane::shfl_source(s, l, &p);
        T.check(it, lastit, op, j, xlane::shfl_operand(seed, op, w, j) | ((u64)p << 32), got);
    }
}

// ---- VOTE ----
__device__ __forceinline__ u64 vote(unsigned form, unsigned x) {
    unsigned d;
    switch (form) {
        case 0:
            asm volatile("{ .reg .pred q; setp.ne.u32 q, %1, 0; vote.sync.ballot.b32 %0, q, 0xffffffff; }" : "=r"(d) : "r"(x & 1u));
            break;
        case 1:
            asm volatile("{ .reg .pred q, r; setp.ne.u32 q, %1, 0; vote.sync.any.pred r, q, 0xffffffff; selp.u32 %0, 1, 0, r; }"
                         : "=r"(d) : "r"(x & 1u));
            break;
        case 2:
            asm volatile("{ .reg .pred q, r; setp.ne.u32 q, %1, 0; vote.sync.all.pred r, q, 0xffffffff; selp.u32 %0, 1, 0, r; }"
                         : "=r"(d) : "r"(x & 1u));
            break;
        default:
            asm volatile("{ .reg .pred q, r; setp.ne.u32 q, %1, 0; vote.sync.uni.pred r, q, 0xffffffff; selp.u32 %0, 1, 0, r; }"
                         : "=r"(d) : "r"(x & 1u));
            break;
    }
    return d;
}

__device__ __forceinline__ void leg_vote(Tally& T, u64 seed, unsigned it, bool lastit, unsigned w, unsigned l, unsigned inj_op,
                                         u64 m) {
#pragma unroll 1
    for (unsigned row = 0; row < CRO_XLANE_VOTE_OPS / xlane::kVoteForms; ++row) {
        const unsigned x = xlane::vote_operand(seed, row, w, l);
        const unsigned b = xlane::vote_ballot(seed, row, w);
#pragma unroll
        for (unsigned f = 0; f < xlane::kVoteForms; ++f) {
            const unsigned op = row * xlane::kVoteForms + f;
            T.check(it, lastit, op, xlane::kNoPeer, xlane::vote_result(f, b), vote(f, x ^ (op == inj_op ? (unsigned)m : 0u)));
        }
    }
}

// ---- MATCH ----
__device__ __forceinline__ u64 match(unsigned form, unsigned a, u64 b) {
    unsigned d, p = 0;
    switch (form) {
        case 0: asm volatile("match.any.sync.b32 %0, %1, 0xffffffff;" : "=r"(d) : "r"(a)); break;
        case 1:
            asm volatile("{ .reg .pred q; match.all.sync.b32 %0|q, %2, 0xffffffff; selp.u32 %1, 1, 0, q; }" : "=r"(d), "=r"(p) : "r"(a));
            break;
        case 2: asm volatile("match.any.sync.b64 %0, %1, 0xffffffff;" : "=r"(d) : "l"(b)); break;
        default:
            asm volatile("{ .reg .pred q; match.all.sync.b64 %0|q, %2, 0xffffffff; selp.u32 %1, 1, 0, q; }" : "=r"(d), "=r"(p) : "l"(b));
            break;
    }
    return d | ((u64)p << 32);
}

__device__ __forceinline__ void leg_match(Tally& T, u64 seed, unsigned it, bool lastit, unsigned w, unsigned l, unsigned inj_op,
                                          u64 m) {
#pragma unroll 1
    for (unsigned row = 0; row < CRO_XLANE_MATCH_OPS / xlane::kMatchForms; ++row) {
        const unsigned a = xlane::match_value32(seed, row, w, l);
        const u64 b = xlane::match_value64(seed, row, w, l);
        u64 e[4];
        xlane::match_results(seed, row, w, l, e);
#pragma unroll
        for (unsigned f = 0; f < xlane::kMatchForms; ++f) {
            const unsigned op = row * xlane::kMatchForms + f;
            const u64 mm = op == inj_op ? m : 0ull;
            T.check(it, lastit, op, xlane::kNoPeer, e[f], match(f, a ^ (unsigned)mm, b ^ mm));
        }
    }
}

// ---- REDUX ----
__device__ __forceinline__ unsigned redux(unsigned form, unsigned x) {
    unsigned d;
    switch (form) {
        case 0: asm volatile("redux.sync.add.u32 %0, %1, 0xffffffff;" : "=r"(d) : "r"(x)); break;
        case 1: asm volatile("redux.sync.add.s32 %0, %1, 0xffffffff;" : "=r"(d) : "r"(x)); break;
        case 2: asm volatile("redux.sync.min.u32 %0, %1, 0xffffffff;" : "=r"(d) : "r"(x)); break;
        case 3: asm volatile("redux.sync.max.u32 %0, %1, 0xffffffff;" : "=r"(d) : "r"(x)); break;
        case 4: asm volatile("redux.sync.min.s32 %0, %1, 0xffffffff;" : "=r"(d) : "r"(x)); break;
        case 5: asm volatile("redux.sync.max.s32 %0, %1, 0xffffffff;" : "=r"(d) : "r"(x)); break;
        case 6: asm volatile("redux.sync.and.b32 %0, %1, 0xffffffff;" : "=r"(d) : "r"(x)); break;
        case 7: asm volatile("redux.sync.or.b32 %0, %1, 0xffffffff;" : "=r"(d) : "r"(x)); break;
        default: asm volatile("redux.sync.xor.b32 %0, %1, 0xffffffff;" : "=r"(d) : "r"(x)); break;
    }
    return d;
}

__device__ __forceinline__ void leg_redux(Tally& T, u64 seed, unsigned it, bool lastit, unsigned w, unsigned l, unsigned inj_op,
                                          u64 m) {
    constexpr unsigned F = xlane::kReduxForms;
#pragma unroll 1
    for (unsigned row = 0; row < CRO_XLANE_REDUX_OPS / F; ++row) {
        const unsigned x = xlane::redux_operand(seed, row, w, l);
        unsigned acc[F];
        const unsigned x0 = xlane::redux_operand(seed, row, w, 0);
#pragma unroll
        for (unsigned f = 0; f < F; ++f) acc[f] = x0;
#pragma unroll 1
        for (unsigned j = 1; j < 32; ++j) {
            const unsigned y = xlane::redux_operand(seed, row, w, j);
#pragma unroll
            for (unsigned f = 0; f < F; ++f) xlane::redux_fold(f, &acc[f], y);
        }
#pragma unroll
        for (unsigned f = 0; f < F; ++f) {
            const unsigned op = row * F + f;
            T.check(it, lastit, op, xlane::kNoPeer, acc[f], redux(f, x ^ (op == inj_op ? (unsigned)m : 0u)));
        }
    }
}

// ---- ATOMS ----
__device__ __forceinline__ void st_u64(unsigned a, u64 v) { asm volatile("st.shared.u64 [%0], %1;" ::"r"(a), "l"(v) : "memory"); }
__device__ __forceinline__ u64 ld_u64(unsigned a) {
    u64 v;
    asm volatile("ld.shared.u64 %0, [%1];" : "=l"(v) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ void st_u8(unsigned a, unsigned v) { asm volatile("st.shared.u8 [%0], %1;" ::"r"(a), "r"(v) : "memory"); }
__device__ __forceinline__ unsigned ld_u8(unsigned a) {
    unsigned v;
    asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(a) : "memory");
    return v;
}
#define XL_ATOM32(op, type)                                                                                              \
    asm volatile("atom.shared." op "." type " %0, [%1], %2;" : "=r"(o32) : "r"(addr), "r"((unsigned)v) : "memory")

// One op of one kind for the whole CTA (every thread calls it; control flow is uniform but for the cas retries).
__device__ __forceinline__ void atoms_op(Tally& T, u64 seed, unsigned it, bool lastit, unsigned w, unsigned l, unsigned op,
                                         u64 m, unsigned arena) {
    using namespace xlane;
    const unsigned kind = op / kAtomsShapes, t = 32 * w + l;
    const AtomsShape s = atoms_shape(op % kAtomsShapes, w, l);
    const unsigned addr = arena + 8u * s.slot, pres = arena + 8u * kArenaWords + s.base;
    const u64 init = atoms_init(seed, op, s.group);
    if (s.rank == 0) st_u64(addr, init);
    st_u8(arena + 8u * kArenaWords + 2u * t, 0u);
    st_u8(arena + 8u * kArenaWords + 2u * t + 1u, 0u);
    __syncthreads();
    const bool wide = kind == kAtExch64 || kind == kAtCas64 || kind == kAtAdd64;
    const u64 v = (atoms_value(seed, op, w, l) ^ m) & (wide ? ~0ull : 0xFFFFFFFFull);
    unsigned o32 = 0;
    u64 o64 = 0;
    bool ok = true;
    switch (kind) {
        case kAtAdd: XL_ATOM32("add", "u32"); break;
        case kAtInc: XL_ATOM32("inc", "u32"); break;
        case kAtDec: XL_ATOM32("dec", "u32"); break;
        case kAtMinU: XL_ATOM32("min", "u32"); break;
        case kAtMaxU: XL_ATOM32("max", "u32"); break;
        case kAtMinS: XL_ATOM32("min", "s32"); break;
        case kAtMaxS: XL_ATOM32("max", "s32"); break;
        case kAtAnd: XL_ATOM32("and", "b32"); break;
        case kAtOr: XL_ATOM32("or", "b32"); break;
        case kAtXor: XL_ATOM32("xor", "b32"); break;
        case kAtExch: XL_ATOM32("exch", "b32"); break;
        case kAtExch64: asm volatile("atom.shared.exch.b64 %0, [%1], %2;" : "=l"(o64) : "r"(addr), "l"(v) : "memory"); break;
        case kAtAdd64: asm volatile("atom.shared.add.u64 %0, [%1], %2;" : "=l"(o64) : "r"(addr), "l"(v) : "memory"); break;
        case kAtCas: {
            unsigned want = (unsigned)init;
            ok = false;
            for (unsigned k = 0; k < kCasTries && !ok; ++k) {
                asm volatile("atom.shared.cas.b32 %0, [%1], %2, %3;" : "=r"(o32) : "r"(addr), "r"(want), "r"(want + (unsigned)v) : "memory");
                ok = o32 == want;
                want = o32;
            }
            break;
        }
        default: {   // kAtCas64
            u64 want = init;
            ok = false;
            for (unsigned k = 0; k < kCasTries && !ok; ++k) {
                asm volatile("atom.shared.cas.b64 %0, [%1], %2, %3;" : "=l"(o64) : "r"(addr), "l"(want), "l"(want + v) : "memory");
                ok = o64 == want;
                want = o64;
            }
            break;
        }
    }
    // tickets and exchanged values mark their presence slots with plain stores (bounded: a wrong value marks nothing)
    if (kind == kAtInc || kind == kAtDec) {
        const unsigned ticket = kind == kAtInc ? o32 - (unsigned)init : (unsigned)init - o32;
        if (ticket < s.n) st_u8(pres + ticket, 1u);
    } else if (kind == kAtExch || kind == kAtExch64) {
        const u64 idx = (kind == kAtExch ? (u64)o32 : o64) ^ init;
        if (idx <= s.n) st_u8(pres + (unsigned)idx, 1u);
    }
    __syncthreads();
    const u64 fin = ld_u64(addr) & (wide ? ~0ull : 0xFFFFFFFFull);
    if ((kind == kAtExch || kind == kAtExch64) && s.rank == 0 && (fin ^ init) <= s.n) st_u8(pres + (unsigned)(fin ^ init), 1u);
    __syncthreads();
    u64 got;
    if (kind == kAtExch || kind == kAtExch64) got = ld_u8(pres + s.rank + 1u);
    else if (kind == kAtInc || kind == kAtDec) got = (fin << 32) | ld_u8(pres + s.rank);
    else got = ok ? fin : ~fin & (wide ? ~0ull : 0xFFFFFFFFull);
    T.check(it, lastit, op, kNoPeer, atoms_result(seed, op, w, l), got);
    __syncthreads();                                    // every read done before the next op's words are set
}

__device__ __forceinline__ void leg_atoms(Tally& T, u64 seed, unsigned it, bool lastit, unsigned w, unsigned l, unsigned inj_op,
                                          u64 m, unsigned arena) {
#pragma unroll 1
    for (unsigned op = 0; op < CRO_XLANE_ATOMS_OPS; ++op) atoms_op(T, seed, it, lastit, w, l, op, op == inj_op ? m : 0ull, arena);
}

template <unsigned LEG>
__global__ void __launch_bounds__(kT, 1) xlane_kernel(const XlaneArgs a) {
    extern __shared__ __align__(16) unsigned char xlane_smem[];
    unsigned smid, nsmid;
    asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
    asm volatile("mov.u32 %0, %%nsmid;" : "=r"(nsmid));
    const unsigned t = threadIdx.x, w = t >> 5, l = t & 31u;
    const size_t me = (size_t)blockIdx.x * kT + t;
    const bool inj = a.inj_mask && (a.inj_sm < 0 || (unsigned)a.inj_sm == smid) && (a.inj_warp < 0 || (unsigned)a.inj_warp == w) &&
                     (a.inj_lane < 0 || (unsigned)a.inj_lane == l);
    const unsigned arena = (unsigned)__cvta_generic_to_shared(xlane_smem);
    Tally T;
    T.rec = a.rec + me * kR;
    T.leg = LEG;
    T.smid = smid;
    T.warp = w;
    T.lane = l;
    const unsigned long long t0 = lane_timer_ns();
    const long long k0 = clock64();
#pragma unroll 1
    for (unsigned it = 0; it < a.iterations; ++it) {
        const u64 seed = a.seed + it * kNonceStride;
        const bool lastit = it + 1 == a.iterations;
        const u64 m = inj && it == a.inj_iter ? a.inj_mask : 0ull;
        if (LEG == CRO_XLANE_LEG_SHFL) leg_shfl(T, seed, it, lastit, w, l, a.inj_op, m);
        if (LEG == CRO_XLANE_LEG_VOTE) leg_vote(T, seed, it, lastit, w, l, a.inj_op, m);
        if (LEG == CRO_XLANE_LEG_MATCH) leg_match(T, seed, it, lastit, w, l, a.inj_op, m);
        if (LEG == CRO_XLANE_LEG_REDUX) leg_redux(T, seed, it, lastit, w, l, a.inj_op, m);
        if (LEG == CRO_XLANE_LEG_ATOMS) leg_atoms(T, seed, it, lastit, w, l, a.inj_op, m, arena);
    }
    const long long k1 = clock64();
    const unsigned long long t1 = lane_timer_ns();
    T.publish(a.thr[me], a.cta, a.stamp, t0, t1, k0, k1, smid, nsmid);
}

template <unsigned LEG>
cudaError_t plan_leg() {
    return cudaFuncSetAttribute(xlane_kernel<LEG>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBytes);
}

}  // namespace

cudaError_t xlane_plan(int device, unsigned leg) {
    int optin = 0;
    cudaError_t e = cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device);
    if (e) return e;
    if ((size_t)optin < kSmemBytes) return cudaErrorInvalidConfiguration;
    switch (leg) {
        case CRO_XLANE_LEG_SHFL: return plan_leg<CRO_XLANE_LEG_SHFL>();
        case CRO_XLANE_LEG_VOTE: return plan_leg<CRO_XLANE_LEG_VOTE>();
        case CRO_XLANE_LEG_MATCH: return plan_leg<CRO_XLANE_LEG_MATCH>();
        case CRO_XLANE_LEG_REDUX: return plan_leg<CRO_XLANE_LEG_REDUX>();
        default: return plan_leg<CRO_XLANE_LEG_ATOMS>();
    }
}

cudaError_t launch_xlane(unsigned leg, const XlaneArgs& a, int grid, cudaStream_t st) {
    switch (leg) {
        case CRO_XLANE_LEG_SHFL: xlane_kernel<CRO_XLANE_LEG_SHFL><<<grid, kT, kSmemBytes, st>>>(a); break;
        case CRO_XLANE_LEG_VOTE: xlane_kernel<CRO_XLANE_LEG_VOTE><<<grid, kT, kSmemBytes, st>>>(a); break;
        case CRO_XLANE_LEG_MATCH: xlane_kernel<CRO_XLANE_LEG_MATCH><<<grid, kT, kSmemBytes, st>>>(a); break;
        case CRO_XLANE_LEG_REDUX: xlane_kernel<CRO_XLANE_LEG_REDUX><<<grid, kT, kSmemBytes, st>>>(a); break;
        default: xlane_kernel<CRO_XLANE_LEG_ATOMS><<<grid, kT, kSmemBytes, st>>>(a); break;
    }
    return cudaGetLastError();
}

}  // namespace cro
