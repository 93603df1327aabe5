// sweeps.cu — the single sweeps (tests, tuning, bench context: immediate seed, scratch slot) and the test hooks that
// run the verdict kernels and the chase on caller-given inputs (include/croprobe.h, cro_selftest_*).
#include "probe_internal.hpp"

namespace cro {

namespace {

// `iters` launches of `launch` between ev0 and ev1 on the device's stream, `enqueued` once they are all on it, then the
// scratch slot copied back and waited for, with the deadline (wait_stream) or without.  *out gets the bytes (`bytes`
// per launch), the variant, the event time, the slot's timer, its fold when `fold`, and the launch count.
template <class Launch, class Enqueued>
int timed_sweep(cro_ctx* c, Device* d, uint32_t iters, uint64_t bytes, uint32_t variant, Launch launch, Enqueued enqueued,
                bool fold, bool deadline, cro_sweep_result* out) {
    CU_TRY(c, cudaEventRecord(d->ev0, d->stream));
    for (uint32_t i = 0; i < iters; ++i) CU_TRY(c, launch());
    CU_TRY(c, cudaEventRecord(d->ev1, d->stream));
    c->launches += iters;
    enqueued();
    CU_TRY(c, cudaMemcpyAsync(&d->h_out[kSlotScratch], &d->d_out[kSlotScratch], sizeof(SweepOut), cudaMemcpyDeviceToHost,
                              d->stream));
    if (!deadline) CU_TRY(c, cudaStreamSynchronize(d->stream));
    else if (const int rc = wait_stream(c, d)) return rc;
    float ms = 0;
    CU_TRY(c, cudaEventElapsedTime(&ms, d->ev0, d->ev1));
    const SweepOut& s = d->h_out[kSlotScratch];
    memset(out, 0, sizeof *out);
    out->bytes = bytes * iters;
    out->ns = ms_to_ns(ms);
    out->timer_ns = s.t1 - s.t0;
    out->variant = variant;
    out->launches = iters;
    if (fold) {
        out->checksum_xor = s.x;
        out->checksum_sum = s.s;
        out->checksum_wsum = s.w;
    }
    return CRO_OK;
}

}  // namespace

int ctx_fill(cro_ctx* c, int idx, uint32_t iters, cro_sweep_result* out) {
    DeviceGuard g = enter_device(c, idx, out && iters);
    if (g.rc) return g.rc;
    Device* d = g.d;
    int rc = ensure_region(c, d);
    if (rc) return rc;
    auto fill = [&] { return launch_fill(d->plan, d->region, d->sweep_bytes, imm_params(d), d->scratch, &d->d_out[kSlotScratch], d->stream); };
    return timed_sweep(c, d, iters, d->sweep_bytes, 0, fill, [&] { half_a_filled(d); }, /*fold=*/false, /*deadline=*/true, out);
}

int ctx_read(cro_ctx* c, int idx, uint32_t variant, uint32_t iters, bool dst_half, cro_sweep_result* out) {
    DeviceGuard g = enter_device(c, idx, out && iters);
    if (g.rc) return g.rc;
    Device* d = g.d;
    variant = resolve_read_variant(variant, d->sweep_bytes, c->knobs);
    int rc = ensure_filled(c, d);
    if (rc) return rc;
    const unsigned char* base = d->region + (dst_half ? d->sweep_bytes : 0);
    auto read = [&] { return launch_read(d->plan, variant, base, d->sweep_bytes, imm_params(d), d->scratch, &d->d_out[kSlotScratch], d->stream); };
    return timed_sweep(c, d, iters, d->sweep_bytes, variant, read, [] {}, /*fold=*/true, /*deadline=*/true, out);
}

int ctx_copy(cro_ctx* c, int idx, uint32_t variant, uint32_t iters, cro_sweep_result* out) {
    variant = resolve_copy_variant(variant, c->knobs);
    DeviceGuard g = enter_device(c, idx, out && iters);
    if (g.rc) return g.rc;
    Device* d = g.d;
    int rc = ensure_filled(c, d);
    if (rc) return rc;
    CU_TRY(c, cudaMemsetAsync(&d->d_out[kSlotScratch], 0, sizeof(SweepOut), d->stream));
    auto copy = [&] {
        return launch_copy(d->plan, variant, d->region + d->sweep_bytes, d->region, d->sweep_bytes, imm_params(d), d->scratch,
                           &d->d_out[kSlotScratch], d->stream);
    };
    auto b_is_a = [&] {                               // B is a copy of A
        d->half_known[1] = d->half_known[0];
        d->half_seed[1] = d->half_seed[0];
    };
    // the fused copy folds the source as read; the plain copies fold nothing
    return timed_sweep(c, d, iters, 2 * d->sweep_bytes, variant, copy, b_is_a, variant == COPY_TMA_FUSED, /*deadline=*/true, out);
}

int ctx_expected(cro_ctx* c, int idx, cro_sweep_result* out) {
    DeviceGuard g = enter_device(c, idx, out != nullptr);
    if (g.rc) return g.rc;
    Device* d = g.d;
    auto expected = [&] { return launch_expected(d->plan, d->sweep_bytes, imm_params(d), d->scratch, &d->d_out[kSlotScratch], d->stream); };
    return timed_sweep(c, d, 1, 0, 0, expected, [] {}, /*fold=*/true, /*deadline=*/false, out);
}

int ctx_inject(cro_ctx* c, int idx, uint64_t word, uint64_t mask) {
    Device* d = dev_at(c, idx);
    DeviceGuard g = enter_device(c, idx, d && word < 2 * (d->sweep_bytes / 8));   // checked before the lock
    if (g.rc) return g.rc;
    int rc = ensure_filled(c, d);
    if (rc) return rc;
    CU_TRY(c, launch_xor_word(d->region, word, mask, d->stream));
    c->launches++;
    CU_TRY(c, cudaStreamSynchronize(d->stream));
    return CRO_OK;
}

int ctx_read_words(cro_ctx* c, int idx, uint64_t first, uint64_t n, uint64_t* out) {
    Device* d = dev_at(c, idx);
    if (!d || !out) return CRO_ERR_INVALID_ARG;
    const uint64_t limit = 2 * (d->sweep_bytes / 8);
    if (n > limit || first > limit - n) return CRO_ERR_INVALID_ARG;    // no wrap: first + n may not overflow
    if (n == 0) return CRO_OK;
    DeviceGuard g = enter_device(c, idx);
    if (g.rc) return g.rc;
    int rc = ensure_filled(c, d);
    if (rc) return rc;
    CU_TRY(c, cudaMemcpyAsync(out, d->region + first * 8, n * 8, cudaMemcpyDeviceToHost, d->stream));
    CU_TRY(c, cudaStreamSynchronize(d->stream));
    return CRO_OK;
}

// ---------------------------------------------------------------------------
// test hooks: the verdict kernels on caller-given inputs (include/croprobe.h)
// ---------------------------------------------------------------------------
int ctx_selftest_probe_finalize(cro_ctx* c, int idx, const cro_probe_result* tmpl, const cro_sweep_slot* slots,
                                const ProbeParams& pp, uint64_t sweep_bytes, uint32_t R, uint32_t C, uint32_t rv,
                                uint32_t cv, cro_probe_result* out) {
    DeviceGuard g = enter_device(c, idx, tmpl && slots && out && R <= (uint32_t)kMaxSweepsEach && C <= (uint32_t)kMaxSweepsEach);
    if (g.rc) return g.rc;
    Device* d = g.d;
    // [template | result | params | slots]
    constexpr size_t kRes = sizeof(cro_probe_result), kPar = 64, kSlots = sizeof(SweepOut) * kSlotCount;
    std::vector<unsigned char> h(2 * kRes + kPar + kSlots, 0);
    memcpy(h.data(), tmpl, kRes);
    memcpy(h.data() + 2 * kRes, &pp, sizeof pp);
    memcpy(h.data() + 2 * kRes + kPar, slots, kSlots);
    DeviceMem<unsigned char> base;
    CU_TRY(c, cudaMalloc(&base.p, h.size()));
    CU_TRY(c, cudaMemcpyAsync(base.p, h.data(), h.size(), cudaMemcpyHostToDevice, d->stream));
    CU_TRY(c, launch_finalize(finalize_args(reinterpret_cast<const cro_probe_result*>(base.p), reinterpret_cast<cro_probe_result*>(base.p + kRes),
                                            reinterpret_cast<const SweepOut*>(base.p + 2 * kRes + kPar),
                                            reinterpret_cast<const ProbeParams*>(base.p + 2 * kRes), sweep_bytes, R, C, rv, cv),
                              d->stream));
    CU_TRY(c, cudaMemcpyAsync(h.data(), base.p + kRes, kRes, cudaMemcpyDeviceToHost, d->stream));
    CU_TRY(c, cudaStreamSynchronize(d->stream));
    memcpy(out, h.data(), kRes);
    return CRO_OK;
}

int ctx_selftest_p2p_finalize(cro_ctx* c, int idx, cro_probe_result* result, const cro_sweep_slot* slots,
                              const cro_sweep_slot* const* peer_slots, const uint64_t* peer_stamp, const uint64_t* chase_out,
                              const uint32_t* chase_expect, uint32_t n, uint32_t self, uint32_t hops, uint32_t have_push,
                              uint32_t push_folded, uint64_t p2p_bytes, uint64_t stamp) {
    DeviceGuard g = enter_device(c, idx, result && slots && peer_slots && peer_stamp && chase_out && chase_expect && n <= CRO_MAX_DEVICES &&
                                             self < n);
    if (g.rc) return g.rc;
    Device* d = g.d;
    // [result | chase output | this device's slots | peer j's slots, for each j]
    constexpr size_t kRes = sizeof(cro_probe_result), kChase = kChaseOutWords * sizeof(unsigned long long);
    constexpr size_t kSlots = sizeof(SweepOut) * kSlotCount;
    std::vector<unsigned char> h(kRes + kChase + (1 + CRO_MAX_DEVICES) * kSlots, 0);
    memcpy(h.data(), result, kRes);
    memcpy(h.data() + kRes, chase_out, kChase);
    memcpy(h.data() + kRes + kChase, slots, kSlots);
    for (int j = 0; j < CRO_MAX_DEVICES; ++j)
        if (peer_slots[j]) memcpy(h.data() + kRes + kChase + (size_t)(1 + j) * kSlots, peer_slots[j], kSlots);
    DeviceMem<unsigned char> base;
    CU_TRY(c, cudaMalloc(&base.p, h.size()));
    CU_TRY(c, cudaMemcpyAsync(base.p, h.data(), h.size(), cudaMemcpyHostToDevice, d->stream));
    P2PFinalizeArgs pa{};
    pa.out = reinterpret_cast<cro_probe_result*>(base.p);
    pa.chase_out = reinterpret_cast<const unsigned long long*>(base.p + kRes);
    pa.slots = reinterpret_cast<const SweepOut*>(base.p + kRes + kChase);
    for (int j = 0; j < CRO_MAX_DEVICES; ++j) {
        if (peer_slots[j]) pa.peer_slots[j] = reinterpret_cast<const SweepOut*>(base.p + kRes + kChase + (size_t)(1 + j) * kSlots);
        pa.peer_stamp[j] = peer_stamp[j];
        pa.chase_expect[j] = chase_expect[j];
    }
    pa.n = n;
    pa.self = self;
    pa.hops = hops;
    pa.have_push = have_push;
    pa.push_folded = push_folded;
    pa.p2p_bytes = p2p_bytes;
    pa.stamp = stamp;
    CU_TRY(c, launch_p2p_finalize(pa, d->stream));
    CU_TRY(c, cudaMemcpyAsync(h.data(), base.p, kRes, cudaMemcpyDeviceToHost, d->stream));
    CU_TRY(c, cudaStreamSynchronize(d->stream));
    memcpy(result, h.data(), kRes);
    return CRO_OK;
}

int ctx_selftest_chase(cro_ctx* c, int idx, const int32_t* minor_src, const int32_t* minor_dst, uint32_t n, uint32_t hops,
                       uint64_t* out) {
    DeviceGuard g = enter_device(c, idx, minor_src && minor_dst && out && n != 0 && n <= CRO_MAX_DEVICES);
    if (g.rc) return g.rc;
    Device* d = g.d;
    DeviceMem<unsigned long long> tables[CRO_MAX_DEVICES], dout;
    CU_TRY(c, cudaMalloc(&dout.p, kChaseOutWords * sizeof(unsigned long long)));
    ChaseArgs ca{};
    ca.n = n;
    ca.hops = hops;
    std::vector<uint32_t> perm;
    for (uint32_t j = 0; j < n; ++j) {
        if (minor_src[j] < 0) continue;      // a null row: no table, the warp walks nothing
        chase_permutation(minor_src[j], minor_dst[j], &perm);
        const int rc = upload_chase_table(c, perm, &tables[j].p);
        if (rc) return rc;
        ca.table[j] = tables[j].p;
    }
    CU_TRY(c, arm_chase_out(dout.p, d->stream));
    CU_TRY(c, launch_chase(ca, dout.p, d->stream));
    CU_TRY(c, cudaMemcpyAsync(out, dout.p, 2 * (size_t)n * sizeof(unsigned long long), cudaMemcpyDeviceToHost, d->stream));
    CU_TRY(c, cudaStreamSynchronize(d->stream));
    return CRO_OK;
}

// ---------------------------------------------------------------------------
// test hook: one sweep kernel between guard bands (include/croprobe.h, cro_selftest_sweep)
// ---------------------------------------------------------------------------
namespace {

constexpr uint64_t kGuard = CRO_SELFTEST_GUARD_BYTES;
constexpr uint64_t kMaxHookBytes = 1ull << 40;
constexpr uint64_t kMaxHookWords = 1ull << 37;      // locate: word0 + interior words, so the granule bitmap stays small

uint64_t round_up(uint64_t v, uint64_t a) { return (v + a - 1) / a * a; }

bool is_copy(uint32_t k) { return k >= CRO_SELFTEST_SWEEP_COPY_LDG && k <= CRO_SELFTEST_SWEEP_COPY_FUSED; }
bool is_link(uint32_t k) { return k == CRO_SELFTEST_SWEEP_LINK_READ || k == CRO_SELFTEST_SWEEP_LINK_WRITE; }

// The hook's buffer: `total` bytes (a multiple of the guard), interior k at byte at[k].  Every interior starts `offset`
// past a guard boundary; what the interiors leave of [0, total) is guard, at least kGuard of it on each side.
struct HookLayout {
    uint64_t total = 0;
    uint64_t at[2] = {0, 0};
    int interiors = 1;
};

HookLayout hook_layout(const cro_selftest_sweep_opts& o) {
    HookLayout L;
    const uint64_t first = kGuard + o.offset;
    if (o.layout == CRO_SELFTEST_LAYOUT_APART) {
        L.interiors = 2;
        L.at[0] = first;
        L.at[1] = round_up(first + o.bytes, kGuard) + kGuard + o.offset;
        L.total = round_up(L.at[1] + o.bytes, kGuard) + kGuard;
    } else if (o.layout != 0) {
        L.interiors = 2;
        const int src = o.layout == CRO_SELFTEST_LAYOUT_SRC_DST ? 0 : 1;
        L.at[src] = first;
        L.at[1 - src] = first + o.bytes;
        L.total = round_up(first + 2 * o.bytes, kGuard) + kGuard;
    } else {
        L.at[0] = L.at[1] = first;
        L.total = round_up(first + o.bytes, kGuard) + kGuard;
    }
    return L;
}

// (start, bytes) of every guard, in buffer order (adjacent interiors have none between them).
std::vector<std::pair<uint64_t, uint64_t>> hook_guards(const HookLayout& L, uint64_t bytes) {
    uint64_t lo[2] = {std::min(L.at[0], L.at[1]), std::max(L.at[0], L.at[1])};
    std::vector<std::pair<uint64_t, uint64_t>> g;
    uint64_t from = 0;
    for (int k = 0; k < L.interiors; ++k) {
        if (lo[k] > from) g.push_back({from, lo[k] - from});
        from = lo[k] + bytes;
    }
    g.push_back({from, L.total - from});
    return g;
}

// Why the options are refused, or nullptr.
const char* hook_refusal(const cro_selftest_sweep_opts& o) {
    const uint32_t k = o.kernel;
    if (k < CRO_SELFTEST_SWEEP_FILL || k > CRO_SELFTEST_SWEEP_LINK_WRITE) return "unknown kernel";
    if (is_copy(k) ? (o.layout < CRO_SELFTEST_LAYOUT_SRC_DST || o.layout > CRO_SELFTEST_LAYOUT_APART) : o.layout != 0)
        return "a copy takes a layout and no other kernel does";
    if (o.offset % 16 || o.offset >= kGuard) return "the offset must be a multiple of 16 below the guard";
    if (o.bytes < 16 || o.bytes % 16 || o.bytes > kMaxHookBytes) return "the interior must be a multiple of 16 bytes in [16, 2^40]";
    const bool inverts = k == CRO_SELFTEST_SWEEP_FILL || k == CRO_SELFTEST_SWEEP_LOCATE;
    if (o.invert != 0 && !(inverts && o.invert == ~0ull)) return "invert is 0, or all ones for the fill and locate";
    if (k == CRO_SELFTEST_SWEEP_LOCATE ? o.word0 > kMaxHookWords - o.bytes / 8 : o.word0 != 0)
        return "word0 is locate's, with word0 + bytes / 8 at most 2^37";
    const uint64_t n = o.bytes / 8;
    for (int r = 0; r < 2; ++r) {
        if (!o.force_count[r]) continue;
        if (o.force_first[r] >= n || o.force_count[r] > n - o.force_first[r]) return "a force range must lie in the interior";
        if (k != CRO_SELFTEST_SWEEP_LOCATE && !(k == CRO_SELFTEST_SWEEP_FORCE_WORDS && r == 0))
            return "force ranges are locate's, and force_words' range 0";
    }
    if ((o.flags & ~CRO_SELFTEST_F_INTERIORS) || o.reserved) return "unknown flags";
    return nullptr;
}

// Mapped pinned host memory of one call, freed on every way out.
struct HostMem {
    void* p = nullptr;
    HostMem() = default;
    HostMem(const HostMem&) = delete;
    HostMem& operator=(const HostMem&) = delete;
    ~HostMem() { if (p) cudaFreeHost(p); }
};

}  // namespace

int ctx_selftest_sweep(cro_ctx* c, int idx, const cro_selftest_sweep_opts* o, cro_selftest_sweep_out* out, void* buf,
                       uint64_t cap_bytes, cro_fault_word* words, int cap, int* n_words) {
    if (out) memset(out, 0, sizeof *out);
    if (n_words) *n_words = 0;
    const char* why = !o || !out || !n_words || cap < 0 || (cap > 0 && !words) ? "null or negative argument" : hook_refusal(*o);
    HookLayout L;
    if (!why) {
        L = hook_layout(*o);
        out->buf_bytes = L.total;
        if (dev_at(c, idx) && cap_bytes < L.total) return CRO_ERR_BUFFER_SMALL;
        if (!buf) why = "null buffer";
    }
    if (why) c->set_error(std::string("cro_selftest_sweep: ") + why);
    DeviceGuard g = enter_device(c, idx, !why);
    if (g.rc) return g.rc;
    Device* d = g.d;
    const uint32_t kernel = o->kernel;
    const uint64_t bytes = o->bytes;
    const bool host = is_link(kernel);
    cudaStream_t st = d->stream;

    // the buffer, its guard boundaries 2 MiB-aligned (device memory, or mapped host memory for the link rows)
    DeviceMem<unsigned char> dmem;
    HostMem hmem;
    unsigned char* base = nullptr;       // device address
    unsigned char* hbase = nullptr;      // host address (link rows)
    if (host) {
        CU_TRY(c, cudaHostAlloc(&hmem.p, L.total + kGuard, cudaHostAllocMapped));
        void* dp = nullptr;
        CU_TRY(c, cudaHostGetDevicePointer(&dp, hmem.p, 0));
        const uint64_t skew = round_up((uint64_t)(uintptr_t)hmem.p, kGuard) - (uint64_t)(uintptr_t)hmem.p;
        hbase = static_cast<unsigned char*>(hmem.p) + skew;
        base = static_cast<unsigned char*>(dp) + skew;
    } else {
        CU_TRY(c, cudaMalloc(&dmem.p, L.total + kGuard));
        base = dmem.p + (round_up((uint64_t)(uintptr_t)dmem.p, kGuard) - (uint64_t)(uintptr_t)dmem.p);
    }
    // the kernel's counters, records and granule bitmap (one granule to spare past the interior, so a stray record there
    // shows), the interiors' folds after it, and the reduction scratch
    MismatchBuffer mb;
    const KernelPlan& p = d->plan;
    const int grid = std::max({p.read_ldg.grid, p.read_ldg256.grid, p.read_tma.grid, p.copy_fused.grid, p.locate.grid, p.link_grid, 1});
    const uint64_t covered = (kernel == CRO_SELFTEST_SWEEP_LOCATE ? o->word0 * 8 : 0) + bytes + CRO_LOCATE_GRANULE_BYTES;
    int rc = mb.ensure(c, 1, covered, 2, 0, grid, 1);
    if (rc || (rc = mb.zero(c, st))) return rc;
    const MismatchView dv = mb.dev();
    const SweepScratch& sc = mb.scratch[0];

    // guard g: the canary stream from word g * 2^32, so no guard repeats another's words (a stray copy from one guard
    // into the same place of the next shows); the interior: what the kernel's row asks for
    const Params pat{ProbeParams{o->seed, 0}, nullptr};
    const std::vector<std::pair<uint64_t, uint64_t>> guards = hook_guards(L, bytes);
    for (size_t gi = 0; gi < guards.size(); ++gi) {
        const Params canary{ProbeParams{o->canary + (gi << 32), 0}, nullptr};
        CU_TRY(c, launch_fill(p, base + guards[gi].first, guards[gi].second, canary, sc, nullptr, st));
        c->launches++;
    }
    // what the kernel reads holds the pattern (^ invert); what it writes holds the complement of what it should write,
    // so every word it misses shows
    unsigned char* in0 = base + L.at[0];
    unsigned char* in1 = base + L.at[1];
    const bool writes = kernel == CRO_SELFTEST_SWEEP_FILL || kernel == CRO_SELFTEST_SWEEP_LINK_WRITE;
    CU_TRY(c, launch_fill(p, in0, bytes, pat, sc, nullptr, st, (o->invert != 0) != writes));
    if (is_copy(kernel)) CU_TRY(c, launch_fill(p, in1, bytes, pat, sc, nullptr, st, true));
    c->launches += is_copy(kernel) ? 2 : 1;
    if (kernel == CRO_SELFTEST_SWEEP_LOCATE)
        for (int r = 0; r < 2; ++r) {
            CU_TRY(c, launch_force_words(in0, o->force_first[r], o->force_count[r], o->force_and[r], o->force_or[r], p.sm_count, st));
            c->launches += o->force_count[r] ? 1 : 0;
        }

    // the kernel, timed and waited for as the single sweeps are; a kernel that publishes no slot leaves it zero
    SweepOut* slot = &d->d_out[kSlotScratch];
    CU_TRY(c, cudaMemsetAsync(slot, 0, sizeof(SweepOut), st));
    const uint32_t rv = kernel - CRO_SELFTEST_SWEEP_READ_LDG + READ_LDG, cv = kernel - CRO_SELFTEST_SWEEP_COPY_LDG + COPY_LDG;
    const LinkRole off{nullptr, 0, 0, SweepScratch{}, nullptr, 0}, role{in0, bytes, o->seed, sc, slot, (unsigned)kLinkWarps};
    auto run = [&]() -> cudaError_t {
        switch (kernel) {
            case CRO_SELFTEST_SWEEP_FILL: return launch_fill(p, in0, bytes, pat, sc, slot, st, o->invert != 0);
            case CRO_SELFTEST_SWEEP_LOCATE: return launch_locate(p, in0, bytes, o->word0, o->seed, o->invert, dv.check(0), sc, slot, st);
            case CRO_SELFTEST_SWEEP_FORCE_WORDS:
                return launch_force_words(in0, o->force_first[0], o->force_count[0], o->force_and[0], o->force_or[0], p.sm_count, st);
            case CRO_SELFTEST_SWEEP_LINK_READ: return launch_link_stream(role, off, dv.check(0), p.link_grid, 0, st);
            case CRO_SELFTEST_SWEEP_LINK_WRITE: return launch_link_stream(off, role, dv.check(0), p.link_grid, 0, st);
            default: return is_copy(kernel) ? launch_copy(p, cv, in1, in0, bytes, pat, sc, slot, st) : launch_read(p, rv, in0, bytes, pat, sc, slot, st);
        }
    };
    const bool reads = kernel >= CRO_SELFTEST_SWEEP_READ_LDG && kernel <= CRO_SELFTEST_SWEEP_READ_LDG256;
    const bool fold = reads || kernel == CRO_SELFTEST_SWEEP_COPY_FUSED || kernel == CRO_SELFTEST_SWEEP_LOCATE ||
                      kernel == CRO_SELFTEST_SWEEP_LINK_READ;
    if ((rc = timed_sweep(c, d, 1, is_copy(kernel) ? 2 * bytes : bytes, reads ? rv : is_copy(kernel) ? cv : 0, run, [] {}, fold,
                          /*deadline=*/true, &out->sweep)))
        return rc;

    // each interior folded by the LDG read, the counters fetched, the guards (and interiors) copied back
    for (int k = 0; k < L.interiors; ++k) CU_TRY(c, launch_read(p, READ_LDG, base + L.at[k], bytes, pat, sc, &dv.slots[k], st));
    c->launches += L.interiors;
    if ((rc = mb.fetch(c, st))) return rc;
    std::vector<std::pair<uint64_t, uint64_t>> back = guards;
    if (o->flags & CRO_SELFTEST_F_INTERIORS)
        for (int k = 0; k < L.interiors; ++k) back.push_back({L.at[k], bytes});
    unsigned char* hbuf = static_cast<unsigned char*>(buf);
    if (!host)
        for (const auto& seg : back) CU_TRY(c, cudaMemcpyAsync(hbuf + seg.first, base + seg.first, seg.second, cudaMemcpyDeviceToHost, st));
    if ((rc = wait_stream(c, d))) return rc;
    if (host)
        for (const auto& seg : back) memcpy(hbuf + seg.first, hbase + seg.first, seg.second);

    const MismatchView hv = mb.host();
    for (int k = 0; k < 2; ++k) {
        const SweepOut& s = hv.slots[k < L.interiors ? k : 0];
        out->at[k] = L.at[k];
        out->after_xor[k] = s.x;
        out->after_sum[k] = s.s;
        out->after_wsum[k] = s.w;
    }
    out->mismatches = hv.ctr[0].mismatches;
    out->claims = hv.ctr[0].claims;
    for (uint64_t w = 0; w < hv.gran_words; ++w)
        for (unsigned long long bits = hv.gran[w]; bits; bits &= bits - 1) {
            const uint64_t gi = w * 64 + (uint64_t)__builtin_ctzll(bits);
            if (!out->granules++) out->granule_min = gi;
            out->granule_max = gi;
        }
    std::vector<cro_fault_word> rec;
    for (uint64_t j = 0; j < std::min<uint64_t>(hv.ctr[0].claims, kLocateRecords); ++j)
        rec.push_back(cro_fault_word{hv.rec[j].word, hv.rec[j].expected, hv.rec[j].actual, 1u, 0u});
    std::sort(rec.begin(), rec.end(), [](const cro_fault_word& a, const cro_fault_word& b) { return a.word_index < b.word_index; });
    *n_words = (int)std::min<size_t>(rec.size(), (size_t)cap);
    std::copy(rec.begin(), rec.begin() + *n_words, words);
    return CRO_OK;
}

}  // namespace cro
