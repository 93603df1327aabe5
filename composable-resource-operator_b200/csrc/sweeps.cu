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

}  // namespace cro
