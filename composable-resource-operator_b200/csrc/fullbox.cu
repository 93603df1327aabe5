// fullbox.cu — the full-box probe (cro_probe_all): every device's HBM probe at once, NVLink rounds chained by events,
// one NCCL all-gather; and the per-pair detail of the last one (cro_p2p_detail).
#include <dlfcn.h>

#include "probe_internal.hpp"

namespace cro {

int upload_chase_table(cro_ctx* c, const std::vector<uint32_t>& perm, unsigned long long** table) {
    std::vector<unsigned long long> wide(perm.begin(), perm.end());
    CU_TRY(c, cudaMalloc(table, (size_t)kChaseSlots * 128));
    CU_TRY(c, cudaMemset(*table, 0, (size_t)kChaseSlots * 128));
    CU_TRY(c, cudaMemcpy2D(*table, 128, wide.data(), 8, 8, kChaseSlots, cudaMemcpyHostToDevice));
    // the chase runs on a non-blocking stream, which does not wait for the legacy stream these copies went to
    CU_TRY(c, cudaStreamSynchronize(0));
    return CRO_OK;
}

namespace {

// Round-robin 1-factorisation of K_n (n even): n-1 rounds of n/2 disjoint pairs.
std::vector<std::vector<std::pair<int, int>>> one_factorisation(int n) {
    std::vector<std::vector<std::pair<int, int>>> rounds;
    if (n < 2) return rounds;
    const int m = (n % 2 == 0) ? n : n + 1;  // odd n: vertex m-1 is a bye
    for (int r = 0; r < m - 1; ++r) {
        std::vector<std::pair<int, int>> pairs;
        auto add = [&](int a, int b) { if (a < n && b < n) pairs.push_back({a, b}); };
        add(m - 1, r);
        for (int k = 1; k < m / 2; ++k) add((r + k) % (m - 1), (r - k + (m - 1)) % (m - 1));
        rounds.push_back(pairs);
    }
    return rounds;
}

int enable_peers(cro_ctx* c) {
    if (c->peers_enabled) return CRO_OK;
    const int n = (int)c->devs.size();
    for (int a = 0; a < n; ++a) {
        CU_TRY(c, cudaSetDevice(c->devs[a]->ordinal));
        for (int b = 0; b < n; ++b) {
            if (a == b) continue;
            int can = 0;
            CU_TRY(c, cudaDeviceCanAccessPeer(&can, c->devs[a]->ordinal, c->devs[b]->ordinal));
            if (!can) continue;
            cudaError_t e = cudaDeviceEnablePeerAccess(c->devs[b]->ordinal, 0);
            if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) {
                c->set_error(std::string("cudaDeviceEnablePeerAccess: ") + cudaGetErrorString(e));
                cudaGetLastError();
                return CRO_ERR_P2P;
            }
            cudaGetLastError();
        }
    }
    c->peers_enabled = true;
    for (int a = 0; a < n; ++a) {     // p2p_access goes into every device's identity template
        CU_TRY(c, cudaSetDevice(c->devs[a]->ordinal));
        int rc = stage_template(c, c->devs[(size_t)a].get());
        if (rc) return rc;
    }
    return CRO_OK;
}

// Latency permutations: device b holds, for every other device a, the Sattolo cycle a will chase through b's
// memory (slot i lives at table[i*16], one per 128-byte line), and a remembers where `hops` steps must end.
int ensure_chase(cro_ctx* c, uint32_t hops) {
    const int n = (int)c->devs.size();
    bool built = true;
    for (auto& d : c->devs) built = built && (int)d->d_chase_tables.size() == n && d->chase_hops_built == hops;
    if (built) return CRO_OK;
    Range nv(c, "cro.chase.build");
    std::vector<uint32_t> perm;
    for (int b = 0; b < n; ++b) {
        Device* owner = c->devs[(size_t)b].get();
        CU_TRY(c, cudaSetDevice(owner->ordinal));
        if ((int)owner->d_chase_tables.size() != n) owner->d_chase_tables.assign((size_t)n, nullptr);
        for (int a = 0; a < n; ++a) {
            if (a == b) continue;
            Device* chaser = c->devs[(size_t)a].get();
            const int ma = chaser->info.device_minor >= 0 ? chaser->info.device_minor : chaser->ordinal;
            const int mb = owner->info.device_minor >= 0 ? owner->info.device_minor : owner->ordinal;
            chase_permutation(ma, mb, &perm);
            if (!owner->d_chase_tables[(size_t)a]) {
                const int rc = upload_chase_table(c, perm, &owner->d_chase_tables[(size_t)a]);
                if (rc) return rc;
            }
            if ((int)chaser->chase_expect.size() != n) chaser->chase_expect.assign((size_t)n, 0u);
            uint32_t at = 0;
            for (uint32_t h = 0; h < hops; ++h) at = perm[at];
            chaser->chase_expect[(size_t)b] = at;
        }
    }
    for (auto& d : c->devs) d->chase_hops_built = hops;
    return CRO_OK;
}

int load_nccl(cro_ctx* c) {
    if (c->ncclAllGather) return CRO_OK;
    if (!c->nccl_lib) {
        const char* path = getenv("CRO_NCCL_PATH");
        if (path && strcmp(path, "off") == 0) {          // the host does not want NCCL in its process
            c->set_error("NCCL switched off (CRO_NCCL_PATH=off): host-side gather");
            return CRO_ERR_NCCL;
        }
        // 1. whatever NCCL the host process already carries (a torch host brings its own, newer than the system's:
        //    loading the system copy first would make the host's later import fail on a missing symbol)
        c->nccl_lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD | RTLD_LOCAL);
        // 2. an explicit path, 3. the system library — never RTLD_GLOBAL: our copy must not answer anyone else's symbols
        if (!c->nccl_lib) {
            const char* extra = getenv("CRO_NCCL_PATH");
            if (extra && *extra) c->nccl_lib = dlopen(extra, RTLD_NOW | RTLD_LOCAL);
        }
        if (!c->nccl_lib) c->nccl_lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_LOCAL);
        if (!c->nccl_lib) c->nccl_lib = dlopen("libnccl.so", RTLD_NOW | RTLD_LOCAL);
        if (!c->nccl_lib) {
            c->set_error("libnccl.so.2 not found (set CRO_NCCL_PATH)");
            return CRO_ERR_NCCL;
        }
    }
    c->ncclCommInitAll = (int (*)(void**, int, const int*))dlsym(c->nccl_lib, "ncclCommInitAll");
    c->ncclGroupStart = (int (*)())dlsym(c->nccl_lib, "ncclGroupStart");
    c->ncclGroupEnd = (int (*)())dlsym(c->nccl_lib, "ncclGroupEnd");
    c->ncclGetErrorString = (const char* (*)(int))dlsym(c->nccl_lib, "ncclGetErrorString");
    auto ag = (int (*)(const void*, void*, size_t, int, void*, cudaStream_t))dlsym(c->nccl_lib, "ncclAllGather");
    if (!c->ncclCommInitAll || !c->ncclGroupStart || !c->ncclGroupEnd || !ag) {
        c->set_error("libnccl lacks a required symbol");
        return CRO_ERR_NCCL;
    }
    c->ncclAllGather = ag;
    return CRO_OK;
}

}  // namespace

// One call = the full-box probe (BASELINE config 3).  Everything is ENQUEUED first — per-device probe graphs,
// the NVLink rounds chained across devices by events, the device-side verdicts, the all-gather, the copy-back —
// and only then does the host wait, once per device.
int ctx_probe_all(cro_ctx* c, cro_probe_result* out, int cap, int* n_out) {
    if (!c || !out || !n_out) return CRO_ERR_INVALID_ARG;
    const int n = (int)c->devs.size();
    *n_out = n;
    if (cap < n) return CRO_ERR_BUFFER_SMALL;
    if (n == 0) return CRO_OK;
    std::lock_guard<std::mutex> all(c->all_mu);
    const cro_opts& o = c->opts;
    Range nv_all(c, "cro.probe_all");
    const uint64_t t_call = now_ns();
    c->fullbox = FullBoxTimes{};
    uint32_t host_syncs = 0;

    std::vector<std::unique_lock<std::mutex>> locks;
    for (int i = 0; i < n; ++i) locks.emplace_back(c->devs[(size_t)i]->mu);
    for (int i = 0; i < n; ++i) {
        Device* d = c->devs[(size_t)i].get();
        drain_pending(c, d);
        d->done.clear();
        d->lane_head = 0;
    }
    const bool p2p = n > 1 && !(o.flags & CRO_F_SKIP_P2P);
    const bool push = p2p && !(o.flags & CRO_F_SKIP_P2P_WRITE);
    bool use_nccl = n > 1 && !(o.flags & CRO_F_SKIP_NCCL);
    bool nccl_degraded = false;
    int rc;
    // one-time setup (peer mappings, latency tables, communicators) happens BEFORE anything is enqueued
    if (p2p) {
        if ((rc = enable_peers(c))) return rc;
        if ((rc = ensure_chase(c, o.latency_hops))) return rc;
    }
    if (use_nccl && load_nccl(c) != CRO_OK) {
        // no usable libnccl in reach: the structs still come back, per device over pinned memory ("replicas only",
        // SURVEY.md §8e) — the call says so (cro_fullbox_time.gather, last error) instead of failing the attach
        use_nccl = false;
        nccl_degraded = true;
    }
    if (use_nccl) {
        if (!c->nccl_ready) {
            Range nv(c, "cro.nccl.init");
            std::vector<int> ords;
            for (auto& d : c->devs) ords.push_back(d->ordinal);
            c->nccl_comms.assign((size_t)n, nullptr);
            int r = c->ncclCommInitAll(c->nccl_comms.data(), n, ords.data());
            if (r != 0) {
                c->set_error(std::string("ncclCommInitAll: ") + (c->ncclGetErrorString ? c->ncclGetErrorString(r) : "error"));
                return CRO_ERR_NCCL;
            }
            c->nccl_ready = true;
        }
    }
    const auto rounds = p2p ? one_factorisation(n) : std::vector<std::vector<std::pair<int, int>>>();
    for (int i = 0; i < n && p2p; ++i) {
        Device* d = c->devs[(size_t)i].get();
        CU_TRY(c, cudaSetDevice(d->ordinal));
        while (d->ev_push_done.size() < rounds.size()) {
            cudaEvent_t e1, e2;
            CU_TRY(c, cudaEventCreateWithFlags(&e1, cudaEventDisableTiming));
            CU_TRY(c, cudaEventCreateWithFlags(&e2, cudaEventDisableTiming));
            d->ev_push_done.push_back(e1);
            d->ev_reread_done.push_back(e2);
        }
    }

    // ---- phase 1: every device's HBM probe, one graph launch each ---------------------------------------
    {
        Range nv(c, "cro.probe_all.hbm");
        for (int i = 0; i < n; ++i) {
            Device* d = c->devs[(size_t)i].get();
            if ((rc = probe_enqueue(c, d, d->lanes[0]))) return rc;
            if (p2p) {
                // what this device's first p2p_bytes must fold to, for the peers that will read them
                CU_TRY(c, launch_expected(d->plan, std::min<uint64_t>(o.p2p_bytes, d->sweep_bytes), imm_params(d), d->scratch_pfx,
                                          &d->d_out[kSlotPrefix], d->aux));
                c->launches++;
                CU_TRY(c, cudaEventRecord(d->ev_aux_done, d->aux));
                CU_TRY(c, cudaStreamWaitEvent(d->stream, d->ev_aux_done, 0));
                CU_TRY(c, cudaEventRecord(d->ev_hbm_done, d->stream));
            }
        }
    }

    // ---- phase 2: NVLink rounds, 1-factorised so each GPU is in exactly one pair per round ----------------
    // Per round and device (partner p):  [wait p's HBM phase, p's previous re-read]  READ p's half A over the
    // link -> PUSH my prefix into p's half B -> [wait p's push]  RE-READ my own half B locally.  Both directions
    // of a pair run at once; nothing waits on the host.
    const bool unidir = c->knobs.get("CRO_P2P_UNIDIR") != 0;
    const unsigned rvp = c->knobs.get("CRO_P2P_READ_VARIANT"), wvp = c->knobs.get("CRO_P2P_WRITE_VARIANT");
    auto pair_ok = [&](int a, int b) { return a < 8 && b < 8 && c->devs[(size_t)a]->tmpl.p2p_access[b]; };
    auto push_bytes = [&](const Device* a, const Device* b) {
        return std::min<uint64_t>(std::min<uint64_t>(o.p2p_bytes, a->sweep_bytes), b->sweep_bytes);
    };
    if (p2p) {
        Range nv(c, "cro.probe_all.nvlink");
        for (size_t r = 0; r < rounds.size(); ++r) {
            std::vector<std::pair<int, int>> directed;
            for (const auto& p : rounds[r]) {
                directed.push_back({p.first, p.second});
                // CRO_P2P_UNIDIR=1 (measurement only, tools/p2p_variants.py): one direction per pair, to see what the
                // link gives when its other half is idle; the reverse direction's result slots stay zero
                if (!unidir) directed.push_back({p.second, p.first});
            }
            for (const auto& pr : directed) {                       // stage A: read + push
                Device* a = c->devs[(size_t)pr.first].get();
                Device* b = c->devs[(size_t)pr.second].get();
                if (!pair_ok(pr.first, pr.second)) continue;
                CU_TRY(c, cudaSetDevice(a->ordinal));
                CU_TRY(c, cudaStreamWaitEvent(a->stream, b->ev_hbm_done, 0));
                if (r > 0) CU_TRY(c, cudaStreamWaitEvent(a->stream, b->ev_reread_done[r - 1], 0));
                // TMA bulk copies straight out of the peer's HBM (cp.async.bulk on the peer-mapped address) into
                // this GPU's shared memory, checksummed as they land
                CU_TRY(c, launch_read(a->plan, rvp, b->region, std::min<uint64_t>(o.p2p_bytes, b->sweep_bytes), imm_params(a),
                                      a->scratch, &a->d_out[kSlotP2P0 + 3 * pr.second], a->stream));
                c->launches++;
                if (push) {
                    // posted NVLink writes: a streams its own prefix through shared memory (bulk load from local
                    // HBM, bulk store to the peer-mapped address, folded on the way) into half B of b's region
                    CU_TRY(c, launch_copy(a->plan, wvp, b->region + b->sweep_bytes, a->region, push_bytes(a, b), imm_params(a),
                                          a->scratch, &a->d_out[kSlotP2P0 + 3 * pr.second + 1], a->stream));
                    c->launches++;
                }
                CU_TRY(c, cudaEventRecord(a->ev_push_done[r], a->stream));
            }
            for (const auto& pr : directed) {                       // stage B: the receiver checks what landed
                Device* a = c->devs[(size_t)pr.first].get();          // pusher
                Device* b = c->devs[(size_t)pr.second].get();         // receiver
                if (!pair_ok(pr.first, pr.second)) continue;
                CU_TRY(c, cudaSetDevice(b->ordinal));
                if (push) {
                    b->half_known[1] = false;                        // its prefix now holds a's pattern
                    CU_TRY(c, cudaStreamWaitEvent(b->stream, a->ev_push_done[r], 0));
                    CU_TRY(c, launch_read(b->plan, resolve_read_variant(CRO_READ_AUTO, push_bytes(a, b), c->knobs), b->region + b->sweep_bytes,
                                          push_bytes(a, b), imm_params(b), b->scratch, &b->d_out[kSlotP2P0 + 3 * pr.first + 2], b->stream));
                    c->launches++;
                }
                CU_TRY(c, cudaEventRecord(b->ev_reread_done[r], b->stream));
            }
            if (unidir)   // the idle direction's devices still have to publish their round events
                for (const auto& p : rounds[r]) {
                    Device* b = c->devs[(size_t)p.second].get();
                    CU_TRY(c, cudaSetDevice(b->ordinal));
                    CU_TRY(c, cudaEventRecord(b->ev_push_done[r], b->stream));
                    Device* a = c->devs[(size_t)p.first].get();
                    CU_TRY(c, cudaSetDevice(a->ordinal));
                    CU_TRY(c, cudaEventRecord(a->ev_reread_done[r], a->stream));
                }
        }
        // latency: every device chases all its peers at once (one warp per peer, one load in flight each),
        // after EVERY device has finished its bandwidth legs so the links are quiet
        for (int i = 0; i < n; ++i) {
            Device* d = c->devs[(size_t)i].get();
            CU_TRY(c, cudaSetDevice(d->ordinal));
            CU_TRY(c, cudaEventRecord(d->ev_chase_ready, d->stream));
        }
        for (int i = 0; i < n; ++i) {
            Device* d = c->devs[(size_t)i].get();
            CU_TRY(c, cudaSetDevice(d->ordinal));
            ChaseArgs ca{};
            ca.n = (unsigned)n;
            ca.hops = o.latency_hops;
            for (int j = 0; j < n; ++j) {
                if (j == i || !pair_ok(i, j)) continue;
                CU_TRY(c, cudaStreamWaitEvent(d->stream, c->devs[(size_t)j]->ev_chase_ready, 0));
                ca.table[j] = c->devs[(size_t)j]->d_chase_tables[(size_t)i];
            }
            CU_TRY(c, arm_chase_out(d->d_chase_out, d->stream));   // a row the chase does not walk cannot pass
            CU_TRY(c, launch_chase(ca, d->d_chase_out, d->stream));
            c->launches++;
            P2PFinalizeArgs pa{};
            pa.out = d->d_result;
            pa.slots = d->d_out;
            pa.chase_out = d->d_chase_out;
            pa.n = (unsigned)n;
            pa.self = (unsigned)i;
            pa.hops = o.latency_hops;
            pa.have_push = (push && !unidir) ? 1u : 0u;
            pa.push_folded = wvp == COPY_TMA_FUSED ? 1u : 0u;   // the plain copies land bytes but fold nothing: only the receiver checks
            pa.p2p_bytes = o.p2p_bytes;
            pa.stamp = d->nonce_cur;
            for (int j = 0; j < n; ++j) {
                if (j == i || !pair_ok(i, j)) continue;
                pa.peer_slots[j] = c->devs[(size_t)j]->d_out;
                pa.peer_stamp[j] = c->devs[(size_t)j]->nonce_cur;
                pa.chase_expect[j] = d->chase_expect[(size_t)j];
            }
            if (unidir)     // measurement mode: only the pairs' first devices read; check nothing that did not run
                for (const auto& rd : rounds)
                    for (const auto& p : rd)
                        if (p.second == i) pa.peer_slots[p.first] = nullptr;
            CU_TRY(c, launch_p2p_finalize(pa, d->stream));
            c->launches++;
            CU_TRY(c, cudaMemcpyAsync(d->h_chase_out, d->d_chase_out, 2 * CRO_MAX_DEVICES * sizeof(unsigned long long), cudaMemcpyDeviceToHost, d->stream));
            CU_TRY(c, cudaMemcpyAsync(d->h_out, d->d_out, sizeof(SweepOut) * kSlotCount, cudaMemcpyDeviceToHost, d->stream));
        }
    }

    // ---- phase 3: ONE all-gather of the 512-byte structs, enqueued behind the verdict kernels ---------------
    if (use_nccl) {
        Range nv(c, "cro.probe_all.allgather");
        CU_TRY(c, cudaSetDevice(c->devs[0]->ordinal));
        CU_TRY(c, cudaEventRecord(c->devs[0]->ev0, c->devs[0]->stream));
        int r = c->ncclGroupStart();
        for (int i = 0; r == 0 && i < n; ++i) {
            Device* d = c->devs[(size_t)i].get();
            r = c->ncclAllGather(d->d_result, d->d_gather, sizeof(cro_probe_result), /*ncclUint8*/ 1,
                                 c->nccl_comms[(size_t)i], d->stream);
        }
        int r2 = c->ncclGroupEnd();
        if (r != 0 || r2 != 0) {
            c->set_error(std::string("ncclAllGather: ") + (c->ncclGetErrorString ? c->ncclGetErrorString(r ? r : r2) : "error"));
            return CRO_ERR_NCCL;
        }
        CU_TRY(c, cudaSetDevice(c->devs[0]->ordinal));
        CU_TRY(c, cudaEventRecord(c->devs[0]->ev1, c->devs[0]->stream));
        for (int i = 0; i < n; ++i) {
            Device* d = c->devs[(size_t)i].get();
            CU_TRY(c, cudaSetDevice(d->ordinal));
            CU_TRY(c, cudaMemcpyAsync(d->h_gather, d->d_gather, sizeof(cro_probe_result) * (size_t)n, cudaMemcpyDeviceToHost, d->stream));
        }
    } else {
        for (int i = 0; i < n; ++i) {
            Device* d = c->devs[(size_t)i].get();
            CU_TRY(c, cudaSetDevice(d->ordinal));
            CU_TRY(c, cudaMemcpyAsync(d->h_result, d->d_result, sizeof(cro_probe_result), cudaMemcpyDeviceToHost, d->stream));
        }
    }
    c->fullbox.enqueue_ns = now_ns() - t_call;

    // While the GPUs work: a fresh ECC read per device (NVML, milliseconds each — on the critical path it would cost the
    // box more than the NVLink rounds of one pair, and eight of them can outlast the GPUs' own work, so a device is
    // asked at most once a second).  The structs being gathered right now carry the count staged before this call; a
    // count that moved is staged for the next probe, and a FAILING probe re-reads it at once anyway.
    std::vector<int> restage;
    if (n > 1) {
        const auto t_now = std::chrono::steady_clock::now();
        for (int i = 0; i < n; ++i) {
            Device* d = c->devs[(size_t)i].get();
            if (t_now - d->ecc_at < std::chrono::seconds(1)) continue;
            d->ecc_at = t_now;
            refresh_ecc(c, d);
            if (d->tmpl.ecc_errors != d->ecc_uncorrected) restage.push_back(i);
        }
    }

    // ---- the only host waits: one per device ------------------------------------------------------------------
    {
        Range nv(c, "cro.probe_all.wait");
        for (int i = 0; i < n; ++i) {
            Device* d = c->devs[(size_t)i].get();
            CU_TRY(c, cudaSetDevice(d->ordinal));
            if ((rc = wait_stream(c, d))) return rc;
            ++host_syncs;
        }
    }
    for (int i = 0; i < n; ++i) {
        c->devs[(size_t)i]->lanes[0].in_flight = false;
        c->devs[(size_t)i]->last_lane = 0;
    }
    int worst = CRO_OK;
    if (use_nccl) {
        for (int i = 1; i < n; ++i)
            if (memcmp(c->devs[0]->h_gather, c->devs[(size_t)i]->h_gather, sizeof(cro_probe_result) * (size_t)n) != 0) {
                c->set_error("all-gather result differs between rank 0 and rank " + std::to_string(i));
                return CRO_ERR_NCCL;
            }
        memcpy(out, c->devs[0]->h_gather, sizeof(cro_probe_result) * (size_t)n);
        float ms = 0;
        CU_TRY(c, cudaSetDevice(c->devs[0]->ordinal));
        if (cudaEventElapsedTime(&ms, c->devs[0]->ev0, c->devs[0]->ev1) == cudaSuccess) c->fullbox.gather_ns = ms_to_ns(ms);
    } else {
        for (int i = 0; i < n; ++i) out[i] = *c->devs[(size_t)i]->h_result;
    }
    c->m_fullbox++;
    for (int i = 0; i < n; ++i) {
        Device* d = c->devs[(size_t)i].get();
        *d->h_result = out[i];
        d->last = out[i];
        d->have_last = true;
        c->m_probes++;
        if (out[i].status != CRO_OK) c->m_probe_failures++;
        if (out[i].status != CRO_OK) {
            worst = out[i].status;
            c->set_error(describe_failure(d, out[i]));
        }
        c->fullbox.hbm_ns = std::max<uint64_t>(c->fullbox.hbm_ns, out[i].total_ns);
        if (p2p) {
            unsigned long long lo = ~0ull, hi = 0;
            for (int j = 0; j < n; ++j) {
                if (j == i) continue;
                for (int k = 0; k < 3; ++k) {
                    const SweepOut& s = d->h_out[kSlotP2P0 + 3 * j + k];
                    if (s.stamp != d->nonce_cur) continue;
                    lo = std::min(lo, s.t0);
                    hi = std::max(hi, s.t1);
                }
                if (pair_ok(i, j))      // the rows of peers it cannot reach keep the armed value
                    c->fullbox.chase_ns = std::max<uint64_t>(c->fullbox.chase_ns, d->h_chase_out[2 * j + 1]);
            }
            if (hi > lo) c->fullbox.p2p_ns = std::max<uint64_t>(c->fullbox.p2p_ns, hi - lo);
        }
    }
    for (int i : restage) {
        Device* d = c->devs[(size_t)i].get();
        CU_TRY(c, cudaSetDevice(d->ordinal));
        if ((rc = stage_template(c, d))) return rc;
    }
    c->fullbox.rounds = (uint32_t)rounds.size();
    c->fullbox.host_syncs = host_syncs;
    c->fullbox.gather = use_nccl ? CRO_GATHER_NCCL : nccl_degraded ? CRO_GATHER_DEGRADED : CRO_GATHER_HOST;
    c->fullbox.wall_ns = now_ns() - t_call;
    return worst;
}

int ctx_p2p_detail(cro_ctx* c, int idx, int peer, cro_p2p_detail* out) {
    Device* d = dev_at(c, idx);
    Device* p = dev_at(c, peer);
    if (!d || !p || !out || idx == peer) return CRO_ERR_INVALID_ARG;
    std::lock_guard<std::mutex> all(c->all_mu);
    memset(out, 0, sizeof *out);
    const SweepOut& rd = d->h_out[kSlotP2P0 + 3 * peer];
    const SweepOut& ps = d->h_out[kSlotP2P0 + 3 * peer + 1];
    const SweepOut& landed = p->h_out[kSlotP2P0 + 3 * idx + 2];   // the peer's re-read of what this device pushed
    const SweepOut& want = p->h_out[kSlotPrefix];
    if (rd.stamp == d->nonce_cur) {
        out->read_ns = rd.t1 - rd.t0;
        out->read_xor = rd.x; out->read_sum = rd.s; out->read_wsum = rd.w;
    }
    if (ps.stamp == d->nonce_cur) out->push_ns = ps.t1 - ps.t0;
    if (landed.stamp == p->nonce_cur) {
        out->reread_ns = landed.t1 - landed.t0;
        out->landed_xor = landed.x; out->landed_sum = landed.s; out->landed_wsum = landed.w;
    }
    if (want.stamp == p->nonce_cur) { out->expect_xor = want.x; out->expect_sum = want.s; out->expect_wsum = want.w; }
    out->chase_end = (uint32_t)d->h_chase_out[2 * peer];
    out->chase_ns = d->h_chase_out[2 * peer + 1];
    out->chase_expect = (size_t)peer < d->chase_expect.size() ? d->chase_expect[(size_t)peer] : 0;
    out->hops = c->opts.latency_hops;
    out->access = idx < 8 && peer < 8 ? d->tmpl.p2p_access[peer] : 0;
    return CRO_OK;
}

}  // namespace cro
