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

// One stream operation of the full-box plan, and one device's p2p_finalize arguments other than pointers;
// cro_p2p_op and cro_p2p_finalize_plan are their public mirrors (cro_selftest_p2p_plan hands them over as they are).
struct P2POp {
    uint8_t kind, dev, peer, event;   // CRO_P2P_OP_*, the stream's device, the other device, CRO_P2P_EV_*
    uint16_t round, slot;
    uint64_t bytes;
};
struct P2PFinalizePlan {
    uint32_t n, self, have_push, push_folded;
    uint64_t p2p_bytes;
    uint32_t peer_mask, chase_mask;
};
static_assert(sizeof(cro_p2p_op) == sizeof(P2POp) && offsetof(cro_p2p_op, kind) == offsetof(P2POp, kind) &&
                  offsetof(cro_p2p_op, dev) == offsetof(P2POp, dev) && offsetof(cro_p2p_op, peer) == offsetof(P2POp, peer) &&
                  offsetof(cro_p2p_op, event) == offsetof(P2POp, event) && offsetof(cro_p2p_op, round) == offsetof(P2POp, round) &&
                  offsetof(cro_p2p_op, slot) == offsetof(P2POp, slot) && offsetof(cro_p2p_op, bytes) == offsetof(P2POp, bytes),
              "cro_p2p_op mirrors P2POp");
static_assert(sizeof(cro_p2p_finalize_plan) == sizeof(P2PFinalizePlan) &&
                  offsetof(cro_p2p_finalize_plan, n) == offsetof(P2PFinalizePlan, n) &&
                  offsetof(cro_p2p_finalize_plan, self) == offsetof(P2PFinalizePlan, self) &&
                  offsetof(cro_p2p_finalize_plan, have_push) == offsetof(P2PFinalizePlan, have_push) &&
                  offsetof(cro_p2p_finalize_plan, push_folded) == offsetof(P2PFinalizePlan, push_folded) &&
                  offsetof(cro_p2p_finalize_plan, p2p_bytes) == offsetof(P2PFinalizePlan, p2p_bytes) &&
                  offsetof(cro_p2p_finalize_plan, peer_mask) == offsetof(P2PFinalizePlan, peer_mask) &&
                  offsetof(cro_p2p_finalize_plan, chase_mask) == offsetof(P2PFinalizePlan, chase_mask),
              "cro_p2p_finalize_plan mirrors P2PFinalizePlan");
static_assert(sizeof(cro_p2p_plan) == 66336 && offsetof(cro_p2p_plan, fin) == 288 && offsetof(cro_p2p_plan, op) == 800,
              "cro_p2p_plan layout");

struct P2PPlan {
    uint64_t p2p_bytes = 0;                                 // P: every leg's bytes, the prefix's and the finalize's
    std::vector<std::vector<std::pair<int, int>>> rounds;
    std::vector<P2POp> ops;                                 // in enqueue order; a wait binds to the last record before it
    P2PFinalizePlan fin[CRO_MAX_DEVICES] = {};
};

// The full-box probe's schedule (include/croprobe.h, cro_selftest_p2p_plan, states the rules): a pure function of the
// device count, each device's S after degradation, the options and the access rows (access[8 * i + j]).
P2PPlan make_p2p_plan(int n, const uint64_t* sweep_bytes, uint64_t p2p_bytes, const uint8_t* access, uint32_t flags, bool unidir,
                      uint32_t write_variant) {
    P2PPlan p;
    const bool nvlink = n > 1 && !(flags & CRO_F_SKIP_P2P);
    const bool push = nvlink && !(flags & CRO_F_SKIP_P2P_WRITE);
    auto op = [&](uint8_t kind, int dev, int peer, uint8_t event, size_t round, int slot, uint64_t bytes) {
        p.ops.push_back(P2POp{kind, (uint8_t)dev, (uint8_t)peer, event, (uint16_t)round, (uint16_t)slot, bytes});
    };
    if (nvlink) {
        // one prefix for the whole call: a pair of unequal sizes would otherwise move, fold and expect different lengths
        p.p2p_bytes = p2p_bytes;
        for (int i = 0; i < n; ++i) p.p2p_bytes = std::min(p.p2p_bytes, sweep_bytes[i]);
    }
    const uint64_t P = p.p2p_bytes;
    for (int i = 0; i < n; ++i) {
        op(CRO_P2P_OP_HBM, i, i, 0, 0, 0, 0);
        if (!nvlink) continue;
        op(CRO_P2P_OP_PREFIX, i, i, 0, 0, kSlotPrefix, P);
        op(CRO_P2P_OP_RECORD, i, i, CRO_P2P_EV_HBM, 0, 0, 0);
    }
    if (!nvlink) return p;
    // a pair is scheduled only when both directions are reachable: one-way access would leave a push unchecked
    auto linked = [&](int a, int b) { return a < 8 && b < 8 && access[8 * a + b] && access[8 * b + a]; };
    p.rounds = one_factorisation(n);
    for (size_t r = 0; r < p.rounds.size(); ++r) {
        std::vector<std::pair<int, int>> directed;
        for (const auto& pr : p.rounds[r]) {
            if (!linked(pr.first, pr.second)) continue;
            directed.push_back(pr);
            // CRO_P2P_UNIDIR=1 (measurement only, tools/p2p_variants.py): one direction per pair, to see what the link
            // gives when its other half is idle; the reverse direction's result slots stay zero
            if (!unidir) directed.push_back({pr.second, pr.first});
        }
        for (const auto& [a, b] : directed) {                   // stage A: read + push
            op(CRO_P2P_OP_WAIT, a, b, CRO_P2P_EV_HBM, 0, 0, 0);
            if (r > 0) op(CRO_P2P_OP_WAIT, a, b, CRO_P2P_EV_REREAD, r - 1, 0, 0);
            op(CRO_P2P_OP_READ, a, b, 0, r, kSlotP2P0 + 3 * b, P);
            if (push) op(CRO_P2P_OP_PUSH, a, b, 0, r, kSlotP2P0 + 3 * b + 1, P);
        }
        // every device publishes both round events, byes and unscheduled pairs included: the next round's pusher waits
        // on its partner's re-read event of this round, and a device that sat out must not leave a stale one there
        for (int i = 0; i < n; ++i) op(CRO_P2P_OP_RECORD, i, i, CRO_P2P_EV_PUSH, r, 0, 0);
        for (const auto& [a, b] : directed) {                   // stage B: the receiver checks what landed
            if (!push) continue;
            op(CRO_P2P_OP_WAIT, b, a, CRO_P2P_EV_PUSH, r, 0, 0);
            op(CRO_P2P_OP_REREAD, b, a, 0, r, kSlotP2P0 + 3 * a + 2, P);
        }
        for (int i = 0; i < n; ++i) op(CRO_P2P_OP_RECORD, i, i, CRO_P2P_EV_REREAD, r, 0, 0);
    }
    // latency: every device chases all its peers at once (one warp per peer, one load in flight each), after EVERY
    // device has finished its bandwidth legs so the links are quiet
    for (int i = 0; i < n; ++i) op(CRO_P2P_OP_RECORD, i, i, CRO_P2P_EV_CHASE, 0, 0, 0);
    for (int i = 0; i < n; ++i) {
        for (int j = 0; j < n; ++j)
            if (j != i) op(CRO_P2P_OP_WAIT, i, j, CRO_P2P_EV_CHASE, 0, 0, 0);
        op(CRO_P2P_OP_CHASE, i, i, 0, 0, 0, 0);
        op(CRO_P2P_OP_FINALIZE, i, i, 0, 0, 0, 0);
        P2PFinalizePlan& f = p.fin[i];
        f.n = (uint32_t)n;
        f.self = (uint32_t)i;
        f.have_push = (push && !unidir) ? 1u : 0u;
        f.push_folded = write_variant == COPY_TMA_FUSED ? 1u : 0u;   // the plain copies land bytes but fold nothing
        f.p2p_bytes = P;
        for (int j = 0; j < n; ++j)
            if (j != i && linked(i, j)) f.chase_mask |= 1u << j;
        f.peer_mask = f.chase_mask;
        if (unidir)     // measurement mode: only the pairs' first devices read; check nothing that did not run
            for (const auto& rd : p.rounds)
                for (const auto& pr : rd)
                    if (pr.second == i) f.peer_mask &= ~(1u << pr.first);
    }
    return p;
}

cudaEvent_t plan_event(Device* d, const P2POp& o) {
    switch (o.event) {
        case CRO_P2P_EV_HBM: return d->ev_hbm_done;
        case CRO_P2P_EV_PUSH: return d->ev_push_done[o.round];
        case CRO_P2P_EV_REREAD: return d->ev_reread_done[o.round];
        default: return d->ev_chase_ready;
    }
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
    // the plan needs every device's S after any CRO_F_DEGRADE_ON_OOM halving, so the regions exist before it is made
    std::vector<uint64_t> sizes((size_t)n);
    std::vector<uint8_t> access((size_t)n * 8);
    for (int i = 0; i < n; ++i) {
        Device* d = c->devs[(size_t)i].get();
        if ((rc = ensure_region(c, d))) return rc;
        sizes[(size_t)i] = d->sweep_bytes;
        memcpy(&access[(size_t)i * 8], d->tmpl.p2p_access, 8);
    }
    const unsigned rvp = c->knobs.get("CRO_P2P_READ_VARIANT"), wvp = c->knobs.get("CRO_P2P_WRITE_VARIANT");
    const P2PPlan plan = make_p2p_plan(n, sizes.data(), o.p2p_bytes, access.data(), o.flags, c->knobs.get("CRO_P2P_UNIDIR") != 0, wvp);
    for (int i = 0; i < n && p2p; ++i) {
        Device* d = c->devs[(size_t)i].get();
        CU_TRY(c, cudaSetDevice(d->ordinal));
        while (d->ev_push_done.size() < plan.rounds.size()) {
            cudaEvent_t e1, e2;
            CU_TRY(c, cudaEventCreateWithFlags(&e1, cudaEventDisableTiming));
            CU_TRY(c, cudaEventCreateWithFlags(&e2, cudaEventDisableTiming));
            d->ev_push_done.push_back(e1);
            d->ev_reread_done.push_back(e2);
        }
    }

    // ---- phases 1 and 2: every device's HBM probe, then the NVLink rounds, 1-factorised so each GPU is in exactly one
    // pair per round and chained across devices by events, then the chase and the verdict; nothing waits on the host.
    // Per round and device (partner p):  [wait p's HBM phase, p's previous re-read]  READ p's half A over the link ->
    // PUSH my prefix into p's half B -> [wait p's push]  RE-READ my own half B locally.
    {
        Range nv(c, "cro.probe_all.enqueue");
        for (const P2POp& op : plan.ops) {
            Device* d = c->devs[op.dev].get();
            Device* p = c->devs[op.peer].get();
            CU_TRY(c, cudaSetDevice(d->ordinal));
            switch (op.kind) {
                case CRO_P2P_OP_HBM:
                    if ((rc = probe_enqueue(c, d, d->lanes[0]))) return rc;
                    break;
                case CRO_P2P_OP_PREFIX:   // what this device's first P bytes must fold to, for the peers that will read them
                    CU_TRY(c, launch_expected(d->plan, op.bytes, imm_params(d), d->scratch_pfx, &d->d_out[op.slot], d->aux));
                    c->launches++;
                    CU_TRY(c, cudaEventRecord(d->ev_aux_done, d->aux));
                    CU_TRY(c, cudaStreamWaitEvent(d->stream, d->ev_aux_done, 0));
                    break;
                case CRO_P2P_OP_RECORD:
                    CU_TRY(c, cudaEventRecord(plan_event(d, op), d->stream));
                    break;
                case CRO_P2P_OP_WAIT:
                    CU_TRY(c, cudaStreamWaitEvent(d->stream, plan_event(p, op), 0));
                    break;
                case CRO_P2P_OP_READ:
                    // TMA bulk copies straight out of the peer's HBM (cp.async.bulk on the peer-mapped address) into this
                    // GPU's shared memory, checksummed as they land.  Fold only, as is the re-read below: the words are the
                    // peer's pattern, and p2p_finalize compares the fold with the peer's own closed form.
                    CU_TRY(c, launch_read(d->plan, rvp, p->region, op.bytes, imm_params(d), d->scratch, &d->d_out[op.slot], d->stream,
                                          /*compare=*/false));
                    c->launches++;
                    break;
                case CRO_P2P_OP_PUSH:
                    // posted NVLink writes: d streams its own prefix through shared memory (bulk load from local HBM,
                    // bulk store to the peer-mapped address, folded on the way) into half B of p's region
                    CU_TRY(c, launch_copy(d->plan, wvp, p->region + p->sweep_bytes, d->region, op.bytes, imm_params(d), d->scratch,
                                          &d->d_out[op.slot], d->stream));
                    c->launches++;
                    break;
                case CRO_P2P_OP_REREAD:
                    d->half_known[1] = false;                        // its prefix now holds p's pattern
                    CU_TRY(c, launch_read(d->plan, resolve_read_variant(CRO_READ_AUTO, op.bytes, c->knobs), d->region + d->sweep_bytes,
                                          op.bytes, imm_params(d), d->scratch, &d->d_out[op.slot], d->stream, /*compare=*/false));
                    c->launches++;
                    break;
                case CRO_P2P_OP_CHASE: {
                    ChaseArgs ca{};
                    ca.n = (unsigned)n;
                    ca.hops = o.latency_hops;
                    for (int j = 0; j < n; ++j)
                        if (plan.fin[op.dev].chase_mask >> j & 1) ca.table[j] = c->devs[(size_t)j]->d_chase_tables[op.dev];
                    CU_TRY(c, arm_chase_out(d->d_chase_out, d->stream));   // a row the chase does not walk cannot pass
                    CU_TRY(c, launch_chase(ca, d->d_chase_out, d->stream));
                    c->launches++;
                    break;
                }
                case CRO_P2P_OP_FINALIZE: {
                    const P2PFinalizePlan& f = plan.fin[op.dev];
                    P2PFinalizeArgs pa{};
                    pa.out = d->d_result;
                    pa.slots = d->d_out;
                    pa.chase_out = d->d_chase_out;
                    pa.n = f.n;
                    pa.self = f.self;
                    pa.hops = o.latency_hops;
                    pa.have_push = f.have_push;
                    pa.push_folded = f.push_folded;
                    pa.p2p_bytes = f.p2p_bytes;
                    pa.stamp = d->nonce_cur;
                    for (int j = 0; j < n; ++j) {
                        if (f.peer_mask >> j & 1) {
                            pa.peer_slots[j] = c->devs[(size_t)j]->d_out;
                            pa.peer_stamp[j] = c->devs[(size_t)j]->nonce_cur;
                        }
                        if (f.chase_mask >> j & 1) pa.chase_expect[j] = d->chase_expect[(size_t)j];
                    }
                    CU_TRY(c, launch_p2p_finalize(pa, d->stream));
                    c->launches++;
                    CU_TRY(c, cudaMemcpyAsync(d->h_chase_out, d->d_chase_out, 2 * CRO_MAX_DEVICES * sizeof(unsigned long long), cudaMemcpyDeviceToHost, d->stream));
                    CU_TRY(c, cudaMemcpyAsync(d->h_out, d->d_out, sizeof(SweepOut) * kSlotCount, cudaMemcpyDeviceToHost, d->stream));
                    break;
                }
                default:
                    c->set_error("full-box plan: unknown op " + std::to_string(op.kind));
                    return CRO_ERR_INTERNAL;
            }
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
                if (plan.fin[i].chase_mask >> j & 1)      // the rows of peers it does not chase keep the armed value
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
    c->fullbox.rounds = (uint32_t)plan.rounds.size();
    c->fullbox.host_syncs = host_syncs;
    c->fullbox.gather = use_nccl ? CRO_GATHER_NCCL : nccl_degraded ? CRO_GATHER_DEGRADED : CRO_GATHER_HOST;
    c->fullbox.wall_ns = now_ns() - t_call;
    return worst;
}

int selftest_p2p_plan(uint32_t n, const uint64_t* sweep_bytes, uint64_t p2p_bytes, const uint8_t* access, uint32_t flags,
                      uint32_t unidir, uint32_t write_variant, cro_p2p_plan* out) {
    if (!sweep_bytes || !access || !out || n > CRO_MAX_DEVICES) return CRO_ERR_INVALID_ARG;
    const P2PPlan p = make_p2p_plan((int)n, sweep_bytes, p2p_bytes, access, flags, unidir != 0, write_variant);
    if (p.ops.size() > CRO_P2P_PLAN_OPS || p.rounds.size() > CRO_P2P_PLAN_ROUNDS) {
        set_thread_error("full-box plan larger than cro_p2p_plan holds");
        return CRO_ERR_INTERNAL;
    }
    memset(out, 0, sizeof *out);
    out->p2p_bytes = p.p2p_bytes;
    out->n_rounds = (uint32_t)p.rounds.size();
    out->n_ops = (uint32_t)p.ops.size();
    for (size_t r = 0; r < p.rounds.size(); ++r) {
        out->n_pairs[r] = (uint8_t)p.rounds[r].size();
        for (size_t k = 0; k < p.rounds[r].size(); ++k) {
            out->pair[r][2 * k] = (uint8_t)p.rounds[r][k].first;
            out->pair[r][2 * k + 1] = (uint8_t)p.rounds[r][k].second;
        }
    }
    memcpy(out->fin, p.fin, sizeof p.fin);
    memcpy(out->op, p.ops.data(), p.ops.size() * sizeof(P2POp));
    return CRO_OK;
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
