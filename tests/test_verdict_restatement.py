"""The host restatement of the device-side verdict (oracle/verdict.py) on hand-worked cases, so that the GPU tests that
hold the finalize kernels against it do not rest on the restatement checking itself.  No GPU needed."""
import os
import random
import sys

import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
import verdict as V  # noqa: E402

M = V.MASK64
NONCE, SEED = 7, 0x1234
S = 1 << 20                      # sweep bytes
E = (0xAAAA, 0xBBBB, 0xCCCC)     # the closed form the slots are compared with


def slot(fold=E, t0=0, t1=0, stamp=NONCE, n_words=S // 8):
    return V.Slot(fold[0], fold[1], fold[2], t0, t1, stamp, n_words)


def healthy(C, R, read_ns=None, copy_ns=None):
    """Slots of a probe that passed: fill [100, 150), then copies and reads back to back."""
    sl = [V.ARMED] * V.SLOT_COUNT
    sl[V.SLOT_FILL] = slot((0, 0, 0), 100, 150)
    sl[V.SLOT_EXPECT] = slot(E, 120, 130)
    t = 150
    for i in range(C):
        d = copy_ns[i] if copy_ns else 20
        sl[V.SLOT_SWEEP0 + i] = slot(E, t, t + d)
        t += d
    for i in range(R):
        d = read_ns[i] if read_ns else 10
        sl[V.SLOT_SWEEP0 + C + i] = slot(E, t, t + d)
        t += d
    return sl


TMPL = bytes(random.Random(5).randrange(256) for _ in range(512))


def fin(sl, C, R, cv=V.COPY_TMA_FUSED, rv=1):
    return V.Result(V.probe_finalize(TMPL, sl, SEED, NONCE, S, R, C, rv, cv))


def test_a_healthy_probe():
    r = fin(healthy(2, 3, read_ns=[30, 10, 20], copy_ns=[25, 15]), C=2, R=3)
    assert (r.get("status"), r.get("fail_code"), r.get("fail_index")) == (0, 0, 0)
    assert r.get("copy_verified") == 2                           # copy 1 (folded copy 0's output) + read 0
    assert (r.get("read_best_ns"), r.get("read_median_ns")) == (10, 20)
    assert (r.get("copy_best_ns"), r.get("copy_median_ns")) == (15, 25)   # sorted [15, 25][1]: the upper median
    assert (r.get("fill_ns"), r.get("t_start_ns"), r.get("total_ns")) == (50, 100, 150 + 25 + 15 + 30 + 10 + 20 - 100)
    assert (r.get("checksum_xor"), r.get("checksum_sum"), r.get("checksum_wsum")) == E
    assert (r.get("copy_checksum_xor"), r.get("expect_wsum")) == (E[0], E[2])
    assert (r.get("seed"), r.get("nonce"), r.get("sweep_bytes"), r.get("copy_variant"), r.get("read_variant")) == (SEED, NONCE, S, 3, 1)
    # the fields the verdict does not own come from the template, byte for byte
    t = V.Result(TMPL)
    for name in ("abi_version", "gpu_uuid", "pci_bus_id", "sm_count", "ecc_errors", "p2p_read_ns", "p2p_access", "p2p_bytes",
                 "p2p_write_ns", "rank", "world", "p2p_ok", "reserved8"):
        assert r.get(name) == t.get(name), name


def test_even_counts_take_the_upper_median():
    assert V.best_and_median([40, 10, 30, 20]) == (10, 30)
    assert V.best_and_median([5, 5]) == (5, 5) and V.best_and_median([]) == (0, 0)


def test_the_closed_form_check_comes_first():
    sl = healthy(1, 1)
    sl[V.SLOT_FILL] = sl[V.SLOT_FILL]._replace(stamp=NONCE - 1)
    sl[V.SLOT_EXPECT] = sl[V.SLOT_EXPECT]._replace(n_words=S // 8 - 1)
    r = fin(sl, 1, 1)
    assert (r.get("status"), r.get("fail_code"), r.get("fail_index")) == (V.ERR_CHECKSUM, V.FAIL_EXPECT, 0)
    sl = healthy(1, 1)
    sl[V.SLOT_FILL] = sl[V.SLOT_FILL]._replace(n_words=S // 8 + 1)
    assert (fin(sl, 1, 1).get("fail_code"), fin(sl, 1, 1).get("fail_index")) == (V.FAIL_STALE, 0)


def test_a_plain_copy_that_did_not_run_is_stale_and_its_fold_is_not_checked():
    sl = healthy(3, 2)
    for i in range(3):                                           # plain copies publish a zero checksum
        sl[V.SLOT_SWEEP0 + i] = sl[V.SLOT_SWEEP0 + i]._replace(x=0, s=0, w=0)
    r = fin(sl, 3, 2, cv=1)
    assert (r.get("status"), r.get("copy_verified"), r.get("copy_variant")) == (0, 1, 1)   # only read 0 verifies
    sl[V.SLOT_SWEEP0 + 1] = V.ARMED
    r = fin(sl, 3, 2, cv=2)
    assert (r.get("fail_code"), r.get("fail_index"), r.get("copy_verified")) == (V.FAIL_STALE, 2, 1)


def test_copies_after_a_failure_still_count_as_verified():
    sl = healthy(3, 1)
    sl[V.SLOT_SWEEP0] = sl[V.SLOT_SWEEP0]._replace(x=1)
    r = fin(sl, 3, 1)
    assert (r.get("fail_code"), r.get("fail_index"), r.get("copy_verified")) == (V.FAIL_COPY_SRC, 0, 3)


def test_the_struct_shows_the_read_that_failed_first():
    sl = healthy(1, 3)
    bad = (1, 2, 3)
    sl[V.SLOT_SWEEP0 + 2] = slot(bad, 5, 6)                      # read 1: wrong fold
    sl[V.SLOT_SWEEP0 + 3] = slot((9, 9, 9), 7, 8, stamp=0)        # read 2: stale
    r = fin(sl, 1, 3)
    assert (r.get("fail_code"), r.get("fail_index")) == (V.FAIL_READ, 1)
    assert (r.get("checksum_xor"), r.get("checksum_sum"), r.get("checksum_wsum")) == bad
    assert (r.get("copy_checksum_xor"), r.get("copy_verified")) == (E[0], 1)
    sl = healthy(2, 2)
    sl[V.SLOT_SWEEP0 + 3] = sl[V.SLOT_SWEEP0 + 3]._replace(stamp=NONCE + 1)
    r = fin(sl, 2, 2)
    assert (r.get("fail_code"), r.get("fail_index"), r.get("checksum_xor")) == (V.FAIL_STALE, 4, E[0])  # launch order: 1 + C + 1


@pytest.mark.parametrize("count", [1, 2, 1 << 32, M])
def test_a_read_whose_fold_matches_but_whose_words_differ_fails_at_its_index(count):
    """A multi-word fault the fold cannot see: the read's fold equals the closed form, its word count does not."""
    for C, R in ((2, 3), (0, 2), (3, 1)):
        for i in range(R):
            sl = healthy(C, R)
            sl[V.SLOT_SWEEP0 + C + i] = sl[V.SLOT_SWEEP0 + C + i]._replace(mismatches=count)
            r = fin(sl, C, R)
            assert (r.get("status"), r.get("fail_code"), r.get("fail_index")) == (V.ERR_CHECKSUM, V.FAIL_READ, i), (C, R, i)
            assert (r.get("checksum_xor"), r.get("checksum_sum"), r.get("checksum_wsum")) == E     # the shown fold is that read's
            # read 0 verifies the last copy only when it passed
            assert r.get("copy_verified") == (C - 1 if C else 0) + (1 if C and i > 0 else 0), (C, R, i)
    # a copy's slot carries no count the verdict reads
    sl = healthy(2, 1)
    sl[V.SLOT_SWEEP0] = sl[V.SLOT_SWEEP0]._replace(mismatches=count)
    assert (fin(sl, 2, 1).get("status"), fin(sl, 2, 1).get("copy_verified")) == (0, 2)


def test_a_stale_read_is_stale_before_its_count_is_looked_at():
    sl = healthy(1, 2)
    sl[V.SLOT_SWEEP0 + 1] = sl[V.SLOT_SWEEP0 + 1]._replace(stamp=NONCE + 1, mismatches=5)
    r = fin(sl, 1, 2)
    assert (r.get("fail_code"), r.get("fail_index"), r.get("copy_verified")) == (V.FAIL_STALE, 2, 0)
    sl = healthy(1, 2)                                             # the first failing read wins: the stale one
    sl[V.SLOT_SWEEP0 + 1] = sl[V.SLOT_SWEEP0 + 1]._replace(n_words=0)
    sl[V.SLOT_SWEEP0 + 2] = sl[V.SLOT_SWEEP0 + 2]._replace(mismatches=1)
    assert (fin(sl, 1, 2).get("fail_code"), fin(sl, 1, 2).get("fail_index")) == (V.FAIL_STALE, 2)
    sl = healthy(1, 2)                                             # ... or the counting one, when it comes first
    sl[V.SLOT_SWEEP0 + 1] = sl[V.SLOT_SWEEP0 + 1]._replace(mismatches=1)
    sl[V.SLOT_SWEEP0 + 2] = sl[V.SLOT_SWEEP0 + 2]._replace(stamp=0)
    assert (fin(sl, 1, 2).get("fail_code"), fin(sl, 1, 2).get("fail_index")) == (V.FAIL_READ, 0)


def test_no_copies():
    r = fin(healthy(0, 1), C=0, R=1)
    t = V.Result(TMPL)
    assert (r.get("status"), r.get("copy_variant"), r.get("copy_verified"), r.get("copy_best_ns"), r.get("copy_median_ns")) == (0, 0, 0, 0, 0)
    assert r.get("copy_checksum_xor") == t.get("copy_checksum_xor")   # not written without copies


def test_total_time_wraps_modulo_2_64():
    sl = healthy(0, 1)                                             # read 0: [150, 160)
    sl[V.SLOT_FILL] = sl[V.SLOT_FILL]._replace(t0=M - 4, t1=M)
    r = fin(sl, 0, 1)
    assert (r.get("total_ns"), r.get("fill_ns")) == (4, 4)         # the latest t1 is the fill's own
    sl[V.SLOT_FILL] = sl[V.SLOT_FILL]._replace(t0=200, t1=100)     # every t1 below the fill's t0
    r = fin(sl, 0, 1)
    assert (r.get("total_ns"), r.get("fill_ns"), r.get("t_start_ns")) == ((160 - 200) & M, (100 - 200) & M, 200)


def peer_state(n, self_index, access, hops=1024):
    """A healthy p2p state: every reachable peer's prefix folds to P, every leg matches, every chase ends where it must."""
    P = (0x11, 0x22, 0x33)
    PB = 1 << 16
    res = fin(healthy(1, 1), 1, 1)
    res.set("p2p_access", access)
    res.set("status", 0)
    res.set("fail_code", 0)
    mine = [V.ARMED] * V.SLOT_COUNT
    mine[V.SLOT_PREFIX] = slot(P, stamp=NONCE, n_words=PB // 8)
    peers, stamps = [None] * V.MAX_DEVICES, [0] * V.MAX_DEVICES
    chase, expect = [V.MASK64] * (2 * V.MAX_DEVICES), [0] * V.MAX_DEVICES
    for j in range(n):
        if j == self_index:
            continue
        ps = [V.ARMED] * V.SLOT_COUNT
        ps[V.SLOT_PREFIX] = slot(P, stamp=100 + j, n_words=PB // 8)
        peers[j], stamps[j] = ps, 100 + j
        for k in range(3):
            mine[V.SLOT_P2P0 + 3 * j + k] = slot(P, 10 * j, 10 * j + 5 + k, NONCE, PB // 8)
        chase[2 * j], chase[2 * j + 1], expect[j] = 40 + j, 64 * hops, 40 + j
    return dict(result=res.bytes(), slots=mine, peer_slots=peers, peer_stamp=stamps, chase_out=chase, chase_expect=expect,
                n=n, self_index=self_index, hops=hops, have_push=True, push_folded=True, p2p_bytes=PB, stamp=NONCE)


def test_p2p_healthy_and_one_bad_chase():
    st = peer_state(3, 0, [0, 1, 1, 0, 0, 0, 0, 0])
    r = V.Result(V.p2p_finalize(**st))
    assert (r.get("status"), r.get("p2p_ok"), r.get("p2p_bytes")) == (0, 0b110, 1 << 16)
    assert r.get("p2p_latency_ns_x16")[1:3] == [64 * 16, 64 * 16] and r.get("p2p_read_ns")[1:3] == [5, 5]
    assert r.get("p2p_write_ns")[1:3] == [6, 6] and r.get("p2p_checksum_xor")[2] == 0x11
    st["chase_out"][2 * 2] = V.MASK64                         # the chase into peer 2 never ran: the armed value
    r = V.Result(V.p2p_finalize(**st))
    assert (r.get("status"), r.get("fail_code"), r.get("fail_index"), r.get("p2p_ok")) == (V.ERR_CHECKSUM, V.FAIL_P2P_CHASE, 2, 0b010)


def test_p2p_skips_self_unreachable_and_absent_peers_and_keeps_an_earlier_failure():
    st = peer_state(3, 1, [1, 0, 0, 0, 0, 0, 0, 0])           # peer 2 unreachable: not even its bad read matters
    st["slots"][V.SLOT_P2P0 + 3 * 2] = V.ARMED
    r = V.Result(V.p2p_finalize(**st))
    assert (r.get("status"), r.get("p2p_ok")) == (0, 0b001)
    st["peer_slots"][0] = None                                # absent peer: no check at all
    assert V.Result(V.p2p_finalize(**st)).get("p2p_ok") == 0
    st = peer_state(3, 0, [0, 1, 1, 0, 0, 0, 0, 0])
    res = V.Result(st["result"])
    res.set("status", V.ERR_CHECKSUM), res.set("fail_code", V.FAIL_READ), res.set("fail_index", 4)
    st["result"] = res.bytes()
    st["slots"][V.SLOT_P2P0 + 3 * 1 + 2] = V.ARMED            # a bad re-read of peer 1's push
    r = V.Result(V.p2p_finalize(**st))
    assert (r.get("status"), r.get("fail_code"), r.get("fail_index"), r.get("p2p_ok")) == (V.ERR_CHECKSUM, V.FAIL_READ, 4, 0b100)


def test_p2p_stale_prefix_and_push_rules():
    st = peer_state(2, 0, [0, 1, 0, 0, 0, 0, 0, 0])
    st["peer_slots"][1][V.SLOT_PREFIX] = st["peer_slots"][1][V.SLOT_PREFIX]._replace(n_words=1)
    r = V.Result(V.p2p_finalize(**st))
    assert (r.get("fail_code"), r.get("fail_index"), r.get("p2p_ok")) == (V.FAIL_EXPECT, 1, 0)
    st = peer_state(2, 0, [0, 1, 0, 0, 0, 0, 0, 0])
    st["slots"][V.SLOT_P2P0 + 3 * 1 + 1] = V.ARMED            # my push slot is stale: no write time
    assert V.Result(V.p2p_finalize(**st)).get("fail_code") == V.FAIL_P2P_PUSH
    st["push_folded"] = False                                 # a plain push folds nothing: only the receiver checks
    r = V.Result(V.p2p_finalize(**st))
    assert (r.get("status"), r.get("p2p_write_ns")[1]) == (0, V.Result(st["result"]).get("p2p_write_ns")[1])
    st["have_push"], st["hops"] = False, 0
    st["slots"][V.SLOT_P2P0 + 3 * 1 + 2] = V.ARMED
    st["chase_out"][2] = 5
    assert V.Result(V.p2p_finalize(**st)).get("p2p_ok") == 0b10   # no push leg, no chase: neither is checked


@pytest.mark.parametrize("ns,hops,want", [(1000, 16, 1000), (7, 3, 37), (1 << 28, 1, 0xFFFFFFFF), (1 << 62, 1 << 20, 0xFFFFFFFF),
                                          (V.MASK64, 65536, 0xFFFFFFFF), (1 << 60, 1 << 31, 0xFFFFFFFF),
                                          (1 << 58, 1 << 31, 0x80000000)])
def test_latency_saturates_without_wrapping(ns, hops, want):
    assert V.latency_x16(ns, hops) == want
