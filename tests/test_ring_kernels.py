"""The shared-memory ring kernels across their legal knob space, against the oracle.

hbm_read_tma_kernel, hbm_copy_tma_kernel and hbm_copy_fused_kernel hold the project's hand-written synchronisation
(mbarrier phase parity, per-warp "empty" barriers, the end-of-work mark, bulk-group read waits, dynamic tile claims).
Its behaviour depends on the CRO_* ring knobs, and every value env.cpp accepts is a supported configuration, so each
row of CONFIGS below gets its own context at sizes chosen around the tile: one word, one tile either side, eight tiles
with a partial last one, and enough tiles for every CTA's ring to wrap its phase several times.

The module keeps to itself: each configuration opens and closes its own context, and no context here outlives its test.
Every context has a deadline, so a ring that never drains fails with CRO_ERR_DEADLINE instead of hanging."""
import os

import pytest

from test_env_knobs import largest_ring_tile

pytestmark = pytest.mark.gpu

MASK = (1 << 64) - 1
MiB = 1 << 20
SMS = 132                       # H100 SXM
DEADLINE_MS = 20000
LDG, TMA, LDG256 = 1, 2, 3      # READ_* and COPY_* share the first two numbers
FUSED = 3
DEFAULT_TILE, DEFAULT_STAGES = 32768, 4


def _rings(tile, stages, threads=None, chunk=None):
    """The same tile and depth on all three rings (and the same threads / chunk where the ring has that knob)."""
    env = {}
    for p in ("CRO_TMA_READ", "CRO_TMA_COPY", "CRO_FUSED"):
        env[p + "_TILE"], env[p + "_STAGES"] = tile, stages
        if chunk is not None:
            env[p + "_CHUNK"] = chunk
    if threads is not None:
        env["CRO_TMA_READ_THREADS"] = env["CRO_FUSED_THREADS"] = threads
    return env


# name -> knobs.  "largest" rows take the largest ring cro_validate_env accepts at that depth, found at run time.
CONFIGS = {
    "smallest": _rings(1024, 2, threads=64),
    "ragged-tile": _rings(1040, 3, threads=96, chunk=7),            # 65 vectors a tile over 64 consumer threads
    "deepest": _rings(8192, 16, threads=1024),                      # full_bar[16] / tile_of[16] exactly full, 31 consumer warps
    "largest-tile": _rings(114688, 2, chunk=4096),                  # one CTA claims every tile, the others none
    "static-oversubscribed": dict(_rings(4096, 5), CRO_TMA_READ_DYN=0, CRO_TMA_COPY_DYN=0,
                                  CRO_TMA_READ_WAVES=4, CRO_TMA_COPY_WAVES=4),
    **{"hints-%d" % h: dict(CRO_TMA_READ_HINT=1, CRO_TMA_COPY_HINT=h) for h in (1, 2, 4, 3, 6, 7)},
    "ldg-waves-1": dict(CRO_READ_WAVES=1, CRO_COPY_WAVES=1, CRO_FILL_WAVES=1),
    "ldg-waves-1024": dict(CRO_READ_WAVES=1024, CRO_COPY_WAVES=1024, CRO_FILL_WAVES=1024),   # grids clamped to the tiles
    "largest-read-ring": {"largest": ("CRO_TMA_READ", 4)},
    "largest-fused-ring": {"largest": ("CRO_FUSED", 8)},
}
# the "wrap" size: at least 4 * 132 * stages tiles, capped at 256 MiB.  The static, oversubscribed row runs several CTAs
# per SM on four waves, so it takes the cap to wrap its rings too.
CAP = 256 * MiB
SIZES = ["16", "T-16", "T", "T+16", "7T+48", "wrap"]


def _apply(monkeypatch, cro, cfg):
    """Sets the row's knobs; returns (tile, stages) of the ring the sizes are built around."""
    cfg = dict(cfg)
    largest = cfg.pop("largest", None)
    for k, v in cfg.items():
        monkeypatch.setenv(k, str(v))
    if largest:
        prefix, stages = largest
        return largest_ring_tile(cro, monkeypatch, prefix, stages), stages
    if "CRO_FUSED_TILE" in cfg:                 # rows that set a ring set all three alike
        return int(cfg["CRO_FUSED_TILE"]), int(cfg["CRO_FUSED_STAGES"])
    return DEFAULT_TILE, DEFAULT_STAGES


def _size(label, T, D, name):
    if label == "wrap":
        tiles = 4 * SMS * D if name != "static-oversubscribed" else CAP // T
        return min(tiles * T, CAP - T) + 48
    return {"16": 16, "T-16": T - 16, "T": T, "T+16": T + 16, "7T+48": 7 * T + 48}[label]


def _want(coracle, seed, n_words):
    return coracle.checksum(seed, 0, n_words, threads=os.cpu_count() or 1)


def _flipped(coracle, seed, want, word, bit):
    """The checksum of the pattern with one bit of one word flipped: xor by that bit, the sum by the change, the
    weighted sum by the change times (2 * word + 1)."""
    w = coracle.pattern_word(seed, word)
    d = ((w ^ (1 << bit)) - w) & MASK
    return want[0] ^ (1 << bit), (want[1] + d) & MASK, (want[2] + d * (2 * word + 1)) & MASK


def _probe_ok(coracle, r, S, copy_verified):
    want = _want(coracle, r.seed, S // 8)
    assert r.status == 0 and r.fail_code == 0, (r.status, r.fail_code, r.fail_index)
    assert r.checksum == r.expect == want
    assert r.copy_verified == copy_verified


def _check_rings(cro, coracle, T, D, S):
    """Every ring kernel at sweep size S with tile T and depth D: checksums, copied words, located faults, a whole probe."""
    with cro.ProbeContext(sweep_bytes=S, devices=[0], read_sweeps=2, copy_sweeps=3, read_variant=TMA, copy_variant=FUSED,
                          deadline_ms=DEADLINE_MS, seed_base=0x5EED000000000000) as c:
        n = S // 8
        seed = c.seed(0)
        want = _want(coracle, seed, n)
        for rv in (TMA, LDG, LDG256):
            assert c.hbm_read_checksum(0, rv).checksum == want, ("read", rv)

        # words either side of tile boundaries (first ones, around slot 0's reuse, the last one) and the last word
        tw = T // 8
        ks = sorted({k for k in (1, 2, D - 1, D, D + 1, (n - 1) // tw) if k >= 1 and k * tw < n})
        spans = [(k * tw - 1, 2) for k in ks] + [(0, 1), (n - 1, 1)]
        for cv in (LDG, TMA, FUSED):
            c.inject_fault(0, n, 0xFFFF)                 # dirty the destination's first and last word
            c.inject_fault(0, 2 * n - 1, 0xFFFF << 48)
            k = c.hbm_copy(0, cv)
            assert k.variant == cv
            if cv == FUSED:
                assert k.checksum == want, "the checksumming copy's own fold"
            for rv in (LDG, TMA):
                assert c.hbm_read_checksum(0, rv, dst=True).checksum == want, ("copy", cv, "read", rv)
            for first, cnt in spans:
                got = c.read_words(0, n + first, cnt)
                assert got == [coracle.pattern_word(seed, first + i) for i in range(cnt)], ("copy", cv, "word", first)

        # one flipped bit at a time: word 0, the last word (partial last tile), the first word of tile D (slot 0's
        # second use under static striding)
        faults = {(0, 0), (n - 1, 63)} | ({(D * tw, 17)} if D * tw < n else set())
        for word, bit in sorted(faults):
            c.inject_fault(0, word, 1 << bit)
            bad = _flipped(coracle, seed, want, word, bit)
            assert c.hbm_read_checksum(0, TMA).checksum == bad, ("read", word, bit)
            assert c.hbm_copy(0, FUSED).checksum == bad, ("fused copy", word, bit)
            c.inject_fault(0, word, 1 << bit)            # undo
        assert c.hbm_read_checksum(0, TMA).checksum == want

        r = c.probe_device(0)
        assert r.read_variant == TMA and r.copy_variant == FUSED
        _probe_ok(coracle, r, S, copy_verified=3)
        assert r.copy_checksum == r.checksum


@pytest.mark.parametrize("label", SIZES)
@pytest.mark.parametrize("name", list(CONFIGS))
def test_ring_configuration(cro, coracle, monkeypatch, name, label):
    T, D = _apply(monkeypatch, cro, CONFIGS[name])
    assert cro.validate_env() == ""
    _check_rings(cro, coracle, T, D, _size(label, T, D, name))


def test_tile_counter_under_contention(cro, coracle, monkeypatch):
    """1 GiB with chunked dynamic claims on all three rings: thousands of claims race for the one counter."""
    for p, chunk in (("CRO_TMA_READ", 3), ("CRO_TMA_COPY", 5), ("CRO_FUSED", 3)):
        monkeypatch.setenv(p + "_CHUNK", str(chunk))
    S = (1 << 30) + 48
    with cro.ProbeContext(sweep_bytes=S, devices=[0], read_sweeps=2, copy_sweeps=3, read_variant=TMA, copy_variant=FUSED,
                          deadline_ms=DEADLINE_MS) as c:
        want = _want(coracle, c.seed(0), S // 8)
        assert c.hbm_read_checksum(0, TMA).checksum == want
        for cv in (TMA, FUSED):
            k = c.hbm_copy(0, cv)
            if cv == FUSED:
                assert k.checksum == want
            assert c.hbm_read_checksum(0, TMA, dst=True).checksum == want, cv
        _probe_ok(coracle, c.probe_device(0), S, copy_verified=3)


def test_one_ring_step_past_the_largest_is_refused_by_its_knob(cro, monkeypatch):
    tile = largest_ring_tile(cro, monkeypatch, "CRO_FUSED", 4)
    monkeypatch.setenv("CRO_FUSED_TILE", str(tile + 16))
    with pytest.raises(cro.ProbeError) as e:
        cro.ProbeContext(sweep_bytes=1 << 20, devices=[0], deadline_ms=DEADLINE_MS)
    assert e.value.code == cro.ERR_INVALID_ARG
    assert "the env variable CRO_FUSED_TILE has an invalid value: '%d'" % (tile + 16) in str(e.value)


# ---- the whole probe across its variants and paths ---------------------------------------------------------------
RAGGED = (32 << 20) + 32784


@pytest.mark.parametrize("cv", [LDG, TMA, FUSED])
@pytest.mark.parametrize("rv", [LDG, TMA, LDG256])
def test_probe_variants(cro, coracle, rv, cv):
    """Without the checksumming copy the finalize kernel has no copy-source folds to judge: only read sweep 0, which
    re-reads the last copy's destination, verifies a copy."""
    with cro.ProbeContext(sweep_bytes=RAGGED, devices=[0], read_sweeps=2, copy_sweeps=3, read_variant=rv, copy_variant=cv,
                          deadline_ms=DEADLINE_MS) as c:
        for _ in range(2):                        # graph capture, then replay
            r = c.probe_device(0)
            assert r.read_variant == rv and r.copy_variant == cv
            _probe_ok(coracle, r, RAGGED, copy_verified=3 if cv == FUSED else 1)
            assert r.copy_checksum == r.checksum


@pytest.mark.parametrize("rv", [LDG, TMA])
@pytest.mark.parametrize("cv", [LDG, TMA])
def test_plain_copies_carry_a_corrupt_fill_to_read_sweep_0(cro, coracle, rv, cv):
    """A word corrupted right after the fill travels through every plain copy (they check nothing), so the first sweep
    that folds it is read sweep 0, and no copy counts as verified."""
    word, bit = 123457, 33
    with cro.ProbeContext(sweep_bytes=RAGGED, devices=[0], read_sweeps=2, copy_sweeps=3, read_variant=rv, copy_variant=cv,
                          deadline_ms=DEADLINE_MS, inject=(0, word, 1 << bit)) as c:
        r = c.probe_device(0, allow_checksum_error=True)
        want = _want(coracle, r.seed, RAGGED // 8)
        assert r.expect == want
        assert r.status == cro.ERR_CHECKSUM and r.fail_code == cro.FAIL_READ and r.fail_index == 0
        assert r.copy_verified == 0
        assert r.checksum == _flipped(coracle, r.seed, want, word, bit)


@pytest.mark.parametrize("knob", ["CRO_USE_GRAPH", "CRO_EXPECT_OVERLAP"])
def test_probe_paths_agree(cro, coracle, monkeypatch, knob):
    """Direct launches instead of the graph, and the closed form on the main stream instead of beside the copies: the
    same verdict and the same sweeps as the default path."""
    kinds = {}
    for value in ("1", "0"):
        monkeypatch.setenv(knob, value)
        with cro.ProbeContext(sweep_bytes=RAGGED, devices=[0], read_sweeps=2, copy_sweeps=3, deadline_ms=DEADLINE_MS) as c:
            for _ in range(2):
                r = c.probe_device(0)
                _probe_ok(coracle, r, RAGGED, copy_verified=3)
                assert r.copy_checksum == r.checksum
            times = c.sweep_times(0)
            assert all(t.event_ns > 0 and t.timer_ns > 0 for t in times), (knob, value)
            kinds[value] = [(t.kind, t.index, t.bytes) for t in times]
    assert kinds["0"] == kinds["1"]
    assert [k for k, _, _ in kinds["1"]] == [0] + [1] * 3 + [2] * 2


# ---- knobs belong to the context ---------------------------------------------------------------------------------
def _check_context(coracle, c, S, rv, cv, copy_verified):
    r = c.probe_device(0)
    assert (r.read_variant, r.copy_variant) == (rv, cv)
    _probe_ok(coracle, r, S, copy_verified)
    assert c.hbm_read_checksum(0, TMA).checksum == _want(coracle, c.seed(0), S // 8)
    k = c.hbm_copy(0, FUSED)
    assert k.checksum == _want(coracle, c.seed(0), S // 8)


def test_a_second_context_with_smaller_rings_leaves_the_first_intact(cro, coracle, monkeypatch):
    """The dynamic shared-memory ceiling of a kernel is process-wide.  A context planned with small rings must not
    lower it under one planned with the default 128 KiB rings."""
    S = (64 << 20) + 48
    with cro.ProbeContext(sweep_bytes=S, devices=[0], read_sweeps=2, copy_sweeps=3, read_variant=TMA, copy_variant=FUSED,
                          deadline_ms=DEADLINE_MS) as a:
        _check_context(coracle, a, S, TMA, FUSED, 3)
        for p in ("CRO_TMA_READ", "CRO_TMA_COPY", "CRO_FUSED"):
            monkeypatch.setenv(p + "_TILE", "16384")
            monkeypatch.setenv(p + "_STAGES", "2")
        with cro.ProbeContext(sweep_bytes=S, devices=[0], read_sweeps=2, copy_sweeps=3, read_variant=TMA,
                              copy_variant=FUSED, deadline_ms=DEADLINE_MS, seed_base=0x0BBB000000000000) as b:
            _check_context(coracle, b, S, TMA, FUSED, 3)
            _check_context(coracle, a, S, TMA, FUSED, 3)
            assert a.hbm_copy(0, TMA).variant == TMA
            assert a.hbm_read_checksum(0, TMA, dst=True).checksum == _want(coracle, a.seed(0), S // 8)
            _check_context(coracle, b, S, TMA, FUSED, 3)


def test_knobs_are_read_once_per_context(cro, coracle, monkeypatch):
    """Checking the environment, or opening another context under a changed one, does not change what a live context
    probes with: its read and copy variants stay the ones it resolved at init."""
    S = RAGGED
    monkeypatch.delenv("CRO_READ_VARIANT", raising=False)
    monkeypatch.delenv("CRO_COPY_VARIANT", raising=False)
    with cro.ProbeContext(sweep_bytes=S, devices=[0], read_sweeps=2, copy_sweeps=3, deadline_ms=DEADLINE_MS) as a:
        _check_context(coracle, a, S, LDG, FUSED, 3)           # by size: 128-bit LDG reads up to 128 MiB
        monkeypatch.setenv("CRO_COPY_VARIANT", "1")
        monkeypatch.setenv("CRO_READ_VARIANT", "3")
        assert cro.validate_env() == ""
        _check_context(coracle, a, S, LDG, FUSED, 3)
        assert a.hbm_read_checksum(0).variant == LDG and a.hbm_copy(0).variant == FUSED
        with cro.ProbeContext(sweep_bytes=S, devices=[0], read_sweeps=2, copy_sweeps=3, deadline_ms=DEADLINE_MS,
                              seed_base=0x0BBB000000000000) as b:
            _check_context(coracle, b, S, LDG256, LDG, 1)
            assert b.hbm_read_checksum(0).variant == LDG256 and b.hbm_copy(0).variant == LDG
            _check_context(coracle, a, S, LDG, FUSED, 3)


# ---- peer variants (two or more GPUs) ----------------------------------------------------------------------------
@pytest.fixture(scope="module")
def n_gpus(cro):
    with cro.ProbeContext(sweep_bytes=1 << 20, flags=cro.F_LAZY_ALLOC) as c:
        return c.device_count()


@pytest.mark.parametrize("wvp", [1, 2, 3])
@pytest.mark.parametrize("rvp", [1, 2, 3])
def test_peer_variants(cro, coracle, monkeypatch, n_gpus, rvp, wvp):
    if n_gpus < 2:
        pytest.skip("needs two GPUs")
    monkeypatch.setenv("CRO_P2P_READ_VARIANT", str(rvp))
    monkeypatch.setenv("CRO_P2P_WRITE_VARIANT", str(wvp))
    monkeypatch.setenv("CRO_TMA_READ_TILE", "16400")       # a ragged, non-default read ring for the TMA read leg
    monkeypatch.setenv("CRO_TMA_READ_STAGES", "6")
    S, P = 64 << 20, (16 << 20) + 32784
    with cro.ProbeContext(sweep_bytes=S, p2p_bytes=P, read_sweeps=1, copy_sweeps=1, latency_hops=256,
                          deadline_ms=DEADLINE_MS) as c:
        res = c.probe_all()
        assert len(res) == n_gpus
        for i, r in enumerate(res):
            assert r.status == 0 and r.checksum == _want(coracle, r.seed, S // 8), (i, r.status, r.fail_code, r.fail_index)
            for j in range(min(n_gpus, 8)):
                if j == i or not r.p2p_access[j]:
                    continue
                assert r.p2p_ok & (1 << j), (i, j)
                prefix = coracle.checksum(res[j].seed, 0, P // 8)
                d = c.p2p_detail(i, j)
                assert (d.read_xor, d.read_sum, d.read_wsum) == prefix == (d.expect_xor, d.expect_sum, d.expect_wsum)
                assert (d.landed_xor, d.landed_sum, d.landed_wsum) == coracle.checksum(r.seed, 0, P // 8)
