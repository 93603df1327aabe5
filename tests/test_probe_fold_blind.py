"""The probe's read sweeps against the multi-word faults the fold cannot see, on one GPU.

tests/test_fold_blind_spots.py works out on the CPU which faults leave the fold unchanged.  Here they are placed in
device memory by software (XOR and stuck-at ranges; nothing waits for a real fault) and:
  kernel level (cro_selftest_sweep): each read variant and the checksumming copy fold exactly what the restatement
          (oracle/faults.py) folds for the faulted words, and each read counts exactly the words that differ;
  probe level (CRO_F_TEST_INJECT with a run of words): status, failing sweep and verified copies equal what
          oracle/verdict.py makes of the slots the restated sweeps would write.  A copy's fold cannot see these shapes,
          so the first read of a half that holds one names it; a one-word row beside each keeps the copies' part."""
import pytest

import faults as F
import oracle
import verdict as V
from test_ring_kernels import DEADLINE_MS, DEFAULT_TILE

pytestmark = pytest.mark.gpu

MASK = F.U64
SEED = 0x5EED_F00D_0000_0001
CANARY = 0xCA4A_8D00_0000_0007
T = DEFAULT_TILE
SIZES = [T - 16, T + 16, 7 * T + 48, (64 << 10) + 16, (3 << 20) + 112]     # ring and LDG-tile edges, ragged tails
SEED_BASE = 0x00C0FFEE00000000


def _place(seed, bit, dirs, stride, n, near_end):
    """A run of the directions asked for that fits in n words, near the end (the ragged tail) or near the start."""
    span = (len(dirs) - 1) * stride + 1
    start = max(0, n - span - 512) if near_end else 0
    a = F.find_directions(seed, bit, dirs, start=start, stride=stride, limit=n - span - start + 1)
    return a


def _shapes(seed, n, near_end):
    """(name, faults, blind) of each shape on the pattern of seed over n words: the fold-blind ones, stuck-at runs of
    bit 63 with an even and an odd number of changed words, and a single flip."""
    out = []
    a = n - 2 if near_end else 0
    out.append(("bit 63 pair", [F.xor_run(a, 1 << 63, 2)], True))
    a = _place(seed, 62, (1, -1), 2, n, near_end)
    out.append(("bit 62 opposite pair two apart", [F.xor_run(a, 1 << 62), F.xor_run(a + 2, 1 << 62)], True))
    a = _place(seed, 17, (1, -1, -1, 1), 1, n, near_end)
    out.append(("bit 17 +--+", [F.xor_run(a, 1 << 17, 4)], True))
    for value in (0, 1):
        for parity in (0, 1):
            first = max(0, n - 40) if near_end else 0
            for count in range(2, 40):
                wrong = sum(oracle.pattern_word(seed, i) >> 63 != value for i in range(first, first + count))
                if wrong and wrong % 2 == parity:
                    out.append(("bit 63 stuck at %d, %d words changed" % (value, wrong), [F.stuck_run(first, count, 63, value)],
                                parity == 0))
                    break
    out.append(("one word", [F.xor_run(n // 2, 1 << 40)], False))
    return out


def _force(faults):
    """cro_selftest_sweep's force ranges and XOR flag for faults of one kind."""
    xor = all(f[2] == MASK and f[3] == 0 for f in faults)
    return [(f[0], f[1], f[2], f[4] if xor else f[3]) for f in faults], xor


KERNELS = ["READ_LDG", "READ_TMA", "READ_LDG256", "COPY_FUSED"]


@pytest.mark.parametrize("n_bytes", SIZES)
def test_kernels_fold_and_count_the_faulted_words(cro, n_bytes):
    n = n_bytes // 8
    clean = oracle.checksum_np(SEED, 0, n)
    fails, blind_seen = [], 0
    with cro.ProbeContext(sweep_bytes=1 << 20, devices=[0], flags=cro.F_LAZY_ALLOC, deadline_ms=DEADLINE_MS) as c:
        for kname in KERNELS:
            kernel = getattr(cro, "SELFTEST_SWEEP_" + kname)
            copy = kname == "COPY_FUSED"
            layout = cro.SELFTEST_LAYOUT_SRC_DST if copy else 0
            out, _, _ = c.selftest_sweep(0, kernel, n_bytes, layout=layout, seed=SEED, canary=CANARY)
            if out.sweep.checksum != clean or (not copy and out.mismatches != 0):
                fails.append("%s clean: fold %s, %d mismatches" % (kname, out.sweep.checksum, out.mismatches))
            for near_end in (False, True):
                for name, fl, blind in _shapes(SEED, n, near_end):
                    force, xor = _force(fl)
                    out, _, _ = c.selftest_sweep(0, kernel, n_bytes, layout=layout, seed=SEED, canary=CANARY, force=force, xor=xor)
                    want, count = F.faulted_fold(SEED, n, fl), F.word_mismatches(SEED, n, fl)
                    assert (want == clean) == blind, (name, n)               # the shape is what it says it is
                    what = "%s, %s%s" % (kname, name, " near the end" if near_end else "")
                    if out.sweep.checksum != want:
                        fails.append("%s: fold %s, not %s" % (what, out.sweep.checksum, want))
                    if not copy and out.mismatches != count:
                        fails.append("%s: counted %d mismatches, not %d" % (what, out.mismatches, count))
                    if copy and out.after(1) != want:
                        fails.append("%s: the destination folds to %s, not %s" % (what, out.after(1), want))
                    blind_seen += blind and not copy and out.mismatches == count > 0
    assert not fails, "\n".join(["%d bytes" % n_bytes] + fails)
    assert blind_seen >= 3 * 2 * 4


# ---- the probe --------------------------------------------------------------------------------------------------------
def _read_half(C, i):
    return 0 if C == 0 else (C & 1 if i % 2 == 0 else 1 - (C & 1))


def _restated(seed, n, C, R, after, run):
    """(status, fail_code, fail_index, copy_verified) oracle/verdict.py gives for the slots of a probe whose run of
    faults (region words) is injected behind sweep `after`: the fill writes half A, copy i copies half i & 1 into the
    other half and folds its source, read i folds and compares read_half(C, i)."""
    halves = [[], []]
    first, count, mask = run

    def inject(k):
        if k == after:
            h = first // n
            halves[h] = halves[h] + [F.xor_run(first - h * n, mask, count)]
    E = oracle.checksum_np(seed, 0, n)
    sl = [V.ARMED] * V.SLOT_COUNT
    sl[V.SLOT_FILL] = V.Slot(0, 0, 0, 0, 1, 0, n)
    sl[V.SLOT_EXPECT] = V.Slot(*E, 0, 1, 0, n)
    inject(0)
    for i in range(C):
        s = i & 1
        sl[V.SLOT_SWEEP0 + i] = V.Slot(*F.faulted_fold(seed, n, halves[s]), 0, 1, 0, n)
        halves[1 - s] = list(halves[s])
        inject(1 + i)
    for i in range(R):
        h = _read_half(C, i)
        sl[V.SLOT_SWEEP0 + C + i] = V.Slot(*F.faulted_fold(seed, n, halves[h]), 0, 1, 0, n, F.word_mismatches(seed, n, halves[h]))
        inject(1 + C + i)
    r = V.Result(V.probe_finalize(bytes(512), sl, seed, 0, 8 * n, R, C, 1, V.COPY_TMA_FUSED))
    return r.get("status"), r.get("fail_code"), r.get("fail_index"), r.get("copy_verified")


S = 4 << 20
N = S // 8
R = 2


@pytest.fixture(scope="module")
def probe_seed(cro, coracle):
    with cro.ProbeContext(sweep_bytes=1 << 20, devices=[0], flags=cro.F_LAZY_ALLOC) as c:
        d = c.own_devices()[0]
    return coracle.probe_seed(SEED_BASE, max(d.device_minor, 0), 0)       # a new context's first probe


def _probe_runs(seed, half):
    """(name, (region word, count, mask), blind) of the probe-level shapes in one half.  One XOR run each: the bit 62
    shape is a run of four in the directions +, -, +, - (blind at bit 62, tests/test_fold_blind_spots.py)."""
    base = half * N + 1000
    rel = lambda a: half * N + a                                           # noqa: E731
    return [
        ("bit 63 pair", (base, 2, 1 << 63), True),
        ("bit 62 +-+-", (rel(F.find_directions(seed, 62, (1, -1, 1, -1), start=5000)), 4, 1 << 62), True),
        ("bit 29 +--+", (rel(F.find_directions(seed, 29, (1, -1, -1, 1), start=N - 4000)), 4, 1 << 29), True),
        ("one word", (base, 1, 1 << 33), False),
    ]


@pytest.mark.parametrize("rv", ["READ_LDG", "READ_TMA", "READ_LDG256"])
@pytest.mark.parametrize("C", [3, 2, 0])
def test_probe_names_the_read_that_sees_a_fold_blind_fault(cro, coracle, probe_seed, C, rv):
    fails, caught = [], set()
    for after in range(1 + C + R):
        half = after & 1
        for name, run, blind in _probe_runs(probe_seed, half):
            want = _restated(probe_seed, N, C, R, after, run)
            if blind:                    # no copy sees it; a read of a half that holds it always does
                assert want[1] in (V.FAIL_NONE, V.FAIL_READ), (name, after, want)
            flags = cro.F_SKIP_COPY if C == 0 else 0
            with cro.ProbeContext(sweep_bytes=S, devices=[0], flags=flags, read_sweeps=R, copy_sweeps=C or 1,
                                  read_variant=getattr(cro, rv), inject=(after, run[0], run[2], run[1])) as c:
                r = c.probe_device(0, allow_checksum_error=True)
            assert r.seed == probe_seed and r.read_variant == getattr(cro, rv)
            got = (r.status, r.fail_code, r.fail_index, r.copy_verified)
            if got != want:
                fails.append("%s after sweep %d (half %d): device %s, restatement %s" % (name, after, half, got, want))
            if blind and want[1] == V.FAIL_READ:
                caught.add(name)
    assert not fails, "\n".join(["C=%d, %s" % (C, rv)] + fails)
    assert caught == {"bit 63 pair", "bit 62 +-+-", "bit 29 +--+"}
