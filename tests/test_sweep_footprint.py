"""Every sweep kernel touches exactly its own bytes: guard bands around the interior, at every ring setting.

The other GPU tests check the words a kernel was meant to touch.  A kernel that stores one vector or one tile past its
end, or folds a word before its start or after its end, passes them as long as nobody reads there.  cro_selftest_sweep
runs one kernel on a buffer of its own, [guard | interior(s) | guard] with each guard at least 2 MiB (more than any ring
a knob accepts, so a stray access stays inside the hook's allocation) and filled with canary words of its own, which
no word of the interior's pattern or of another guard repeats.  What a kernel writes starts as the complement of what
it should write.  Then:
  writers (fill, its complement, the three copies in three layouts, force_words, link write): every guard word is still
          the canary, the interior is the plain reference, a copy's source is unchanged, force_words changes exactly its
          range;
  readers (three reads, locate, link read): the fold is the oracle's checksum of exactly the interior (a folded guard
          word would change it), and the word-checking kernels count no mismatch on a clean interior (every guard word
          is one) and exactly the forced words on a forced one.
Interiors up to 8 MiB are compared word for word on the host; above that their folds (taken by the LDG read after the
kernel) are compared with the C oracle's checksum.

Each ring configuration of test_ring_kernels gets its own context, at each of its sizes, with the interior at three
offsets past a 2 MiB boundary.  Every context has a deadline."""
import ctypes
import functools
import os
import subprocess

import numpy as np
import pytest

import oracle                        # tests/conftest.py puts oracle/ on the path
from test_ring_kernels import CONFIGS, DEADLINE_MS, SIZES, _apply, _size

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MASK = (1 << 64) - 1
GUARD = 2 << 20
SEED = 0x5EED_F00D_0000_0001
CANARY = 0xCA4A_8D00_0000_0007       # the guards' stream: far from SEED, so no guard word repeats an interior word
OFFSETS = (0, 16, 112)
WORD_FOR_WORD = 8 << 20              # interiors up to this are copied back and compared word for word
WORD0 = (5 << 18) - 3                # locate's scan index of the interior's first word: 3 words below granule 5
FORCE_AND, FORCE_OR = 0x00FF00FF00FF00FF, 0x8000000000000001


@functools.lru_cache(maxsize=3)
def _canary(g):
    """Guard g's canary words: word j is pattern_word(CANARY, g * 2^32 + j).  No guard reaches three guard lengths."""
    return oracle.pattern_words_np(CANARY, g << 32, 3 * GUARD // 8)


@functools.lru_cache(maxsize=4)
def _pattern(n):
    return oracle.pattern_words_np(SEED, 0, n)


def _complement_fold(f, n):
    """The fold of the complement of n words from theirs: ~p = -1 - p, and the weights 2i + 1 of n words sum to n^2."""
    return f[0] ^ (MASK if n & 1 else 0), (-n - f[1]) & MASK, (-n * n - f[2]) & MASK


def _changed_fold(f, changes):
    """The fold after word i changed from old to new, for every (i, old, new)."""
    x, s, w = f
    for i, old, new in changes:
        d = (new - old) & MASK
        x, s, w = x ^ old ^ new, (s + d) & MASK, (w + d * (2 * i + 1)) & MASK
    return x, s, w


def _forced(old):
    return (old & FORCE_AND) | FORCE_OR


class Row:
    """One kernel's run on a guarded buffer: what it returned, and every check on it that failed, as one line each."""

    def __init__(self, ctx, name, kernel, n_bytes, offset, layout=0, **kw):
        self.name, self.n, self.fails = name, n_bytes // 8, []
        self.interiors = n_bytes <= WORD_FOR_WORD
        self.out, self.buf, self.words = ctx.selftest_sweep(
            0, kernel, n_bytes, offset=offset, layout=layout, seed=SEED, canary=CANARY, interiors=self.interiors,
            alloc=lambda nb: np.empty(nb // 8, dtype=np.uint64), **kw)
        self.at = [self.out.at[0] // 8, self.out.at[1] // 8]
        self._check_layout(n_bytes, offset, layout)
        self._check_guards()

    def fail(self, what):
        self.fails.append("%s: %s" % (self.name, what))

    def _check_layout(self, n_bytes, offset, layout):
        at, total = list(self.out.at), self.out.buf_bytes
        ok = total % GUARD == 0 and min(at) % GUARD == offset and min(at) >= GUARD + offset
        ok &= total - (max(at) + n_bytes) >= GUARD
        ok &= {0: at[0] == at[1], 1: at[1] == at[0] + n_bytes, 2: at[0] == at[1] + n_bytes,
               3: at[1] % GUARD == offset and at[1] >= at[0] + n_bytes + GUARD}[layout]
        if not ok:
            self.fail("layout %s of %d bytes" % (at, total))

    def _check_guards(self):
        """Every word outside the interiors is still its guard's canary."""
        start, g = 0, 0
        for a in sorted(set(self.at)) + [len(self.buf)]:
            if a > start:                                # adjacent interiors have no guard between them
                bad = np.flatnonzero(self.buf[start:a] != _canary(g)[:a - start])
                if bad.size:
                    self.fail("%d words of guard %d changed, the first %d words into it (interiors at words %s, %d "
                              "words each)" % (bad.size, g, bad[0], self.at, self.n))
                g += 1
            start = a + self.n

    def interior(self, k, want, want_fold):
        """Interior k (0: the one the kernel read, a copy's source; 1: a copy's destination) against the reference:
        its fold after the kernel, and word for word (want() is the array) when it was copied back."""
        if self.out.after(k) != want_fold:
            self.fail("interior %d folds to %s after the kernel, not %s" % (k, self.out.after(k), want_fold))
        if self.interiors:
            bad = np.flatnonzero(self.buf[self.at[k]:self.at[k] + self.n] != want())
            if bad.size:
                self.fail("interior %d: %d words differ, the first at word %d" % (k, bad.size, bad[0]))

    def fold(self, want):
        if self.out.sweep.checksum != want:
            self.fail("the kernel folded %s, not %s" % (self.out.sweep.checksum, want))

    def counts(self, mismatches, granules=(0, 0, 0)):
        """The word-checking kernels: exact count, record slots claimed (one per mismatch) and granules set."""
        o = self.out
        got = (o.mismatches, o.claims, (o.granules, o.granule_min, o.granule_max))
        if got != (mismatches, mismatches, tuple(granules)):
            self.fail("counted (mismatches, claims, (granules, min, max)) %s, not %s" % (got, (mismatches, mismatches, granules)))


def _rows(cro, ctx, want, S, offset):
    """Every kernel once on interiors of S bytes at `offset`; returns the failures.  want: the oracle's checksum of
    the pattern over S / 8 words."""
    n = S // 8
    pat = functools.partial(_pattern, n)
    comp = _complement_fold(want, n)
    rows = []

    def row(name, kernel, **kw):
        rows.append(Row(ctx, "%s, offset %d" % (name, offset), kernel, S, offset, **kw))
        return rows[-1]

    # writers
    row("fill", cro.SELFTEST_SWEEP_FILL).interior(0, pat, want)
    row("fill complement", cro.SELFTEST_SWEEP_FILL, invert=MASK).interior(0, lambda: ~pat(), comp)
    for kernel, kname in ((cro.SELFTEST_SWEEP_COPY_LDG, "ldg"), (cro.SELFTEST_SWEEP_COPY_TMA, "tma"),
                          (cro.SELFTEST_SWEEP_COPY_FUSED, "fused")):
        for layout, lname in ((cro.SELFTEST_LAYOUT_SRC_DST, "src|dst"), (cro.SELFTEST_LAYOUT_DST_SRC, "dst|src"),
                              (cro.SELFTEST_LAYOUT_APART, "src|guard|dst")):
            r = row("copy %s %s" % (kname, lname), kernel, layout=layout)
            r.interior(0, pat, want)                     # the source is unchanged
            r.interior(1, pat, want)                     # the destination is the source
            if kernel == cro.SELFTEST_SWEEP_COPY_FUSED:
                r.fold(want)                             # the checksumming copy's fold of its source
    first = n // 3
    count = min(n - first, 1000)
    olds = [oracle.pattern_word(SEED, first + i) for i in range(count)]

    def forced_range():
        w = pat().copy()
        w[first:first + count] = [_forced(o) for o in olds]
        return w
    row("force_words [%d, %d)" % (first, first + count), cro.SELFTEST_SWEEP_FORCE_WORDS,
        force=[(first, count, FORCE_AND, FORCE_OR)]).interior(
        0, forced_range, _changed_fold(want, [(first + i, o, _forced(o)) for i, o in enumerate(olds)]))
    row("link write", cro.SELFTEST_SWEEP_LINK_WRITE).interior(0, pat, want)

    # readers
    for kernel, kname in ((cro.SELFTEST_SWEEP_READ_LDG, "ldg"), (cro.SELFTEST_SWEEP_READ_TMA, "tma"),
                          (cro.SELFTEST_SWEEP_READ_LDG256, "ldg256")):
        r = row("read " + kname, kernel)
        r.fold(want)
        r.interior(0, pat, want)
    r = row("link read", cro.SELFTEST_SWEEP_LINK_READ)
    r.fold(want)
    r.counts(0)
    r.interior(0, pat, want)
    # a clean interior as the scan's complement pass meets it, then one whose first and last words are forced
    r = row("locate clean", cro.SELFTEST_SWEEP_LOCATE, word0=WORD0, invert=MASK)
    r.fold(comp)
    r.counts(0)
    r.interior(0, lambda: ~pat(), comp)
    ends = [0, n - 1]
    olds = [oracle.pattern_word(SEED, i) for i in ends]
    assert all(_forced(o) != o for o in olds)
    changed = [(i, o, _forced(o)) for i, o in zip(ends, olds)]
    grans = sorted({(WORD0 + i) * 8 // cro.LOCATE_GRANULE_BYTES for i in ends})

    def forced_ends():
        w = pat().copy()
        w[ends] = [_forced(o) for o in olds]
        return w
    r = row("locate forced ends", cro.SELFTEST_SWEEP_LOCATE, word0=WORD0,
            force=[(0, 1, FORCE_AND, FORCE_OR), (n - 1, 1, FORCE_AND, FORCE_OR)])
    r.fold(_changed_fold(want, changed))
    r.counts(2, (len(grans), grans[0], grans[-1]))
    r.interior(0, forced_ends, _changed_fold(want, changed))
    got = [(w.word_index, w.expected, w.actual, w.passes) for w in r.words]
    if got != [(WORD0 + i, o, f, 1) for i, o, f in changed]:
        r.fail("records %s" % [tuple(hex(v) for v in g) for g in got])
    return [f for r in rows for f in r.fails]


@pytest.mark.gpu
@pytest.mark.parametrize("label", SIZES)
@pytest.mark.parametrize("name", list(CONFIGS))
def test_sweep_footprint(cro, coracle, monkeypatch, name, label):
    T, D = _apply(monkeypatch, cro, CONFIGS[name])
    assert cro.validate_env() == ""
    S = _size(label, T, D, name)
    want = coracle.checksum(SEED, 0, S // 8, threads=os.cpu_count() or 1)
    fails = []
    with cro.ProbeContext(sweep_bytes=1 << 20, devices=[0], flags=cro.F_LAZY_ALLOC, deadline_ms=DEADLINE_MS) as c:
        for offset in OFFSETS:
            fails += _rows(cro, c, want, S, offset)
    assert not fails, "\n".join(["S = %d bytes, tile %d, %d stages" % (S, T, D)] + fails)


@pytest.mark.gpu
def test_invalid_arguments_are_refused(cro):
    with cro.ProbeContext(sweep_bytes=1 << 20, devices=[0], flags=cro.F_LAZY_ALLOC, deadline_ms=DEADLINE_MS) as c:
        # [2 MiB guard | 4 KiB | the rest of that 2 MiB and one more]
        out, buf, _ = c.selftest_sweep(0, cro.SELFTEST_SWEEP_FILL, 4096, seed=SEED, canary=CANARY)
        assert out.buf_bytes == 3 * GUARD and len(buf) == 3 * GUARD and list(out.at) == [GUARD, GUARD]
        for kernel, n_bytes, kw in [
            (cro.SELFTEST_SWEEP_FILL, 4096, dict(offset=8)),                          # offset not a multiple of 16
            (cro.SELFTEST_SWEEP_FILL, 4096, dict(offset=GUARD)),                      # offset past the guard
            (cro.SELFTEST_SWEEP_FILL, 0, {}),                                          # empty interior
            (cro.SELFTEST_SWEEP_READ_TMA, 4104, {}),                                   # not a multiple of 16
            (0, 4096, {}), (12, 4096, {}),                                             # unknown kernels
            (cro.SELFTEST_SWEEP_READ_LDG, 4096, dict(layout=cro.SELFTEST_LAYOUT_SRC_DST)),   # a layout for a non-copy
            (cro.SELFTEST_SWEEP_LOCATE, 4096, dict(layout=cro.SELFTEST_LAYOUT_APART)),
            (cro.SELFTEST_SWEEP_COPY_TMA, 4096, {}),                                   # a copy without a layout
            (cro.SELFTEST_SWEEP_COPY_LDG, 4096, dict(layout=4)),
            (cro.SELFTEST_SWEEP_READ_LDG, 4096, dict(invert=MASK)),                    # invert is the fill's / locate's
            (cro.SELFTEST_SWEEP_FILL, 4096, dict(invert=1)),
            (cro.SELFTEST_SWEEP_FILL, 4096, dict(word0=1)),                            # word0 is locate's
            (cro.SELFTEST_SWEEP_LOCATE, 4096, dict(word0=(1 << 37) - 511)),           # granule bitmap past 2^37 words
            (cro.SELFTEST_SWEEP_READ_LDG, 4096, dict(force=[(0, 1, 0, 0)])),          # force ranges are locate's ...
            (cro.SELFTEST_SWEEP_FORCE_WORDS, 4096, dict(force=[(0, 1, 0, 0), (1, 1, 0, 0)])),   # ... force_words' first
            (cro.SELFTEST_SWEEP_LOCATE, 4096, dict(force=[(500, 13, 0, 0)])),        # past the interior's 512 words
        ]:
            with pytest.raises(cro.ProbeError) as e:
                c.selftest_sweep(0, kernel, n_bytes, seed=SEED, canary=CANARY, **kw)
            assert e.value.code == cro.ERR_INVALID_ARG, (kernel, n_bytes, kw)
            assert "cro_selftest_sweep: " in str(e.value), (kernel, n_bytes, kw)
        # a short buffer is refused before anything runs, with the size it needs
        o, out = cro.SelftestSweepOpts(), cro.SelftestSweepOut()
        o.kernel, o.bytes = cro.SELFTEST_SWEEP_FILL, 4096
        n = ctypes.c_int()
        small = ctypes.create_string_buffer(GUARD)
        assert cro.lib.cro_selftest_sweep(c.handle, 0, ctypes.byref(o), ctypes.byref(out), small, GUARD, None, 0,
                                          ctypes.byref(n)) == cro.ERR_BUFFER_SMALL
        assert out.buf_bytes == 3 * GUARD
        assert cro.lib.cro_selftest_sweep(c.handle, 1 << 20, ctypes.byref(o), ctypes.byref(out), small, GUARD, None, 0,
                                          ctypes.byref(n)) == cro.ERR_INVALID_ARG


# ---- without a GPU ----------------------------------------------------------------------------------------------
def test_selftest_sweep_without_a_context_is_refused(cro):
    o, out = cro.SelftestSweepOpts(), cro.SelftestSweepOut()
    o.kernel, o.bytes = cro.SELFTEST_SWEEP_FILL, 4096
    n = ctypes.c_int(-1)
    buf = ctypes.create_string_buffer(16)
    assert cro.lib.cro_selftest_sweep(None, 0, ctypes.byref(o), ctypes.byref(out), buf, 16, None, 0,
                                      ctypes.byref(n)) == cro.ERR_INVALID_ARG
    assert cro.lib.cro_selftest_sweep(None, 0, None, None, None, 0, None, 0, None) == cro.ERR_INVALID_ARG


def test_ctypes_layout_and_constants_match_the_header(cro, tmp_path):
    fields = {
        "cro_selftest_sweep_opts": ("SelftestSweepOpts", ["kernel", "layout", "offset", "bytes", "seed", "canary", "invert",
                                                          "word0", "force_first", "force_count", "force_and", "force_or",
                                                          "flags", "reserved"]),
        "cro_selftest_sweep_out": ("SelftestSweepOut", ["sweep", "buf_bytes", "at", "after_xor", "after_sum", "after_wsum",
                                                        "mismatches", "claims", "granules", "granule_min", "granule_max"]),
    }
    consts = ["CRO_SELFTEST_SWEEP_" + k for k in ("FILL", "COPY_LDG", "COPY_TMA", "COPY_FUSED", "READ_LDG", "READ_TMA",
                                                    "READ_LDG256", "LOCATE", "FORCE_WORDS", "LINK_READ", "LINK_WRITE")]
    consts += ["CRO_SELFTEST_LAYOUT_SRC_DST", "CRO_SELFTEST_LAYOUT_DST_SRC", "CRO_SELFTEST_LAYOUT_APART",
               "CRO_SELFTEST_GUARD_BYTES", "CRO_SELFTEST_F_INTERIORS"]
    src = ['#include <stdio.h>', '#include <stddef.h>', '#include "croprobe.h"', "int main(void) {"]
    for cname, (_py, fl) in fields.items():
        src.append('printf("%s sizeof %%zu\\n", sizeof(%s));' % (cname, cname))
        src += ['printf("%s %s %%zu\\n", offsetof(%s, %s));' % (cname, f, cname, f) for f in fl]
    src += ['printf("const %s %%lld\\n", (long long)(%s));' % (k, k) for k in consts]
    src.append("return 0; }")
    c = tmp_path / "layout.c"
    c.write_text("\n".join(src))
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-std=c11", "-I" + os.path.join(ROOT, "include"), str(c), "-o", str(exe)])
    got = {}
    for ln in subprocess.check_output([str(exe)], text=True).splitlines():
        name, field, v = ln.split()
        got[(name, field)] = int(v)
    for cname, (py, fl) in fields.items():
        cls = getattr(cro, py)
        assert ctypes.sizeof(cls) == got[(cname, "sizeof")], cname
        for f in fl:
            assert getattr(cls, f).offset == got[(cname, f)], (cname, f)
    for k in consts:
        assert getattr(cro, k[len("CRO_"):]) == got[("const", k)], k
