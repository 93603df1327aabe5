"""The multi-word faults the probe's fold cannot see, worked on the CPU, and the word-by-word count that sees them.

Every sweep folds its words into (xor, wrapping sum, sum of w[i] * (2i + 1) mod 2^64) (DESIGN.md §3).  All three parts
are linear mod 2^64, so some faults of several words leave all three unchanged:
  - any even number of flips of bit 63, at any positions and in either direction (+-2^63 are the same number);
  - two flips of bit k in opposite directions at a distance that is a multiple of 2^(63 - k);
  - four flips of one bit k at words a .. a + 3 in the directions +, -, -, + (the weights' second difference is 0).
Each shape is placed on a seeded pattern with oracle/faults.py, and its fold is compared with the clean one while the
word count is not.  The limits are pinned too: a single flip, two same-direction flips of bit 62 and opposite flips at a
distance the rule does not allow are all seen by the fold."""
import random

import pytest

import faults as F
import oracle

N = 1 << 12                               # words of the region
SEEDS = [0x00C0FFEE00000000, 0x5EED_F00D_0000_0001, 0xD1B54A32D192ED03 * 7 & F.U64]
CLEAN = {seed: oracle.checksum_np(seed, 0, N) for seed in SEEDS}


def seen(seed, faults):
    """(fold differs from the clean fold, words that differ)"""
    return F.faulted_fold(seed, N, faults) != CLEAN[seed], F.word_mismatches(seed, N, faults)


# ---- the restated fold itself -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", SEEDS)
def test_faulted_fold_is_the_fold_of_the_faulted_words(seed):
    """faulted_fold against a plain fold of the words with the faults written in, for XOR and stuck-at runs that overlap."""
    fl = [F.xor_run(5, 1 << 40, 3), F.stuck_run(6, 9, 63, 1), F.stuck_run(0, 4, 0, 0), F.xor_run(N - 1, F.U64)]
    words = [oracle.pattern_word(seed, i) for i in range(N)]
    for first, count, a, o, x in fl:
        for i in range(first, first + count):
            words[i] = ((words[i] & a) | o) ^ x
    x = s = w = 0
    for i, v in enumerate(words):
        x, s, w = x ^ v, (s + v) & F.U64, (w + v * (2 * i + 1)) & F.U64
    assert F.faulted_fold(seed, N, fl) == (x, s, w)
    assert F.word_mismatches(seed, N, fl) == sum(v != oracle.pattern_word(seed, i) for i, v in enumerate(words))
    assert F.word_mismatches(seed, N, [F.xor_run(3, 1 << 7), F.xor_run(3, 1 << 7)]) == 0      # two XORs undo each other


# ---- the blind classes --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", SEEDS)
def test_even_counts_of_bit_63_flips_are_blind(seed):
    rng = random.Random(seed)
    for k in (2, 4, 6, 64):
        idx = rng.sample(range(N), k)
        assert seen(seed, [F.xor_run(i, 1 << 63) for i in idx]) == (False, k), idx
        assert seen(seed, [F.xor_run(i, 1 << 63) for i in idx[:-1]]) == (True, k - 1), idx       # an odd count is seen
    assert seen(seed, [F.xor_run(100, 1 << 63, 2)]) == (False, 2)                               # a run of two


@pytest.mark.parametrize("seed", SEEDS)
def test_opposite_flips_at_a_multiple_of_2_to_the_63_minus_k_are_blind(seed):
    for bit, d in ((62, 2), (62, 10), (61, 4), (60, 8), (55, 256), (52, 2048)):
        a = F.find_directions(seed, bit, (1, -1), stride=d)
        assert seen(seed, [F.xor_run(a, 1 << bit), F.xor_run(a + d, 1 << bit)]) == (False, 2), (bit, d, a)
        b = F.find_directions(seed, bit, (-1, 1), stride=d)
        assert seen(seed, [F.xor_run(b, 1 << bit), F.xor_run(b + d, 1 << bit)]) == (False, 2), (bit, d, b)


@pytest.mark.parametrize("seed", SEEDS)
@pytest.mark.parametrize("bit", [0, 17, 33, 62, 63])
def test_four_flips_plus_minus_minus_plus_are_blind_at_any_bit(seed, bit):
    a = F.find_directions(seed, bit, (1, -1, -1, 1))
    assert seen(seed, [F.xor_run(a, 1 << bit, 4)]) == (False, 4)
    # the same shape as i, j, i + d, j + d
    i = F.find_directions(seed, bit, (1, -1), stride=37)
    j = F.find_directions(seed, bit, (-1, 1), start=i + 38, stride=37)
    assert seen(seed, [F.xor_run(w, 1 << bit) for w in (i, i + 37, j, j + 37)]) == (False, 4)


@pytest.mark.parametrize("seed", SEEDS)
def test_bit_62_runs_of_four_with_balanced_directions_are_blind(seed):
    """The probe hook XORs one contiguous run, so at bit 62 the opposite pair two words apart is placed as +, -, +, -:
    the pairs (a, a + 2) and (a + 1, a + 3) are each the same direction, but the whole is still blind at bit 62."""
    a = F.find_directions(seed, 62, (1, -1, 1, -1))
    assert seen(seed, [F.xor_run(a, 1 << 62, 4)]) == (False, 4)
    b = F.find_directions(seed, 61, (1, -1, 1, -1))              # at bit 61 the same directions are seen
    assert seen(seed, [F.xor_run(b, 1 << 61, 4)]) == (True, 4)


@pytest.mark.parametrize("seed", SEEDS)
@pytest.mark.parametrize("value", [0, 1])
def test_bit_63_stuck_over_a_run_is_blind_exactly_when_the_count_is_even(seed, value):
    """A data line stuck at bit 63: the words whose bit 63 disagrees change, and the fold sees them only when they are
    odd in number."""
    rng = random.Random(seed ^ value)
    parities = set()
    for _ in range(40):
        first, count = rng.randrange(N - 64), rng.randrange(1, 64)
        wrong = sum(oracle.pattern_word(seed, i) >> 63 != value for i in range(first, first + count))
        assert seen(seed, [F.stuck_run(first, count, 63, value)]) == (wrong % 2 == 1, wrong)
        parities.add(wrong % 2)
    assert parities == {0, 1}


# ---- the limits ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", SEEDS)
def test_single_flips_are_seen_at_every_bit(seed):
    for bit in range(64):
        assert seen(seed, [F.xor_run(bit * 31, 1 << bit)]) == (True, 1), bit


@pytest.mark.parametrize("seed", SEEDS)
def test_same_direction_bit_62_pairs_are_seen(seed):
    for d in (1, 2, 4, 100):
        for sign in (1, -1):
            a = F.find_directions(seed, 62, (sign, sign), stride=d)
            assert seen(seed, [F.xor_run(a, 1 << 62), F.xor_run(a + d, 1 << 62)]) == (True, 2), (d, sign)


@pytest.mark.parametrize("seed", SEEDS)
def test_opposite_flips_at_other_distances_are_seen(seed):
    for bit, d in ((62, 1), (62, 3), (61, 2), (61, 6), (55, 128), (40, 1 << 11)):
        assert d % (1 << (63 - bit)) != 0
        a = F.find_directions(seed, bit, (1, -1), stride=d)
        assert seen(seed, [F.xor_run(a, 1 << bit), F.xor_run(a + d, 1 << bit)]) == (True, 2), (bit, d)


def test_find_directions_finds_what_it_was_asked_for():
    seed = SEEDS[0]
    for bit, dirs, stride in ((5, (1, -1, -1, 1), 1), (62, (-1, 1), 2), (63, (1, 1, 1), 3)):
        a = F.find_directions(seed, bit, dirs, start=1000, stride=stride)
        assert a >= 1000
        assert [F.flip_direction(seed, a + m * stride, bit) for m in range(len(dirs))] == list(dirs)
        assert all([F.flip_direction(seed, b + m * stride, bit) for m in range(len(dirs))] != list(dirs) for b in range(1000, a))
    with pytest.raises(ValueError):
        F.find_directions(seed, 0, (1,) * 40, limit=4)
