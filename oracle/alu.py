"""Restatement of the ALU probe (cro_probe_alu) from the PTX ISA: the table's operands from the call's seed, each form's
exact result, the closed form of the fold and what a test injection makes.  Python integers for the integer forms and
fractions.Fraction for the rounding, so nothing is shared with the library's C++.  The classification and the
annotations are the cross-lane probe's (oracle/xlane.py) under the ALU's own names."""
from __future__ import annotations

from fractions import Fraction
from typing import Dict, List, Tuple

import xlane
from oracle import go_marshal_string_map, pattern_word

U32, U64 = (1 << 32) - 1, (1 << 64) - 1
LEGS, THREADS, WARPS = 5, 256, 8
LOGIC, SHIFT, IADD, IMUL, FLOAT = range(5)
FORMS = [269, 19, 50, 25, 45]
ROWS = [2, 4, 4, 4, 8]
OPS = [f * r for f, r in zip(FORMS, ROWS)]
NAMES = ["logic", "shift", "iadd", "imul", "float"]
STRIDE = 0xD1B54A32D192ED03
SEED_OFFSET = 1 << 53


def call_seed(seed_dev: int, k: int) -> int:
    return (seed_dev + SEED_OFFSET + k * STRIDE) & U64


def s32(x: int) -> int:
    x &= U32
    return x - (1 << 32) if x >> 31 else x


def sx(x: int, bits: int) -> int:
    x &= (1 << bits) - 1
    return x - (1 << bits) if x >> (bits - 1) else x


# ---- operands ------------------------------------------------------------------------------------------------------
def word(seed, leg, op, k, t):
    return pattern_word(seed, (((leg * 1024 + op) * 8 + k) << 8) | t)


def mix32(x):
    sel = x >> 61
    if sel == 4:
        return [0, U32, 0x80000000, 0x7FFFFFFF][(x >> 32) & 3]
    if sel == 5:
        return 1 << (x & 31)
    if sel == 6:
        return ~(1 << (x & 31)) & U32
    if sel == 7:
        return ((x & 15) - 8) & U32
    return x & U32


def mix64(x):
    sel = x >> 61
    if sel == 4:
        return [0, U64, 1 << 63, (1 << 63) - 1][(x >> 32) & 3]
    if sel == 5:
        return 1 << (x & 63)
    if sel == 6:
        return ~(1 << (x & 63)) & U64
    if sel == 7:
        return ((x & 15) - 8) & U64
    return x


def count(x):
    return x & 63 if x >> 62 else x & U32


# ---- IEEE binary32 / binary64 from the definition -----------------------------------------------------------------
class Fmt:
    def __init__(self, p, ebits):
        self.p, self.ebits = p, ebits
        self.bias = (1 << (ebits - 1)) - 1
        self.top = (1 << ebits) - 1
        self.fmask = (1 << (p - 1)) - 1
        self.sign = 1 << (p - 1 + ebits)


F32, F64 = Fmt(24, 8), Fmt(53, 11)
RN, RZ, RM, RP = range(4)


def fbits(f, sign, biased, frac):
    return ((sign & 1) << (f.p - 1 + f.ebits)) | (biased << (f.p - 1)) | (frac & f.fmask)


def fexp(f, b):
    return (b >> (f.p - 1)) & f.top


def is_nan(f, b):
    return fexp(f, b) == f.top and b & f.fmask != 0


def is_zero(f, b):
    return b & ~f.sign == 0


def value(f, b) -> Fraction:
    """The finite value of b."""
    e, frac = fexp(f, b), b & f.fmask
    m = Fraction(frac, 1 << (f.p - 1)) if e == 0 else 1 + Fraction(frac, 1 << (f.p - 1))
    v = m * Fraction(2) ** ((1 if e == 0 else e) - f.bias)
    return -v if b & f.sign else v


def round_to(f, v: Fraction, mode: int, zero_sign: int) -> int:
    """v rounded to the format in the mode (IEEE 754 with unbounded exponent then overflow; subnormals kept); an
    exact zero takes zero_sign."""
    if v == 0:
        return fbits(f, zero_sign, 0, 0)
    neg = v < 0
    a = -v if neg else v
    e = a.numerator.bit_length() - a.denominator.bit_length()
    while Fraction(2) ** e > a:
        e -= 1
    while Fraction(2) ** (e + 1) <= a:
        e += 1
    q = max(e, 1 - f.bias) - (f.p - 1)                     # exponent of the result's lsb
    scaled = a / Fraction(2) ** q
    m = scaled.numerator // scaled.denominator
    rest = scaled - m
    if rest:
        if mode == RN:
            m += 1 if rest > Fraction(1, 2) or (rest == Fraction(1, 2) and m % 2) else 0
        elif mode == RM:
            m += 1 if neg else 0
        elif mode == RP:
            m += 0 if neg else 1
    if m == 1 << f.p:
        m >>= 1
        q += 1
    if q + (f.p - 1) > f.top - 1 - f.bias:                 # past the largest finite exponent
        inf = mode == RN or (mode == RM and neg) or (mode == RP and not neg)
        return fbits(f, neg, f.top, 0) if inf else fbits(f, neg, f.top - 1, f.fmask)
    if m < 1 << (f.p - 1):
        return fbits(f, neg, 0, m)
    return fbits(f, neg, q + (f.p - 1) + f.bias, m)


def f_add(f, a, b, mode):
    sa, sb = a >> (f.p - 1 + f.ebits), b >> (f.p - 1 + f.ebits)
    v = value(f, a) + value(f, b)
    if v == 0:   # x + (-x) is +0 but -0 rounding down; (-0) + (-0) is -0
        zs = sa if sa == sb and is_zero(f, a) and is_zero(f, b) else (1 if mode == RM else 0)
        return round_to(f, v, mode, zs)
    return round_to(f, v, mode, 0)


def f_mul(f, a, b, mode):
    s = (a ^ b) >> (f.p - 1 + f.ebits) & 1
    return round_to(f, value(f, a) * value(f, b), mode, s)


def f_fma(f, a, b, c, mode):
    ps = (a ^ b) >> (f.p - 1 + f.ebits) & 1
    cs = c >> (f.p - 1 + f.ebits) & 1
    pv = value(f, a) * value(f, b)
    v = pv + value(f, c)
    if v == 0:
        zs = ps if pv == 0 and is_zero(f, c) and ps == cs else (1 if mode == RM else 0)
        return round_to(f, v, mode, zs)
    return round_to(f, v, mode, 0)


# operand classes (the table's construction; DESIGN.md "The ALU probe")
def f_any(f, x):
    return fbits(f, x >> 63, 1 + (x >> 32) % ((1 << f.ebits) - 2), x)


def f_near(f, x, off, spread):
    return fbits(f, x >> 63, f.bias + off - spread + (x >> 40) % (2 * spread + 1), x)


def f_tiny(f, x):
    return fbits(f, x >> 63, (x >> 40) % 3, x)


def f_huge(f, x):
    return fbits(f, x >> 63, (1 << f.ebits) - 2 - (x >> 40) % 3, x)


def f_special(f, x, inf):
    top, ones = f.top, f.fmask
    v = [0, 0, top - 1, top - 1, 1, 0, 1, 0, f.bias, top if inf else f.bias]
    fr = [0, 0, ones, ones, 0, 1, ones, ones, 0, 0]
    i = (x >> 32) % 10
    return fbits(f, x >> 63, v[i], fr[i])


def f_short(f, x):
    keep = 11 if f.p == 24 else 26
    return f_near(f, x & ~((1 << (f.p - 1 - keep)) - 1) & U64, 0, 8)


def f_nan(f, x):
    return fbits(f, x >> 63, f.top, (1 << (f.p - 2)) | x)


def f_arith(f, sc, fma, s):
    o = [0, 0, 0]
    if sc == 0:
        o = [f_any(f, s[k]) for k in range(3)]
    elif sc == 1:
        o = [f_near(f, s[k], 0, 3) for k in range(3)]
    elif sc == 2:
        o[0] = f_near(f, s[0], 0, 20)
        for k in (1, 2):
            o[k] = fbits(f, s[k] >> 63, fexp(f, o[0]) - (f.p - 1) - (s[k] >> 40) % 3, [0, 1, f.fmask][(s[k] >> 50) % 3])
    elif sc == 3:
        o[0], o[1] = f_near(f, s[0], 0, 30), f_near(f, s[1], 0, 30)
        base = f_mul(f, o[0], o[1], RN) if fma else o[0]
        fr, dl = base & f.fmask, (s[2] >> 40) % 3
        v = base
        if dl == 1 and fr != f.fmask:
            v = base + 1
        if dl == 2 and fr != 0:
            v = base - 1
        if (s[2] >> 50) & 1 or fma:
            v ^= f.sign
        if fma:
            o[2] = v
        else:
            o[1], o[2] = v, f_near(f, s[2], 0, 3)
    elif sc == 4:
        o = [f_tiny(f, s[0]), f_tiny(f, s[1]) if (s[1] >> 62) & 1 else f_near(f, s[1], 0, 12), f_tiny(f, s[2])]
    elif sc == 5:
        o = [f_huge(f, s[0]), f_huge(f, s[1]) if (s[1] >> 62) & 1 else f_near(f, s[1], 0, 1), f_huge(f, s[2])]
    elif sc == 6:
        o = [f_special(f, s[k], False) for k in range(3)]
    else:
        o = [f_short(f, s[k]) for k in range(3)]
    return o


def f_cmp(x):
    c = (x >> 58) % 8
    if c < 2:
        return f_any(F32, x)
    if c == 2:
        return f_near(F32, x, 0, 2)
    if c == 3:
        return f_tiny(F32, x)
    if c < 6:
        return f_special(F32, x, True)
    return f_nan(F32, x)


def fsetp(i, a, b):
    """setp.f32 comparison i (eq ne lt le gt ge equ neu ltu leu gtu geu num nan) from the ISA's table."""
    un = is_nan(F32, a) or is_nan(F32, b)
    if i == 12:
        return not un
    if i == 13:
        return un
    if un:
        return i >= 6
    inf = Fraction(2) ** 200

    def v(x):
        return (-inf if x & F32.sign else inf) if fexp(F32, x) == 255 else value(F32, x)
    x, y = v(a), v(b)
    return [x == y, x != y, x < y, x <= y, x > y, x >= y][i % 6]


def fminmax(i, a, b):
    """min max min.NaN max.NaN min.xorsign.abs max.xorsign.abs .f32."""
    an, bn = is_nan(F32, a), is_nan(F32, b)
    if i in (2, 3) and (an or bn):
        return 0x7FFFFFFF                                   # the canonical NaN
    if an and bn:
        return 0x7FFFFFFF
    if an:
        return b
    if bn:
        return a
    if i >= 4:
        ma, mb = a & 0x7FFFFFFF, b & 0x7FFFFFFF
        lt = fsetp(2, ma, mb)
        m = (mb if lt else ma) if i == 5 else (ma if lt else mb)
        return m | ((a ^ b) & 0x80000000)
    lt = fsetp(2, a, b)
    return (b if lt else a) if i % 2 else (a if lt else b)


# ---- integer forms -------------------------------------------------------------------------------------------------
def bits_of(x, n):
    return [(x >> i) & 1 for i in range(n)]


def lop3(lut, a, b, c):
    return sum(((lut >> ((x << 2) | (y << 1) | z)) & 1) << i for i, (x, y, z) in enumerate(zip(bits_of(a, 32), bits_of(b, 32), bits_of(c, 32))))


def bmsk(a, b, clamp):
    """bmsk: a mask of width b from bit a (PTX ISA semantics, .clamp and .wrap)."""
    a1, b1 = a & 31, b & 31
    mask0 = (U32 << a1) & U32
    total = a1 + b1
    mask1 = (U32 << total) & U32 if total < 32 else 0
    over = total >= 32
    if clamp:
        if a >= 32:
            over, mask0 = True, 0
        if b >= 32:
            over = True
    if over:
        mask1 = 0
    elif b1 == 0:
        mask1 = U32
    return mask0 & ~mask1 & U32


def bfind(a, sgn, shiftamt):
    if sgn and a >> 31:
        a = ~a & U32
    if a == 0:
        return U32
    d = a.bit_length() - 1
    return 31 - d if shiftamt else d


def szext(a, b, clamp, sgn):
    b1 = b & 31
    big = clamp and b >= 32
    if big:
        return a
    mask = (U32 << b1) & U32
    sign = sgn and b1 != 0 and (a >> (b1 - 1)) & 1
    return (a & ~mask & U32) | (mask if sign else 0)


PRMT_MODES = [  # d.b0 .. d.b3 per selector c[1:0]: f4e b4e rc8 ecl ecr rc16
    [[0, 1, 2, 3], [1, 2, 3, 4], [2, 3, 4, 5], [3, 4, 5, 6]],
    [[0, 7, 6, 5], [1, 0, 7, 6], [2, 1, 0, 7], [3, 2, 1, 0]],
    [[0, 0, 0, 0], [1, 1, 1, 1], [2, 2, 2, 2], [3, 3, 3, 3]],
    [[0, 1, 2, 3], [1, 1, 2, 3], [2, 2, 2, 3], [3, 3, 3, 3]],
    [[0, 0, 0, 0], [0, 1, 1, 1], [0, 1, 2, 2], [0, 1, 2, 3]],
    [[0, 1, 0, 1], [2, 3, 2, 3], [0, 1, 0, 1], [2, 3, 2, 3]],
]


def prmt(a, b, c, mode):
    by = [((b << 32 | a) >> (8 * i)) & 0xFF for i in range(8)]
    d = 0
    for i in range(4):
        if mode is None:
            sel = (c >> (4 * i)) & 15
            v = by[sel & 7]
            if sel & 8:
                v = 0xFF if v & 0x80 else 0
        else:
            v = by[PRMT_MODES[mode][c & 3][i]]
        d |= v << (8 * i)
    return d


def halves(a, b, c, sgn, g):
    d = 0
    for h in range(2):
        ext = (lambda v: sx(v >> (16 * h), 16)) if sgn else (lambda v: (v >> (16 * h)) & 0xFFFF)
        d |= (g(ext(a), ext(b), ext(c)) & 0xFFFF) << (16 * h)
    return d


def relu(x):
    return max(x, 0)


def minmax(i, a, b):
    ops = [lambda: min(a, b), lambda: max(a, b), lambda: min(s32(a), s32(b)), lambda: max(s32(a), s32(b)),
           lambda: relu(min(s32(a), s32(b))), lambda: relu(max(s32(a), s32(b))),
           lambda: halves(a, b, 0, False, lambda x, y, z: min(x, y)), lambda: halves(a, b, 0, False, lambda x, y, z: max(x, y)),
           lambda: halves(a, b, 0, True, lambda x, y, z: min(x, y)), lambda: halves(a, b, 0, True, lambda x, y, z: max(x, y)),
           lambda: halves(a, b, 0, True, lambda x, y, z: relu(min(x, y))), lambda: halves(a, b, 0, True, lambda x, y, z: relu(max(x, y)))]
    return ops[i]() & U32


def dpx(i, a, b, c):
    pick = max if i % 2 == 0 else min
    kind = (i % 12) // 2
    if i < 12:
        return [lambda: pick(pick(s32(a), s32(b)), s32(c)), lambda: pick(pick(a, b), c),
                lambda: relu(pick(pick(s32(a), s32(b)), s32(c))),
                lambda: halves(a, b, c, True, lambda x, y, z: pick(pick(x, y), z)),
                lambda: halves(a, b, c, False, lambda x, y, z: pick(pick(x, y), z)),
                lambda: halves(a, b, c, True, lambda x, y, z: relu(pick(pick(x, y), z)))][kind]() & U32
    return [lambda: pick(s32(a + b), s32(c)), lambda: pick((a + b) & U32, c), lambda: relu(pick(s32(a + b), s32(c))),
            lambda: halves(a, b, c, True, lambda x, y, z: pick(sx(x + y, 16), z)),
            lambda: halves(a, b, c, False, lambda x, y, z: pick((x + y) & 0xFFFF, z))][kind]() & U32


def dp(a, b, c, asg, bsg, two):
    """dp4a (two None) and dp2a.lo / .hi (two 0 / 1): c plus the products of a's and b's lanes."""
    ea = (lambda v, n: sx(v, n)) if asg else (lambda v, n: v & ((1 << n) - 1))
    eb = (lambda v: sx(v, 8)) if bsg else (lambda v: v & 0xFF)
    if two is None:
        acc = sum(ea(a >> (8 * i), 8) * eb(b >> (8 * i)) for i in range(4))
    else:
        acc = sum(ea(a >> (16 * i), 16) * eb(b >> (8 * (2 * two + i))) for i in range(2))
    return (acc + c) & U32


# ---- one record ----------------------------------------------------------------------------------------------------
def operands(leg, op, seed, w, l) -> List[int]:
    t, f, row = 32 * w + l, op // ROWS[leg], op % ROWS[leg]
    s = [word(seed, leg, op, k, t) for k in range(4)]
    x = [0, 0, 0, 0]
    if leg == LOGIC:
        x[:3] = [mix32(s[0]), mix32(s[1]), mix32(s[2])]
        if f in (256, 257):
            x[0] = t % 40 if row == 0 else count(s[0])
            x[1] = (t // 40 * 7 + t) % 40 if row == 0 else count(s[1])
        elif f >= 265:
            x[1] = t % 40 if row == 0 else count(s[1])
        elif f == 260:
            x[0] = mix64(s[0])
    elif leg == SHIFT:
        n = t % 72 if row == 0 else count(s[2])
        x[0] = mix64(s[0]) if 8 <= f <= 11 else mix32(s[0])
        x[1] = mix32(s[1])
        x[2] = s[2] & 3 if f >= 13 else s[2] & U32 if f == 12 else n
        if 4 <= f <= 11:
            x[1], x[2] = n, 0
    elif leg == IADD:
        if f <= 3:
            x = [mix64(s[k]) for k in range(4)]
            if f in (0, 2):
                x[2] = x[3] = 0
        else:
            x[0] = mix32(s[0])
            x[1] = x[0] if (s[3] >> 8) & 3 == 0 else mix32(s[1])
            x[2] = mix32(s[2]) if not 14 <= f < 26 else 0
            x[3] = mix32(s[3]) if f < 14 else 0
    elif leg == IMUL:
        x = [mix32(s[k]) for k in range(4)]
        if f == 12:
            x = [mix64(s[0]), mix64(s[1]), 0, 0]
        else:
            if f < 6:
                x[2] = 0
            if f < 9 or f >= 13:
                x[3] = 0
    else:
        sc = (t + 3 * row) % 8
        if f < 25:
            dbl = f >= 16
            fm = F64 if dbl else F32
            kind = (f - 16) // 3 if dbl else f // 4
            fma = kind == 2 if dbl else kind == 3
            x[:3] = f_arith(fm, sc, fma, s)
            if not fma:
                x[2] = 0
        else:
            x[0] = f_cmp(s[0])
            x[1] = x[0] if (s[3] >> 8) & 7 == 0 else f_cmp(s[1])
            if f < 31:
                i = f - 25
                if i < 2 and is_nan(F32, x[0]) and is_nan(F32, x[1]):
                    x[1] = f_any(F32, s[1])
                if i >= 4:
                    for k in range(2):
                        if is_nan(F32, x[k]):
                            x[k] = f_any(F32, s[k])
                if is_zero(F32, x[0]) and is_zero(F32, x[1]):
                    x[1] = x[0]
    return x


def result(leg, f, x) -> Tuple[int, int, int]:
    """The exact result words of form f of leg on operand words x (PTX ISA)."""
    a, b, c, d = (v & U32 for v in x)
    if leg == LOGIC:
        if f < 256:
            return lop3(f, a, b, c), 0, 0
        if f in (256, 257):
            return bmsk(a, b, f == 256), 0, 0
        if f == 258:
            return int(format(a, "032b")[::-1], 2), 0, 0
        if f == 259:
            return bin(a).count("1"), 0, 0
        if f == 260:
            return bin(x[0]).count("1"), 0, 0
        if f <= 264:
            return bfind(a, f in (262, 264), f >= 263), 0, 0
        return szext(a, b, f <= 266, f in (266, 268)), 0, 0
    if leg == SHIFT:
        if f < 4:
            n = (min(c, 32) if f % 2 else c & 31)
            v = (b << 32) | a
            return (((v << n) >> 32) if f < 2 else (v >> n)) & U32, 0, 0
        if f < 8:
            if f == 4:
                return (a << b) & U32 if b < 32 else 0, 0, 0
            if f == 7:
                return (s32(a) >> min(b, 31)) & U32, 0, 0
            return a >> b if b < 32 else 0, 0, 0
        if f < 12:
            y = x[0]
            if f == 8:
                return (y << b) & U64 if b < 64 else 0, 0, 0
            if f == 11:
                return (sx(y, 64) >> min(b, 63)) & U64, 0, 0
            return y >> b if b < 64 else 0, 0, 0
        return prmt(a, b, c, None if f == 12 else f - 13), 0, 0
    if leg == IADD:
        if f in (0, 2):
            z = x[0] + x[1] if f == 0 else x[0] - x[1]
            return z & U64, (1 if z >> 64 else 0) if f == 0 else (U32 if z < 0 else 0), 0
        if f in (1, 3):
            p, q = x[1] << 64 | x[0], x[3] << 64 | x[2]
            z = p + q if f == 1 else p - q
            carry = (1 if z >> 128 else 0) if f == 1 else (U32 if z < 0 else 0)
            z &= (1 << 128) - 1
            return z & U64, z >> 64, carry
        if f < 14:
            i = f - 4
            xs, ys = (s32(a), s32(b)) if i < 6 else (a, b)
            p = [xs == ys, xs != ys, xs < ys, xs <= ys, xs > ys, xs >= ys][[0, 1, 2, 3, 4, 5, 2, 3, 4, 5][i]]
            return (c if p else d), 0, 0
        if f < 26:
            return minmax(f - 14, a, b), 0, 0
        if f < 48:
            return dpx(f - 26, a, b, c), 0, 0
        if f == 48:
            return (c + abs(a - b)) & U32, 0, 0
        return (c + abs(s32(a) - s32(b))) & U32, 0, 0
    if leg == IMUL:
        pu, ps = a * b, s32(a) * s32(b)
        if f in (0, 1):
            return pu & U32, 0, 0
        if f == 2:
            return (ps >> 32) & U32, 0, 0
        if f == 3:
            return pu >> 32, 0, 0
        if f == 4:
            return ps & U64, 0, 0
        if f == 5:
            return pu, 0, 0
        if f == 6:
            return (pu + c) & U32, 0, 0
        if f == 7:
            return ((pu >> 32) + c) & U32, 0, 0
        if f == 8:
            return ((ps >> 32) + c) & U32, 0, 0
        if f == 9:
            z = pu + (d << 32 | c)
            return z & U64, z >> 64, 0
        if f == 10:
            return (ps + (d << 32 | c)) & U64, 0, 0
        if f == 11:
            r0 = (pu >> 32) + c
            r1 = ((pu & U32) + d + (r0 >> 32)) & U32
            return r1 << 32 | (r0 & U32), 0, 0
        if f == 12:
            return (x[0] * x[1]) & U64, 0, 0
        i = (f - 13) % 4
        two = None if f < 17 else 0 if f < 21 else 1
        return dp(a, b, c, i >= 2, i % 2 == 1, two), 0, 0
    if f < 16:
        kind, mode = f // 4, f % 4
        if kind == 3:
            return f_fma(F32, a, b, c, mode), 0, 0
        if kind == 2:
            return f_mul(F32, a, b, mode), 0, 0
        return f_add(F32, a, b ^ (F32.sign if kind == 1 else 0), mode), 0, 0
    if f < 25:
        kind, mode = (f - 16) // 3, 1 + (f - 16) % 3
        if kind == 2:
            return f_fma(F64, x[0], x[1], x[2], mode), 0, 0
        if kind == 1:
            return f_mul(F64, x[0], x[1], mode), 0, 0
        return f_add(F64, x[0], x[1], mode), 0, 0
    if f < 31:
        return fminmax(f - 25, a, b), 0, 0
    return int(fsetp(f - 31, a, b)), 0, 0


def record(leg, op, seed, w, l) -> Tuple[List[int], Tuple[int, int, int]]:
    x = operands(leg, op, seed, w, l)
    return x, result(leg, op // ROWS[leg], x)


def expected(leg, seed, w) -> List[Tuple[List[int], Tuple[int, int, int]]]:
    """The table of leg for warp w: (operands, result) indexed op * 32 + lane."""
    return [record(leg, op, seed, w, l) for op in range(OPS[leg]) for l in range(32)]


def fold_value(out) -> int:
    return (out[0] + 2 * out[1] + 4 * out[2]) & U64


def fold(leg, seed) -> Tuple[int, int, int]:
    x = s = wt = 0
    for w in range(WARPS):
        for i, (_x, out) in enumerate(expected(leg, seed, w)):
            v = fold_value(out)
            x ^= v
            s += v
            wt += v * (2 * (i // 32) + 1)
    return x, s & U64, wt & U64


def injected(leg, seed, op, w, l, operand, mask):
    """The record an injection of mask into operand word `operand` of (op, w, l) makes: (operands, expected, actual),
    or None when the form ignores the changed bits."""
    x, out = record(leg, op, seed, w, l)
    y = list(x)
    y[operand] ^= mask
    got = result(leg, op // ROWS[leg], y)
    return None if tuple(got) == tuple(out) else (x, tuple(out), tuple(got))


# ---- classification and annotations: the cross-lane probe's, with the ALU's op counts --------------------------------
def classify(call: Dict, expect: Dict[int, Tuple[int, int, int]]):
    saved = xlane.OPS
    xlane.OPS = OPS
    try:
        return xlane.classify(call, expect)
    finally:
        xlane.OPS = saved


def annotations(r: Dict) -> Dict[str, str]:
    m = xlane.annotations(dict(r, failed_legs=0))
    out = {k.replace("probe-xlane-", "probe-alu-"): v for k, v in m.items()}
    legs = [NAMES[b] for b in range(LEGS) if r["failed_legs"] >> b & 1]
    if legs:
        out["cohdi.io/probe-alu-legs"] = ",".join(legs)
    return out


def annotations_json(r: Dict) -> bytes:
    return go_marshal_string_map(annotations(r)).encode("utf-8")
