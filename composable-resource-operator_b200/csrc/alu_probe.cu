// alu_probe.cu — the ALU probe (cro_probe_alu, cro_probe_alu_uuid): every SM's integer, bit-manipulation, DPX and
// directed-rounding floating-point instructions checked form by form on every lane, one launch per leg.  The host
// builds the call's table here, in integer arithmetic: no operand and no expected value comes from the unit under
// test, and no host FPU rounding mode is involved.
#include "alu_kernels.cuh"
#include "lane_report.hpp"

namespace cro {

namespace alu {
namespace {

typedef uint64_t u64;
typedef unsigned __int128 u128;
constexpr u64 U32 = 0xFFFFFFFFull;

// ---- operands ----
// The seeded word k (0 .. 3) of (leg, op, warp, lane).
u64 word(u64 seed, unsigned leg, unsigned op, unsigned k, unsigned t) {
    return pattern_word(seed, ((((u64)leg * 1024 + op) * 8 + k) << 8) | t);
}
// A 32-bit operand: half seeded, the rest 0 / all ones / INT_MIN / INT_MAX, a walking one or zero, or a small
// signed value.
u64 mix32(u64 x) {
    static const u64 E[4] = {0, U32, 0x80000000ull, 0x7FFFFFFFull};
    switch (x >> 61) {
        case 4: return E[(x >> 32) & 3];
        case 5: return 1ull << (x & 31);
        case 6: return ~(1ull << (x & 31)) & U32;
        case 7: return ((x & 15) - 8) & U32;
        default: return x & U32;
    }
}
u64 mix64(u64 x) {
    static const u64 E[4] = {0, ~0ull, 1ull << 63, (1ull << 63) - 1};
    switch (x >> 61) {
        case 4: return E[(x >> 32) & 3];
        case 5: return 1ull << (x & 63);
        case 6: return ~(1ull << (x & 63));
        case 7: return (x & 15) - 8;
        default: return x;
    }
}
// A shift count or bit position: three in four below 64, else any 32-bit value.
u64 count(u64 x) { return (x >> 62) ? x & 63 : x & U32; }

// ---- exact floating point: sign, M (< 2^127), E: the value (-1)^sign * M * 2^E ----
struct Fmt {
    int p, ebits;
    int bias() const { return (1 << (ebits - 1)) - 1; }
    int emin() const { return 1 - bias() - (p - 1); }                   // exponent of the lsb of a subnormal
    int emax() const { return (1 << ebits) - 2 - bias() - (p - 1); }    // ... of the largest finite value
};
constexpr Fmt kF32{24, 8}, kF64{53, 11};
enum { RN, RZ, RM, RP };
struct Exact {
    bool s;
    u128 m;
    int e;
};

int msb(u128 m) {
    const u64 hi = (u64)(m >> 64), lo = (u64)m;
    return hi ? 127 - __builtin_clzll(hi) : lo ? 63 - __builtin_clzll(lo) : -1;
}
u64 pack(const Fmt& f, bool s, u64 biased, u64 frac) { return ((u64)s << (f.p - 1 + f.ebits)) | (biased << (f.p - 1)) | frac; }
u64 zero(const Fmt& f, bool s) { return pack(f, s, 0, 0); }
Exact unpack(const Fmt& f, u64 b) {
    const bool s = b >> (f.p - 1 + f.ebits) & 1;
    const u64 ef = b >> (f.p - 1) & ((1ull << f.ebits) - 1), frac = b & ((1ull << (f.p - 1)) - 1);
    if (ef == 0) return Exact{s, frac, f.emin()};
    return Exact{s, frac | (1ull << (f.p - 1)), (int)ef - f.bias() - (f.p - 1)};
}
// Round a nonzero exact value to the format in the mode.
u64 round(const Fmt& f, const Exact& x, int mode) {
    int e = x.e + msb(x.m) + 1 - f.p;
    if (e < f.emin()) e = f.emin();
    const int sh = e - x.e;
    u128 m;
    bool up = false;
    if (sh <= 0) {
        m = x.m << -sh;
    } else {
        const u128 rem = sh >= 128 ? x.m : x.m & (((u128)1 << sh) - 1);
        const u128 half = sh > 128 ? 0 : (u128)1 << (sh - 1);   // past 128 bits, every M < 2^127 is below half
        m = sh >= 128 ? 0 : x.m >> sh;
        const bool over = sh <= 128 && rem > half, tie = sh <= 128 && rem == half;
        if (rem) switch (mode) {
                case RN: up = over || (tie && (m & 1)); break;
                case RM: up = x.s; break;
                case RP: up = !x.s; break;
                default: break;
            }
    }
    if (up && ++m == (u128)1 << f.p) {
        m >>= 1;
        ++e;
    }
    if (e > f.emax()) {
        const bool inf = mode == RN || (mode == RM && x.s) || (mode == RP && !x.s);
        return inf ? pack(f, x.s, (1ull << f.ebits) - 1, 0) : pack(f, x.s, (1ull << f.ebits) - 2, (1ull << (f.p - 1)) - 1);
    }
    if (m < (u128)1 << (f.p - 1)) return pack(f, x.s, 0, (u64)m);
    return pack(f, x.s, (u64)(e - f.emin() + 1), (u64)m & ((1ull << (f.p - 1)) - 1));
}
// x + y exactly enough to round: both aligned high, the smaller shifted right with a sticky bit.  Exact zeros take
// the sign of equal-signed operands, else +0 (-0 rounding down).
u64 add_exact(const Fmt& f, Exact x, Exact y, int mode) {
    if (!x.m && !y.m) return zero(f, x.s == y.s ? x.s : mode == RM);
    if (!x.m) return round(f, y, mode);
    if (!y.m) return round(f, x, mode);
    for (Exact* v : {&x, &y}) {
        const int sh = 125 - msb(v->m);
        v->m <<= sh;
        v->e -= sh;
    }
    if (x.e < y.e) std::swap(x, y);
    const int d = x.e - y.e;
    const u128 small = d >= 126 ? 1 : (y.m >> d) | ((y.m & (((u128)1 << d) - 1)) ? 1 : 0);
    Exact r{x.s, 0, x.e};
    if (x.s == y.s) r.m = x.m + small;
    else if (x.m >= small) r.m = x.m - small;
    else {
        r.m = small - x.m;
        r.s = y.s;
    }
    if (!r.m) return zero(f, mode == RM);
    return round(f, r, mode);
}
Exact product(const Fmt& f, u64 a, u64 b) {
    const Exact x = unpack(f, a), y = unpack(f, b);
    return Exact{x.s != y.s, x.m * y.m, x.e + y.e};
}
u64 fadd(const Fmt& f, u64 a, u64 b, int mode) { return add_exact(f, unpack(f, a), unpack(f, b), mode); }
u64 fmul(const Fmt& f, u64 a, u64 b, int mode) {
    const Exact p = product(f, a, b);
    return p.m ? round(f, p, mode) : zero(f, p.s);
}
u64 ffma(const Fmt& f, u64 a, u64 b, u64 c, int mode) { return add_exact(f, product(f, a, b), unpack(f, c), mode); }

// ---- float operands ----
u64 fbits(const Fmt& f, u64 sign, u64 biased, u64 frac) { return pack(f, sign & 1, biased, frac & ((1ull << (f.p - 1)) - 1)); }
u64 fexp(const Fmt& f, u64 b) { return b >> (f.p - 1) & ((1ull << f.ebits) - 1); }
// Normal, exponent uniform over the whole range.
u64 f_any(const Fmt& f, u64 x) { return fbits(f, x >> 63, 1 + (x >> 32) % ((1ull << f.ebits) - 2), x); }
// Normal, exponent within `spread` of 2^off (biased bias + off).
u64 f_near(const Fmt& f, u64 x, int off, int spread) {
    return fbits(f, x >> 63, (u64)(f.bias() + off - spread + (int)((x >> 40) % (u64)(2 * spread + 1))), x);
}
u64 f_tiny(const Fmt& f, u64 x) { return fbits(f, x >> 63, (x >> 40) % 3, x); }                           // subnormal or near
u64 f_huge(const Fmt& f, u64 x) { return fbits(f, x >> 63, (1ull << f.ebits) - 2 - (x >> 40) % 3, x); }   // near the top
u64 f_special(const Fmt& f, u64 x, bool inf) {
    const u64 top = (1ull << f.ebits) - 1, ones = (1ull << (f.p - 1)) - 1;
    const u64 v[10] = {0, 0, top - 1, top - 1, 1, 0, 1, 0, (u64)f.bias(), inf ? top : (u64)f.bias()};
    const u64 fr[10] = {0, 0, ones, ones, 0, 1, ones, ones, 0, 0};
    const unsigned i = (unsigned)((x >> 32) % 10);
    return fbits(f, x >> 63, v[i], fr[i]);
}
// Short mantissa: only the top 11 (f32) or 26 (f64) fraction bits, so a product sits on or near a halfway point.
u64 f_short(const Fmt& f, u64 x) {
    const int keep = f.p == 24 ? 11 : 26;
    return f_near(f, x & ~(((1ull << (f.p - 1 - keep)) - 1)), 0, 8);
}
u64 f_nan(const Fmt& f, u64 x) { return fbits(f, x >> 63, (1ull << f.ebits) - 1, (1ull << (f.p - 2)) | x); }
bool is_nan(const Fmt& f, u64 b) { return fexp(f, b) == (1ull << f.ebits) - 1 && (b & ((1ull << (f.p - 1)) - 1)); }
bool is_zero(const Fmt& f, u64 b) { return (b & ~(1ull << (f.p - 1 + f.ebits))) == 0; }

// Arithmetic operands (a, b, c) of scenario sc: 0 any exponent, 1 close exponents, 2 b (and c) at, just below or
// just above half an ulp of a, 3 cancellation (b and c near -a or -a*b), 4 subnormal, 5 overflow, 6 special values, 7
// short mantissas.  No NaN or infinity: arithmetic on them leaves NaN payloads open.
void f_arith(const Fmt& f, unsigned sc, bool fma, const u64 s[4], u64 o[3]) {
    const u64 sign = 1ull << (f.p - 1 + f.ebits), ones = (1ull << (f.p - 1)) - 1;
    switch (sc) {
        case 0: for (int k = 0; k < 3; ++k) o[k] = f_any(f, s[k]); break;
        case 1: for (int k = 0; k < 3; ++k) o[k] = f_near(f, s[k], 0, 3); break;
        case 2: {
            o[0] = f_near(f, s[0], 0, 20);
            const u64 fr[3] = {0, 1, ones};
            for (int k = 1; k < 3; ++k)
                o[k] = fbits(f, s[k] >> 63, fexp(f, o[0]) - (u64)(f.p - 1) - (s[k] >> 40) % 3, fr[(s[k] >> 50) % 3]);
            break;
        }
        case 3: {
            o[0] = f_near(f, s[0], 0, 30);
            o[1] = f_near(f, s[1], 0, 30);
            const u64 base = fma ? fmul(f, o[0], o[1], RN) : o[0];
            const u64 fr = base & ones, dl = (s[2] >> 40) % 3;
            u64 v = base;
            if (dl == 1 && fr != ones) v = base + 1;
            if (dl == 2 && fr != 0) v = base - 1;
            v ^= ((s[2] >> 50) & 1) || fma ? sign : 0;
            (fma ? o[2] : o[1]) = v;
            if (!fma) o[2] = f_near(f, s[2], 0, 3);
            break;
        }
        case 4:
            o[0] = f_tiny(f, s[0]);
            o[1] = (s[1] >> 62) & 1 ? f_tiny(f, s[1]) : f_near(f, s[1], 0, 12);
            o[2] = f_tiny(f, s[2]);
            break;
        case 5:
            o[0] = f_huge(f, s[0]);
            o[1] = (s[1] >> 62) & 1 ? f_huge(f, s[1]) : f_near(f, s[1], 0, 1);
            o[2] = f_huge(f, s[2]);
            break;
        case 6: for (int k = 0; k < 3; ++k) o[k] = f_special(f, s[k], false); break;
        default: for (int k = 0; k < 3; ++k) o[k] = f_short(f, s[k]); break;
    }
}

// min / max / setp operands: any, subnormal, special (with infinities), quiet NaN, or equal to the other operand.
u64 f_cmp(u64 x) {
    switch ((x >> 58) % 8) {
        case 0: case 1: return f_any(kF32, x);
        case 2: return f_near(kF32, x, 0, 2);
        case 3: return f_tiny(kF32, x);
        case 4: case 5: return f_special(kF32, x, true);
        default: return f_nan(kF32, x);
    }
}

// ---- expected results ----
unsigned u(u64 x) { return (unsigned)x; }
int s32(u64 x) { return (int)(unsigned)x; }

// The LUT's bit (4a + 2b + c) for each bit position: the OR of the minterms whose LUT bit is set.
u64 lop3(unsigned lut, unsigned a, unsigned b, unsigned c) {
    unsigned d = 0;
    for (unsigned idx = 0; idx < 8; ++idx)
        if (lut >> idx & 1) d |= (idx & 4 ? a : ~a) & (idx & 2 ? b : ~b) & (idx & 1 ? c : ~c);
    return d;
}
u64 bmsk(unsigned a, unsigned b, bool clamp) {
    const unsigned a1 = a & 31, b1 = b & 31, sum = a1 + b1;
    u64 mask0 = (U32 << a1) & U32, mask1 = sum >= 32 ? 0 : (U32 << sum) & U32;
    bool pos_over = false, width_over = false;
    if (clamp) {
        if (a >= 32) {
            pos_over = true;
            mask0 = 0;
        }
        if (b >= 32) width_over = true;
    }
    if (sum >= 32 || pos_over || width_over) mask1 = 0;
    else if (b1 == 0) mask1 = U32;
    return mask0 & ~mask1 & U32;
}
u64 bfind(unsigned a, bool sgn, bool shiftamt) {
    if (sgn && (a >> 31)) a = ~a;
    unsigned d = 0xFFFFFFFFu;
    for (int i = 31; i >= 0; --i)
        if (a >> i & 1) {
            d = (unsigned)i;
            break;
        }
    if (shiftamt && d != 0xFFFFFFFFu) d = 31 - d;
    return d;
}
u64 szext(unsigned a, unsigned b, bool clamp, bool sgn) {
    const unsigned b1 = b & 31;
    const bool too_large = b >= 32 && clamp;
    const unsigned mask = too_large ? 0u : 0xFFFFFFFFu << b1;
    const bool sign = !(b1 == 0 || too_large || !sgn) && ((a >> ((b1 - 1) & 31)) & 1);
    return (a & ~mask) | (sign ? mask : 0u);
}
u64 prmt(unsigned a, unsigned b, unsigned c, int mode) {
    const u64 x = ((u64)b << 32) | a;
    auto byte = [&](unsigned i) { return (unsigned)(x >> (8 * (i & 7)) & 0xFF); };
    static const unsigned char kMode[6][4][4] = {
        {{0, 1, 2, 3}, {1, 2, 3, 4}, {2, 3, 4, 5}, {3, 4, 5, 6}},   // f4e: d.b0 .. d.b3
        {{0, 7, 6, 5}, {1, 0, 7, 6}, {2, 1, 0, 7}, {3, 2, 1, 0}},   // b4e
        {{0, 0, 0, 0}, {1, 1, 1, 1}, {2, 2, 2, 2}, {3, 3, 3, 3}},   // rc8
        {{0, 1, 2, 3}, {1, 1, 2, 3}, {2, 2, 2, 3}, {3, 3, 3, 3}},   // ecl
        {{0, 0, 0, 0}, {0, 1, 1, 1}, {0, 1, 2, 2}, {0, 1, 2, 3}},   // ecr
        {{0, 1, 0, 1}, {2, 3, 2, 3}, {0, 1, 0, 1}, {2, 3, 2, 3}}};  // rc16
    unsigned d = 0;
    for (unsigned i = 0; i < 4; ++i) {
        unsigned v;
        if (mode < 0) {
            const unsigned sel = c >> (4 * i) & 15;
            v = byte(sel & 7);
            if (sel & 8) v = (v & 0x80) ? 0xFF : 0;
        } else {
            v = byte(kMode[mode][c & 3][i]);
        }
        d |= v << (8 * i);
    }
    return d;
}
u64 shf(unsigned a, unsigned b, unsigned c, bool left, bool clamp) {
    const unsigned n = clamp ? (c < 32 ? c : 32) : c & 31;
    const u64 x = ((u64)b << 32) | a;
    return left ? ((x << n) >> 32) & U32 : (x >> n) & U32;
}
// 16x2 lanes: f applied to each half (as signed or unsigned 16-bit values), packed.
template <class G>
u64 halves(unsigned a, unsigned b, unsigned c, bool sgn, G g) {
    u64 d = 0;
    for (int h = 0; h < 2; ++h) {
        auto ext = [&](unsigned v) -> long long { const unsigned x = v >> (16 * h) & 0xFFFF; return sgn ? (long long)(short)x : (long long)x; };
        d |= ((u64)g(ext(a), ext(b), ext(c)) & 0xFFFF) << (16 * h);
    }
    return d;
}
long long mn(long long x, long long y) { return x < y ? x : y; }
long long mx(long long x, long long y) { return x > y ? x : y; }
long long relu(long long x) { return x < 0 ? 0 : x; }

u64 minmax(unsigned i, unsigned a, unsigned b) {
    switch (i) {
        case 0: return mn(a, b);
        case 1: return mx(a, b);
        case 2: return (u64)(unsigned)mn(s32(a), s32(b));
        case 3: return (u64)(unsigned)mx(s32(a), s32(b));
        case 4: return (u64)(unsigned)relu(mn(s32(a), s32(b)));
        case 5: return (u64)(unsigned)relu(mx(s32(a), s32(b)));
        case 6: return halves(a, b, 0, false, [](long long x, long long y, long long) { return mn(x, y); });
        case 7: return halves(a, b, 0, false, [](long long x, long long y, long long) { return mx(x, y); });
        case 8: return halves(a, b, 0, true, [](long long x, long long y, long long) { return mn(x, y); });
        case 9: return halves(a, b, 0, true, [](long long x, long long y, long long) { return mx(x, y); });
        case 10: return halves(a, b, 0, true, [](long long x, long long y, long long) { return relu(mn(x, y)); });
        default: return halves(a, b, 0, true, [](long long x, long long y, long long) { return relu(mx(x, y)); });
    }
}
// The DPX pairs: i < 12 three-operand min / max, else add then min / max.  Sums wrap in their width first.
u64 dpx(unsigned i, unsigned a, unsigned b, unsigned c) {
    const bool isMax = i % 2 == 0;
    auto pick = [&](long long x, long long y) { return isMax ? mx(x, y) : mn(x, y); };
    auto w32s = [](long long x) { return (long long)(int)(unsigned)(unsigned long long)x; };
    auto w32u = [](long long x) { return (long long)(unsigned)(unsigned long long)x; };
    auto w16s = [](long long x) { return (long long)(short)(unsigned short)(unsigned long long)x; };
    auto w16u = [](long long x) { return (long long)(unsigned short)(unsigned long long)x; };
    const unsigned kind = (i % 12) / 2;   // 0 s32, 1 u32, 2 relu.s32, 3 s16x2, 4 u16x2, 5 relu.s16x2
    if (i < 12) {
        switch (kind) {
            case 0: return (unsigned)pick(pick(s32(a), s32(b)), s32(c));
            case 1: return (unsigned)pick(pick(a, b), c);
            case 2: return (unsigned)relu(pick(pick(s32(a), s32(b)), s32(c)));
            case 3: return halves(a, b, c, true, [&](long long x, long long y, long long z) { return pick(pick(x, y), z); });
            case 4: return halves(a, b, c, false, [&](long long x, long long y, long long z) { return pick(pick(x, y), z); });
            default: return halves(a, b, c, true, [&](long long x, long long y, long long z) { return relu(pick(pick(x, y), z)); });
        }
    }
    switch (kind) {
        case 0: return (unsigned)pick(w32s((long long)s32(a) + s32(b)), s32(c));
        case 1: return (unsigned)pick(w32u((long long)a + b), c);
        case 2: return (unsigned)relu(pick(w32s((long long)s32(a) + s32(b)), s32(c)));
        case 3: return halves(a, b, c, true, [&](long long x, long long y, long long z) { return pick(w16s(x + y), z); });
        default: return halves(a, b, c, false, [&](long long x, long long y, long long z) { return pick(w16u(x + y), z); });
    }
}
u64 dp(unsigned a, unsigned b, unsigned c, bool as, bool bs, int two) {
    long long acc = 0;
    if (two < 0) {
        for (int i = 0; i < 4; ++i) {
            const unsigned x = a >> (8 * i) & 0xFF, y = b >> (8 * i) & 0xFF;
            acc += (as ? (long long)(signed char)x : (long long)x) * (bs ? (long long)(signed char)y : (long long)y);
        }
    } else {
        for (int i = 0; i < 2; ++i) {
            const unsigned x = a >> (16 * i) & 0xFFFF, y = b >> (8 * (2 * two + i)) & 0xFF;
            acc += (as ? (long long)(short)x : (long long)x) * (bs ? (long long)(signed char)y : (long long)y);
        }
    }
    return (u64)(unsigned)((unsigned long long)acc + c);
}
bool fsetp(unsigned i, u64 a, u64 b) {
    const bool un = is_nan(kF32, a) || is_nan(kF32, b);
    if (i == 12) return !un;
    if (i == 13) return un;
    if (un) return i >= 6;
    // ordered compare of two non-NaN values as signed magnitudes; zeros of either sign are equal
    int cmp = 0;
    if (!(is_zero(kF32, a) && is_zero(kF32, b))) {
        const long long ma = (long long)(a & 0x7FFFFFFF), mb = (long long)(b & 0x7FFFFFFF);
        const long long vx = a >> 31 ? -ma : ma, vy = b >> 31 ? -mb : mb;
        cmp = vx < vy ? -1 : vx > vy ? 1 : 0;
    }
    switch (i % 6) {
        case 0: return cmp == 0;
        case 1: return cmp != 0;
        case 2: return cmp < 0;
        case 3: return cmp <= 0;
        case 4: return cmp > 0;
        default: return cmp >= 0;
    }
}
u64 fminmax(unsigned i, u64 a, u64 b) {
    const bool isMax = i % 2 == 1;
    const bool an = is_nan(kF32, a), bn = is_nan(kF32, b);
    if (i >= 2 && i < 4 && (an || bn)) return 0x7FFFFFFF;
    if (an && bn) return 0x7FFFFFFF;
    if (an) return b;
    if (bn) return a;
    if (i >= 4) {
        const u64 ma = a & 0x7FFFFFFF, mb = b & 0x7FFFFFFF;
        const u64 m = isMax ? (ma > mb ? ma : mb) : (ma < mb ? ma : mb);
        return m | ((a ^ b) & 0x80000000);
    }
    const bool lt = fsetp(2, a, b);
    return isMax ? (lt ? b : a) : (lt ? a : b);
}

// ---- the table ----
void record(unsigned leg, unsigned op, u64 seed, unsigned w, unsigned l, cro_alu_record* r) {
    const unsigned t = 32 * w + l, f = op / kRows[leg], row = op % kRows[leg];
    u64 s[4];
    for (unsigned k = 0; k < 4; ++k) s[k] = word(seed, leg, op, k, t);
    u64* in = r->in;
    u64* out = r->out;
    *r = cro_alu_record{};
    switch (leg) {
        case CRO_ALU_LEG_LOGIC: {
            in[0] = mix32(s[0]);
            in[1] = mix32(s[1]);
            in[2] = mix32(s[2]);
            if (f == kBmskClamp || f == kBmskWrap) {
                in[0] = row == 0 ? t % 40 : count(s[0]);
                in[1] = row == 0 ? (t / 40 * 7 + t) % 40 : count(s[1]);
            } else if (f >= kSzextClampU) {
                in[1] = row == 0 ? t % 40 : count(s[1]);
            } else if (f == kPopc64) {
                in[0] = mix64(s[0]);
            }
            const unsigned a = u(in[0]), b = u(in[1]), c = u(in[2]);
            if (f < 256) out[0] = lop3(f, a, b, c);
            else if (f <= kBmskWrap) out[0] = bmsk(a, b, f == kBmskClamp);
            else if (f == kBrev) {
                unsigned d = 0;
                for (int i = 0; i < 32; ++i) d |= (a >> i & 1) << (31 - i);
                out[0] = d;
            } else if (f == kPopc32) out[0] = (u64)__builtin_popcount(a);
            else if (f == kPopc64) out[0] = (u64)__builtin_popcountll(in[0]);
            else if (f <= kBfindShS) out[0] = bfind(a, f == kBfindS || f == kBfindShS, f >= kBfindShU);
            else out[0] = szext(a, b, f <= kSzextClampS, f == kSzextClampS || f == kSzextWrapS);
            break;
        }
        case CRO_ALU_LEG_SHIFT: {
            const u64 n = row == 0 ? t % 72 : count(s[2]);
            in[0] = f >= kShl64 && f <= kShrS64 ? mix64(s[0]) : mix32(s[0]);
            in[1] = mix32(s[1]);
            in[2] = f >= kPrmtF4e ? s[2] & 3 : f == kPrmt ? s[2] & U32 : n;
            if (f >= kShl32 && f <= kShrS64) {
                in[1] = n;
                in[2] = 0;
            }
            const unsigned a = u(in[0]), b = u(in[1]), c = u(in[2]);
            const unsigned cl = b < 64 ? b : 64;
            switch (f) {
                case kShfLWrap: case kShfLClamp: out[0] = shf(a, b, c, true, f == kShfLClamp); break;
                case kShfRWrap: case kShfRClamp: out[0] = shf(a, b, c, false, f == kShfRClamp); break;
                case kShl32: out[0] = b >= 32 ? 0 : (u64)(a << b); break;
                case kShrB32: case kShrU32: out[0] = b >= 32 ? 0 : (u64)(a >> b); break;
                case kShrS32: out[0] = (u64)(unsigned)(s32(a) >> (b >= 32 ? 31 : b)); break;
                case kShl64: out[0] = cl >= 64 ? 0 : in[0] << cl; break;
                case kShrB64: case kShrU64: out[0] = cl >= 64 ? 0 : in[0] >> cl; break;
                case kShrS64: out[0] = (u64)((long long)in[0] >> (cl >= 64 ? 63 : cl)); break;
                default: out[0] = prmt(a, b, c, f == kPrmt ? -1 : (int)(f - kPrmtF4e)); break;
            }
            break;
        }
        case CRO_ALU_LEG_IADD: {
            if (f <= kSub128) {
                for (int k = 0; k < 4; ++k) in[k] = mix64(s[k]);
                if (f == kAdd64 || f == kSub64) {
                    in[2] = in[3] = 0;
                    const u64 x = in[0], y = in[1];
                    out[0] = f == kAdd64 ? x + y : x - y;
                    out[1] = f == kAdd64 ? (x + y < x) : (x < y ? U32 : 0);
                } else {
                    const u128 x = ((u128)in[1] << 64) | in[0], y = ((u128)in[3] << 64) | in[2];
                    const u128 z = f == kAdd128 ? x + y : x - y;
                    out[0] = (u64)z;
                    out[1] = (u64)(z >> 64);
                    out[2] = f == kAdd128 ? (z < x) : (x < y ? U32 : 0);
                }
                break;
            }
            in[0] = mix32(s[0]);
            in[1] = ((s[3] >> 8) & 3) == 0 ? in[0] : mix32(s[1]);
            in[2] = mix32(s[2]);
            in[3] = f < kMinMax0 ? mix32(s[3]) : 0;
            const unsigned a = u(in[0]), b = u(in[1]), c = u(in[2]), d = u(in[3]);
            if (f < kMinMax0) {
                static const int kCmp[10] = {0, 1, 2, 3, 4, 5, 2, 3, 4, 5};
                const long long x = f - kSetp0 < 6 ? s32(a) : (long long)a, y = f - kSetp0 < 6 ? s32(b) : (long long)b;
                bool p;
                switch (kCmp[f - kSetp0]) {
                    case 0: p = x == y; break;
                    case 1: p = x != y; break;
                    case 2: p = x < y; break;
                    case 3: p = x <= y; break;
                    case 4: p = x > y; break;
                    default: p = x >= y; break;
                }
                out[0] = p ? c : d;
            } else if (f < kDpx0) {
                in[2] = 0;
                out[0] = minmax(f - kMinMax0, a, b);
            } else if (f < kSadU) {
                out[0] = dpx(f - kDpx0, a, b, c);
            } else {
                const bool sg = f == kSadS;
                const bool lt = sg ? s32(a) < s32(b) : a < b;
                out[0] = (u64)(unsigned)(c + (lt ? b - a : a - b));
            }
            break;
        }
        case CRO_ALU_LEG_IMUL: {
            for (int k = 0; k < 4; ++k) in[k] = mix32(s[k]);
            if (f == kMulLo64) {
                in[0] = mix64(s[0]);
                in[1] = mix64(s[1]);
                in[2] = in[3] = 0;
                out[0] = in[0] * in[1];
                break;
            }
            const unsigned a = u(in[0]), b = u(in[1]), c = u(in[2]), d = u(in[3]);
            const u64 pu = (u64)a * b, ps = (u64)((long long)s32(a) * s32(b));
            if (f < kMadLo) in[2] = 0;                          // mul reads a, b; mad and dp a, b, c; the chains all four
            if (f < kMadccLoHi || f >= kDp4a0) in[3] = 0;
            switch (f) {
                case kMulLoS: case kMulLoU: out[0] = pu & U32; break;
                case kMulHiS: out[0] = ps >> 32; break;
                case kMulHiU: out[0] = pu >> 32; break;
                case kMulWideS: out[0] = ps; break;
                case kMulWideU: out[0] = pu; break;
                case kMadLo: out[0] = (pu + c) & U32; break;
                case kMadHiU: out[0] = ((pu >> 32) + c) & U32; break;
                case kMadHiS: out[0] = ((ps >> 32) + c) & U32; break;
                case kMadccLoHi: {
                    const u128 z = (u128)pu + (((u128)d << 32) | c);
                    out[0] = (u64)z;
                    out[1] = (u64)(z >> 64);
                    break;
                }
                case kMadccLoHiS: out[0] = ps + (((u64)d << 32) | c); break;
                case kMadccHiLo: {
                    const u64 lo32 = (pu >> 32) + c;
                    out[0] = (((pu & U32) + d + (lo32 >> 32)) << 32 & ~U32) | (lo32 & U32);
                    break;
                }
                default: {
                    const unsigned i = (f - kDp4a0) % 4;
                    const int two = f < kDp2aLo0 ? -1 : f < kDp2aHi0 ? 0 : 1;
                    out[0] = dp(a, b, c, i >= 2, i % 2 == 1, two);
                    break;
                }
            }
            break;
        }
        default: {   // FLOAT
            const unsigned sc = (t + 3 * row) % 8;
            if (f < kFMin) {
                const bool dbl = f >= kF64_0;
                const Fmt& fm = dbl ? kF64 : kF32;
                const unsigned kind = dbl ? (f - kF64_0) / 3 : f / 4;   // f32: add sub mul fma; f64: add mul fma
                const int mode = dbl ? 1 + (int)((f - kF64_0) % 3) : (int)(f % 4);
                const bool isFma = dbl ? kind == 2 : kind == 3, isMul = dbl ? kind == 1 : kind == 2, isSub = !dbl && kind == 1;
                f_arith(fm, sc, isFma, s, in);
                if (!isFma) in[2] = 0;
                const u64 sign = 1ull << (fm.p - 1 + fm.ebits);
                if (isFma) out[0] = ffma(fm, in[0], in[1], in[2], mode);
                else if (isMul) out[0] = fmul(fm, in[0], in[1], mode);
                else out[0] = fadd(fm, in[0], isSub ? in[1] ^ sign : in[1], mode);
                break;
            }
            in[0] = f_cmp(s[0]);
            in[1] = ((s[3] >> 8) & 7) == 0 ? in[0] : f_cmp(s[1]);
            if (f < kFSetp0) {
                const unsigned i = f - kFMin;
                if (i < 2 && is_nan(kF32, in[0]) && is_nan(kF32, in[1])) in[1] = f_any(kF32, s[1]);
                if (i >= 4)
                    for (int k = 0; k < 2; ++k)
                        if (is_nan(kF32, in[k])) in[k] = f_any(kF32, s[k]);
                if (is_zero(kF32, in[0]) && is_zero(kF32, in[1])) in[1] = in[0];
                out[0] = fminmax(i, in[0], in[1]);
            } else {
                out[0] = fsetp(f - kFSetp0, in[0], in[1]) ? 1 : 0;
            }
            break;
        }
    }
}

}  // namespace

void table(unsigned leg, u64 seed, unsigned w, cro_alu_record* out) {
    for (unsigned op = 0; op < kOps[leg]; ++op)
        for (unsigned l = 0; l < 32; ++l) record(leg, op, seed, w, l, out + (size_t)op * 32 + l);
}

}  // namespace alu

namespace {
// The legs' tables, by leg then op, warp, lane (the kernels' op * CRO_ALU_THREADS + thread), and the closed form of
// every CTA's fold.
void build(uint64_t seed, uint32_t legs, std::vector<cro_alu_record> tabs[CRO_ALU_LEGS], cro_alu_result* r) {
    for (unsigned leg = 0; leg < CRO_ALU_LEGS; ++leg) {
        if (!(legs >> leg & 1u)) continue;
        const unsigned n = alu::kOps[leg];
        std::vector<cro_alu_record> w(n * 32);
        tabs[leg].resize((size_t)n * CRO_ALU_THREADS);
        uint64_t x = 0, s = 0, f = 0;
        for (unsigned warp = 0; warp < CRO_ALU_WARPS; ++warp) {
            alu::table(leg, seed, warp, w.data());
            for (uint64_t op = 0; op < n; ++op)
                for (unsigned l = 0; l < 32; ++l) {
                    const cro_alu_record& e = w[op * 32 + l];
                    tabs[leg][op * CRO_ALU_THREADS + warp * 32 + l] = e;
                    const uint64_t v = e.out[0] + 2 * e.out[1] + 4 * e.out[2];
                    x ^= v;
                    s += v;
                    f += v * (2 * op + 1);
                }
        }
        r->expect[leg][0] = x;
        r->expect[leg][1] = s;
        r->expect[leg][2] = f;
    }
}

// What the lane probes' host driver (lane_report.hpp) needs of the ALU probe: one table per leg, built on the host.
struct AluProbe {
    using Opts = cro_alu_opts;
    using Result = cro_alu_result;
    using Sm = cro_alu_sm;
    using Fault = cro_alu_fault;
    using Thread = cro_alu_thread;
    using Cta = cro_alu_cta;
    using Args = AluArgs;
    struct Tables {
        std::vector<cro_alu_record> tabs[CRO_ALU_LEGS];
    };
    static constexpr unsigned kLegs = CRO_ALU_LEGS, kAllLegs = CRO_ALU_ALL_LEGS, kThreads = CRO_ALU_THREADS,
                              kThreadRecs = CRO_ALU_THREAD_RECORDS, kRecords = CRO_ALU_RECORDS, kMaxSms = CRO_ALU_MAX_SMS,
                              kMaxIterations = CRO_ALU_MAX_ITERATIONS, kMaxRounds = CRO_ALU_MAX_ROUNDS,
                              kPersistent = CRO_ALU_PERSISTENT, kIntermittent = CRO_ALU_INTERMITTENT, kNone = CRO_ALU_NONE,
                              kSm = CRO_ALU_SM, kAll = CRO_ALU_ALL;
    static constexpr const char* kName = "ALU";
    static constexpr const char* kId = "alu";
    static constexpr const cro_wire& kWire = cro_wire_alu;
    static constexpr uint64_t Device::*kCalls = &Device::alu_calls;
    static constexpr SeedSpace kSeeds = kSeedAlu;
    // Iterations per CTA and leg, and launches per leg, when the caller gives none.  On an H100 80GB HBM3 at a 700 W
    // limit (profiles/h100_700w_alu_rate.jsonl) one iteration of the five legs takes about 0.4 ms of launches, one
    // launch per leg covering all 132 SMs, so 12 iterations (4.9 ms) cost about the SRAM, register-file and cross-lane
    // probes' 5 ms.  The host table build (about 40 ms there) is on top of that, in table_ns.
    static constexpr uint32_t kDefaultIterations = 12, kDefaultRounds = 4;
    static constexpr unsigned kBlobs = 1;

    static unsigned ops(unsigned leg) { return alu::kOps[leg]; }
    static std::string opts_error(const cro_alu_opts& o) { return alu_opts_error(o); }
    static cudaError_t plan(int device, unsigned leg) { return alu_plan(device, leg); }
    static int grids(cro_ctx*, const cro_alu_opts&, uint32_t, int sm_count, int (&grid)[kLegs]) {
        std::fill(grid, grid + kLegs, sm_count);
        return CRO_OK;
    }
    static cudaError_t launch(const cro_alu_opts&, unsigned leg, const AluArgs& a, int grid, cudaStream_t st) {
        return launch_alu(leg, a, grid, st);
    }
    static void open(const cro_alu_opts&, cro_alu_result* r, Tables& tb, bool timed) {
        const uint64_t t0 = now_ns();
        build(r->seed, r->legs, tb.tabs, r);
        if (timed) r->table_ns = now_ns() - t0;
    }
    static std::array<LaneBlob, kBlobs> blobs(const Tables& tb, unsigned leg) {
        return {LaneBlob{tb.tabs[leg].data(), tb.tabs[leg].size() * sizeof(cro_alu_record)}};
    }
    static void args(const cro_alu_opts& o, const cro_alu_result&, unsigned, const std::array<const void*, kBlobs>& on_dev,
                     AluArgs* a) {
        a->table = static_cast<const cro_alu_record*>(on_dev[0]);
        a->inj_operand = o.test_inject_operand;
    }
    static bool no_new_sm_ends(unsigned) { return false; }
    static int close(cro_alu_result* r, LaneTally<AluProbe>& t, std::vector<cro_alu_sm>* sms, std::vector<cro_alu_fault>* faults) {
        return close_lane_call<AluProbe>(r, t, sms, faults);
    }
    static void keep(cro_alu_result* r, const cro_alu_result& from) { r->table_ns = from.table_ns; }
};
}  // namespace

void alu_expected(unsigned leg, uint64_t seed, unsigned warp, cro_alu_record* out) { alu::table(leg, seed, warp, out); }

std::string alu_opts_error(const cro_alu_opts& o) {
    if (!lane_opts_ok<AluProbe>(o) || (o.test_inject_mask && o.test_inject_operand >= 4))
        return "ALU probe: iterations at most " + std::to_string(CRO_ALU_MAX_ITERATIONS) + ", legs at most 0x1F, max_rounds at most " +
               std::to_string(CRO_ALU_MAX_ROUNDS) + ", deadline_ms not negative, and an injection must name a leg the call runs, an SM "
               "id below " + std::to_string(CRO_ALU_MAX_SMS) + ", a warp below 8 and a lane below 32 (each or -1), an op of the "
               "leg, an iteration the call runs and an operand below 4";
    return "";
}

int ctx_probe_alu(cro_ctx* c, int idx, const cro_alu_opts& o, cro_alu_result* r, std::vector<cro_alu_sm>* sms,
                  std::vector<cro_alu_fault>* faults) {
    return probe_lane_legs<AluProbe>(c, idx, o, r, sms, faults);
}

int classify_alu(uint32_t legs, uint32_t iterations, uint64_t seed, uint32_t sm_count, uint64_t k, uint32_t rounds,
                 const cro_alu_cta* ctas, const cro_alu_thread* threads, const cro_alu_fault* records, cro_alu_result* r,
                 std::vector<cro_alu_sm>* sms, std::vector<cro_alu_fault>* faults) {
    cro_alu_opts o{};
    o.legs = legs;
    o.iterations = iterations;
    return classify_lane_legs<AluProbe>(o, seed, sm_count, k, rounds, ctas, threads, records, r, sms, faults);
}

int ctx_probe_alu_uuid(cro_ctx* c, const char* uuid, const cro_alu_opts& o, cro_alu_result* r, std::vector<cro_alu_sm>* sms,
                       std::vector<cro_alu_fault>* faults, int cap) {
    return probe_lane_legs_uuid<AluProbe>(c, uuid, o, r, sms, faults, cap);
}

}  // namespace cro
