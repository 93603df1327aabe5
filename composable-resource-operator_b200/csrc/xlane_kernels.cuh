// xlane_kernels.cuh — the cross-lane probe's ops (cro_probe_xlane): each leg's operands and expected results as plain
// integer arithmetic on the iteration's seed, shared by the kernels (xlane_kernels.cu), which recompute their peers'
// operands from them, and the host (cro_xlane_expected, xlane_probe.cu).  oracle/xlane.py restates them from the PTX
// ISA's definitions.
#pragma once
#include "kernels.cuh"

namespace cro {

struct XlaneArgs {
    cro_xlane_cta* cta;                 // grid entries
    cro_xlane_thread* thr;              // grid * CRO_XLANE_THREADS entries, by block then thread
    cro_xlane_fault* rec;               // CRO_XLANE_THREAD_RECORDS per thread entry
    unsigned long long seed, stamp;     // seed: iteration 0's; iteration i adds i * kNonceStride
    unsigned iterations;
    int inj_sm, inj_warp, inj_lane;     // -1: every SM / warp / lane
    unsigned inj_op, inj_iter;
    unsigned long long inj_mask;        // 0: nothing is injected in this launch (or not in this leg)
};
// Sets the leg's dynamic shared memory request; cudaErrorInvalidConfiguration when the device cannot hold it.
cudaError_t xlane_plan(int device, unsigned leg);
cudaError_t launch_xlane(unsigned leg, const XlaneArgs& a, int grid, cudaStream_t);

namespace xlane {

#define XL_HD __host__ __device__ __forceinline__
typedef unsigned long long u64;

constexpr unsigned kOps[CRO_XLANE_LEGS] = {CRO_XLANE_SHFL_OPS, CRO_XLANE_VOTE_OPS, CRO_XLANE_MATCH_OPS, CRO_XLANE_REDUX_OPS,
                                           CRO_XLANE_ATOMS_OPS};
constexpr unsigned kVoteForms = 4, kMatchForms = 4, kReduxForms = 9, kAtomsShapes = 4;
constexpr unsigned kNoPeer = 0xFFFFFFFFu;

// The operand key: leg, op (or row), warp (0 .. 15: 8 .. 15 name per-row or per-group values) and lane (0 .. 63).
XL_HD u64 word(u64 seed, unsigned leg, unsigned op, unsigned w, unsigned l) {
    return pattern_word(seed, ((u64)leg << 22) | ((u64)op << 10) | ((u64)w << 6) | l);
}

// ---- SHFL: ops 0..31 idx (source lane + op), 32..88 up, 89..145 down, 146..176 bfly (lane mask 1..31) ----------
enum { kShflIdx, kShflUp, kShflDown, kShflBfly };
struct Shfl {
    unsigned mode, b, c;                // b: the lane operand (idx: this lane's source lane), c: clamp and segment mask
};
// up / down op u (0 .. 56): widths 32, 16, 8, 4, 2 in turn, every delta 1 .. width - 1.
XL_HD void shfl_width_delta(unsigned u, unsigned* width, unsigned* delta) {
    unsigned w = 32;
    while (u >= w - 1) {
        u -= w - 1;
        w >>= 1;
    }
    *width = w;
    *delta = u + 1;
}
XL_HD Shfl shfl_op(unsigned op, unsigned lane) {
    if (op < 32) return Shfl{kShflIdx, (lane + op) & 31u, 0x1Fu};
    if (op < 146) {
        unsigned width, delta;
        shfl_width_delta((op - 32) % 57, &width, &delta);
        const bool up = op < 89;
        return Shfl{up ? (unsigned)kShflUp : (unsigned)kShflDown, delta, ((32u - width) << 8) | (up ? 0u : 0x1Fu)};
    }
    return Shfl{kShflBfly, op - 145, 0x1Fu};
}
// The source lane j and the in-range predicate of lane `lane` (PTX ISA, shfl.sync): j = lane when out of range.
XL_HD unsigned shfl_source(const Shfl& s, unsigned lane, bool* pval) {
    const unsigned seg = (s.c >> 8) & 31u, cval = s.c & 31u;
    const int maxl = (int)((lane & seg) | (cval & ~seg)), minl = (int)(lane & seg);
    int j;
    bool p;
    switch (s.mode) {
        case kShflUp: j = (int)lane - (int)s.b; p = j >= maxl; break;
        case kShflDown: j = (int)lane + (int)s.b; p = j <= maxl; break;
        case kShflBfly: j = (int)(lane ^ s.b); p = j <= maxl; break;
        default: j = minl | (int)(s.b & ~seg); p = j <= maxl; break;
    }
    *pval = p;
    return p ? (unsigned)j : lane;
}
XL_HD unsigned shfl_operand(u64 seed, unsigned op, unsigned w, unsigned l) { return (unsigned)word(seed, CRO_XLANE_LEG_SHFL, op, w, l); }

// ---- VOTE: row r = op / 4, form op % 4 (ballot, any, all, uni); lane l's predicate is bit 0 of its operand -------
// rows 0: all clear, 1: all set, 2..33: only lane r - 2 set, 34..65: only lane r - 34 clear, 66..95: seeded.
XL_HD unsigned vote_operand(u64 seed, unsigned row, unsigned w, unsigned l) {
    const unsigned x = (unsigned)word(seed, CRO_XLANE_LEG_VOTE, row, w, l);
    if (row >= 66) return x;
    const unsigned bit = row == 0 ? 0u : row == 1 ? 1u : row < 34 ? (l == row - 2 ? 1u : 0u) : (l == row - 34 ? 0u : 1u);
    return (x & ~1u) | bit;
}
XL_HD unsigned vote_ballot(u64 seed, unsigned row, unsigned w) {
    unsigned b = 0;
    for (unsigned l = 0; l < 32; ++l) b |= (vote_operand(seed, row, w, l) & 1u) << l;
    return b;
}
XL_HD u64 vote_result(unsigned form, unsigned ballot) {
    switch (form) {
        case 0: return ballot;
        case 1: return ballot != 0u;
        case 2: return ballot == ~0u;
        default: return ballot == 0u || ballot == ~0u;
    }
}

// ---- MATCH: row r = op / 4, form op % 4 (any.b32, all.b32, any.b64, all.b64) ----------------------------------------
// Row r maps lane l to a class: rows 0..3 have 1, 2, 3 and 32 classes (32: class = lane), rows 4..15 a seeded count.
// Class c's .b32 value is V32(c); its .b64 value is H(c & ~1) : L(c & ~2), so classes c and c ^ 1 differ only in the
// low word and c and c ^ 2 only in the high word.
XL_HD unsigned match_classes(u64 seed, unsigned row) {
    return row < 3 ? row + 1 : row == 3 ? 32u : 1u + (unsigned)word(seed, CRO_XLANE_LEG_MATCH, row, 8, 0) % 32u;
}
XL_HD unsigned match_class(u64 seed, unsigned row, unsigned w, unsigned l) {
    const unsigned n = match_classes(seed, row);
    return n == 32 ? l : (unsigned)word(seed, CRO_XLANE_LEG_MATCH, row, w, l) % n;
}
XL_HD unsigned match_value32(u64 seed, unsigned row, unsigned w, unsigned l) {
    return (unsigned)word(seed, CRO_XLANE_LEG_MATCH, row, w, 32 + match_class(seed, row, w, l));
}
XL_HD u64 match_value64(u64 seed, unsigned row, unsigned w, unsigned l) {
    const unsigned c = match_class(seed, row, w, l);
    return (word(seed, CRO_XLANE_LEG_MATCH, row, 8 + w, c & ~1u) << 32) | (unsigned)word(seed, CRO_XLANE_LEG_MATCH, row, 8 + w, 32 + (c & ~2u));
}
// Lane l's results of the row's four forms: any = the lanes whose value equals its own; all = all ones and the
// predicate (bit 32) when every lane's value is equal, else 0.
XL_HD void match_results(u64 seed, unsigned row, unsigned w, unsigned l, u64 out[4]) {
    const unsigned a = match_value32(seed, row, w, l);
    const u64 b = match_value64(seed, row, w, l);
    unsigned m32 = 0, m64 = 0;
    for (unsigned j = 0; j < 32; ++j) {
        m32 |= (match_value32(seed, row, w, j) == a ? 1u : 0u) << j;
        m64 |= (match_value64(seed, row, w, j) == b ? 1u : 0u) << j;
    }
    out[0] = m32;
    out[1] = m32 == ~0u ? 0x1FFFFFFFFull : 0ull;
    out[2] = m64;
    out[3] = m64 == ~0u ? 0x1FFFFFFFFull : 0ull;
}

// ---- REDUX: row r = op / 9, form op % 9 (add.u32, add.s32, min.u32, max.u32, min.s32, max.s32, and, or, xor) -------
// rows 32k + j (k < 4): lane j alone is the u32 min (0: and the only clear bit j), the u32 max (~0: the only set bit
// j), the s32 min (0x80000000) and the s32 max (0x7FFFFFFF); rows 128..143 seeded.
XL_HD unsigned redux_operand(u64 seed, unsigned row, unsigned w, unsigned l) {
    const unsigned s = (unsigned)word(seed, CRO_XLANE_LEG_REDUX, row, w, l);
    if (row >= 128) return s;
    const unsigned j = row & 31u, me = l == j;
    switch (row >> 5) {
        case 0: return me ? 0u : s | (1u << j) | 1u;
        case 1: return me ? ~0u : s & ~(1u << j) & ~1u;
        case 2: return me ? 0x80000000u : s & 0x7FFFFFFFu;
        default: return me ? 0x7FFFFFFFu : s | 0x80000000u;
    }
}
XL_HD void redux_fold(unsigned form, unsigned* acc, unsigned x) {
    switch (form) {
        case 0: case 1: *acc += x; break;
        case 2: *acc = x < *acc ? x : *acc; break;
        case 3: *acc = x > *acc ? x : *acc; break;
        case 4: *acc = (int)x < (int)*acc ? x : *acc; break;
        case 5: *acc = (int)x > (int)*acc ? x : *acc; break;
        case 6: *acc &= x; break;
        case 7: *acc |= x; break;
        default: *acc ^= x; break;
    }
}
XL_HD unsigned redux_result(u64 seed, unsigned row, unsigned form, unsigned w) {
    unsigned acc = redux_operand(seed, row, w, 0);
    for (unsigned l = 1; l < 32; ++l) redux_fold(form, &acc, redux_operand(seed, row, w, l));
    return acc;
}

// ---- ATOMS: op = 4 * kind + shape -----------------------------------------------------------------------------------
// kinds: add.u32, inc, dec, min.u32, max.u32, min.s32, max.s32, and, or, xor, exch.b32, exch.b64, cas.b32, cas.b64,
// add.u64.  shapes: 0 one word for the CTA (256 participants, rank t), 1 one word per warp (32, rank l), 2 one word
// per lane index (8, rank w), 3 one word per thread, the 32 lanes of a warp on 32 words of one bank (1, rank 0).
enum { kAtAdd, kAtInc, kAtDec, kAtMinU, kAtMaxU, kAtMinS, kAtMaxS, kAtAnd, kAtOr, kAtXor, kAtExch, kAtExch64, kAtCas,
       kAtCas64, kAtAdd64, kAtKinds };
struct AtomsShape {
    unsigned group, rank, n;            // the thread's group (= its word), its rank in it, the group's size
    unsigned slot;                      // the group's 8-byte word in the arena
    unsigned base;                      // the group's n + 1 presence bytes
};
XL_HD AtomsShape atoms_shape(unsigned shape, unsigned w, unsigned l) {
    switch (shape) {
        case 0: return AtomsShape{0, 32 * w + l, 256, 0, 0};
        case 1: return AtomsShape{w, l, 32, w, 33 * w};
        case 2: return AtomsShape{l, w, 8, l, 9 * l};
        default: return AtomsShape{32 * w + l, 0, 1, 32 * l + w, 2 * (32 * w + l)};
    }
}
// The thread of rank r in group g of the shape.
XL_HD void atoms_member(unsigned shape, unsigned g, unsigned r, unsigned* w, unsigned* l) {
    switch (shape) {
        case 0: *w = r >> 5; *l = r & 31u; break;
        case 1: *w = g; *l = r; break;
        case 2: *w = r; *l = g; break;
        default: *w = g >> 5; *l = g & 31u; break;
    }
}
XL_HD u64 atoms_operand(u64 seed, unsigned op, unsigned w, unsigned l) { return word(seed, CRO_XLANE_LEG_ATOMS, op, w, l); }
// The group's initial word.
XL_HD u64 atoms_init(u64 seed, unsigned op, unsigned g) {
    const u64 v = word(seed, CRO_XLANE_LEG_ATOMS, op, 8 + (g >> 6), g & 63u);
    const unsigned kind = op / kAtomsShapes;
    if (kind == kAtInc) return v & 0x3FFFFFFFull;
    if (kind == kAtDec) return (v & 0x3FFFFFFFull) | 0x40000000ull;
    return kind == kAtExch64 || kind == kAtCas64 || kind == kAtAdd64 ? v : (v & 0xFFFFFFFFull);
}
// The value a thread gives the instruction: exch gives init ^ (rank + 1), so the init and the group's values mark
// presence slots 0 .. n; inc and dec give a bound that never wraps; cas adds its operand.
XL_HD u64 atoms_value(u64 seed, unsigned op, unsigned w, unsigned l) {
    const unsigned kind = op / kAtomsShapes;
    const u64 x = atoms_operand(seed, op, w, l);
    if (kind == kAtExch || kind == kAtExch64) {
        const AtomsShape s = atoms_shape(op % kAtomsShapes, w, l);
        const u64 v = atoms_init(seed, op, s.group) ^ (u64)(s.rank + 1);
        return kind == kAtExch ? (v & 0xFFFFFFFFull) : v;
    }
    if (kind == kAtInc) return (x | 0xC0000000ull) & 0xFFFFFFFFull;
    if (kind == kAtDec) return (x | 0x80000000ull) & 0xFFFFFFFFull;
    return kind == kAtCas64 || kind == kAtAdd64 ? x : (x & 0xFFFFFFFFull);
}
// The group's final word, from its initial word and its members' values as the kernel gives them (v: the value of
// member r, so a caller can change one).
template <class Value>
XL_HD u64 atoms_final(unsigned kind, unsigned n, u64 init, Value v) {
    u64 acc = init;
    for (unsigned r = 0; r < n; ++r) {
        const u64 x = v(r);
        switch (kind) {
            case kAtAdd: case kAtCas: acc = (acc + x) & 0xFFFFFFFFull; break;
            case kAtAdd64: case kAtCas64: acc += x; break;
            case kAtInc: acc += 1; break;
            case kAtDec: acc -= 1; break;
            case kAtMinU: acc = x < acc ? x : acc; break;
            case kAtMaxU: acc = x > acc ? x : acc; break;
            case kAtMinS: acc = (int)(unsigned)x < (int)(unsigned)acc ? x : acc; break;
            case kAtMaxS: acc = (int)(unsigned)x > (int)(unsigned)acc ? x : acc; break;
            case kAtAnd: acc &= x; break;
            case kAtOr: acc |= x; break;
            case kAtXor: acc ^= x; break;
            default: break;             // exch: the final word is one of the values; its presence is what is checked
        }
    }
    return acc;
}
// What a thread checks after the op: exch, its own value's presence slot (1 when marked); inc and dec, its rank's
// ticket slot (bit 0) and the final word (bits 32..63); every other kind the final word.
XL_HD u64 atoms_result(u64 seed, unsigned op, unsigned w, unsigned l) {
    const unsigned kind = op / kAtomsShapes, shape = op % kAtomsShapes;
    const AtomsShape s = atoms_shape(shape, w, l);
    if (kind == kAtExch || kind == kAtExch64) return 1;
    const u64 fin = atoms_final(kind, s.n, atoms_init(seed, op, s.group), [&](unsigned r) {
        unsigned mw, ml;
        atoms_member(shape, s.group, r, &mw, &ml);
        return atoms_value(seed, op, mw, ml);
    });
    return kind == kAtInc || kind == kAtDec ? (fin << 32) | 1u : fin;
}

// Every lane's expected result of every op of `leg` for warp w: out[op * 32 + lane] (the host's cro_xlane_expected).
inline void expected(unsigned leg, u64 seed, unsigned w, u64* out) {
    switch (leg) {
        case CRO_XLANE_LEG_SHFL:
            for (unsigned op = 0; op < CRO_XLANE_SHFL_OPS; ++op)
                for (unsigned l = 0; l < 32; ++l) {
                    bool p;
                    const unsigned j = shfl_source(shfl_op(op, l), l, &p);
                    out[op * 32 + l] = shfl_operand(seed, op, w, j) | ((u64)p << 32);
                }
            break;
        case CRO_XLANE_LEG_VOTE:
            for (unsigned row = 0; row < CRO_XLANE_VOTE_OPS / kVoteForms; ++row) {
                const unsigned b = vote_ballot(seed, row, w);
                for (unsigned f = 0; f < kVoteForms; ++f)
                    for (unsigned l = 0; l < 32; ++l) out[(row * kVoteForms + f) * 32 + l] = vote_result(f, b);
            }
            break;
        case CRO_XLANE_LEG_MATCH:
            for (unsigned row = 0; row < CRO_XLANE_MATCH_OPS / kMatchForms; ++row)
                for (unsigned l = 0; l < 32; ++l) {
                    u64 r[4];
                    match_results(seed, row, w, l, r);
                    for (unsigned f = 0; f < kMatchForms; ++f) out[(row * kMatchForms + f) * 32 + l] = r[f];
                }
            break;
        case CRO_XLANE_LEG_REDUX:
            for (unsigned op = 0; op < CRO_XLANE_REDUX_OPS; ++op) {
                const unsigned v = redux_result(seed, op / kReduxForms, op % kReduxForms, w);
                for (unsigned l = 0; l < 32; ++l) out[op * 32 + l] = v;
            }
            break;
        default:   // every member of a group checks the same value: one per group
            for (unsigned op = 0; op < CRO_XLANE_ATOMS_OPS; ++op) {
                unsigned g = ~0u;
                u64 v = 0;
                for (unsigned l = 0; l < 32; ++l) {
                    const unsigned h = atoms_shape(op % kAtomsShapes, w, l).group;
                    if (h != g) v = atoms_result(seed, op, w, l);
                    g = h;
                    out[op * 32 + l] = v;
                }
            }
            break;
    }
}

}  // namespace xlane
}  // namespace cro
