// Exact, order-independent summation of float contributions: the gradient accumulators of the deterministic backward pass
// (rb_options::deterministic, DESIGN.md section 2).  Host and device code; the device scatter that feeds these accumulators from
// the kernels is in rb_atomic.cuh.
//
// Format.  One accumulator is RB_EXACT_WORDS 64-bit words: RB_EXACT_LIMBS signed limbs, limb k weighing 2^(32 k - 149), then a
// flag word.  Every finite float is m * 2^(p - 149) with an integer 0 <= m < 2^24 and 0 <= p <= 253 (p = biased exponent - 1, or
// 0 for a subnormal), so m << (p & 31) < 2^55 splits into a chunk < 2^32 for limb p >> 5 (<= 7) and a chunk < 2^23 for the next
// limb (<= 8).  Limb 9 only receives carries.  Integer addition is associative, so the limbs hold the exact sum whatever the order.
// Non-finite contributions only set flag bits: the result is NaN after a NaN or after both infinities, else +-inf after one of
// them -- what IEEE summation gives in any order.
//
// Overflow bound.  exact_normalise leaves limbs 0..8 in [0, 2^32); one contribution changes a limb by less than 2^32, so after at
// most RB_EXACT_MAX_ADDS contributions to one accumulator every limb is below 2^32 + (2^31 - 2)(2^32 - 1) < 2^63 in magnitude.
// Whoever adds more must normalise in between (the driver does it after every band).  Limb 9 holds the sum over 2^288 and stays
// far from overflow: |sum| < n * 2^277 for n contributions.
#pragma once
#include <string.h>

#include "rb_math.cuh"

#define RB_EXACT_LIMBS 10
#define RB_EXACT_WORDS (RB_EXACT_LIMBS + 1)
#define RB_EXACT_MAX_ADDS ((1LL << 31) - 2)
enum { RB_EXACT_POS_INF = 1, RB_EXACT_NEG_INF = 2, RB_EXACT_NAN = 4 };
// Gradient buffers are handed to the deterministic kernels as VIRTUAL addresses: element i of the accumulator array is the float
// at RB_EXACT_VBASE + 4 i.  The scatter finds an element's accumulator by subtracting the base; NULL stays NULL, and a kernel that
// dereferenced such an address would fault instead of writing somewhere.
#define RB_EXACT_VBASE ((uintptr_t)4096)
RB_HD float* exact_virtual(long long i) { return (float*)(RB_EXACT_VBASE + 4 * (uintptr_t)i); }
RB_HD long long* exact_slot(long long* acc, const float* addr) { return acc + (((uintptr_t)addr - RB_EXACT_VBASE) >> 2) * RB_EXACT_WORDS; }
// Accumulators [first, first + count) stand for the caller's floats dst[0, count).
struct ExactRange {
    long long first, count;
    float* dst;
};

RB_HD unsigned exact_bits(float v) {
    unsigned u;
    memcpy(&u, &v, 4);
    return u;
}
RB_HD float exact_float(unsigned u) {
    float v;
    memcpy(&v, &u, 4);
    return v;
}
// One contribution split into its two limb chunks (signed) or its flag.
struct ExactTerm {
    int limb;
    long long lo, hi;
    unsigned flag;
};
RB_HD ExactTerm exact_term(float v) {
    const unsigned u = exact_bits(v), e = (u >> 23) & 0xffu;
    unsigned m = u & 0x7fffffu;
    ExactTerm t;
    t.limb = 0;
    t.lo = t.hi = 0;
    t.flag = 0;
    if (e == 0xffu) {
        t.flag = m ? RB_EXACT_NAN : (u >> 31) ? RB_EXACT_NEG_INF : RB_EXACT_POS_INF;
        return t;
    }
    if (e) m |= 0x800000u;
    const int p = e ? (int)e - 1 : 0;
    const unsigned long long w = (unsigned long long)m << (p & 31);
    t.limb = p >> 5;
    t.lo = (long long)(w & 0xffffffffull);
    t.hi = (long long)(w >> 32);
    if (u >> 31) {
        t.lo = -t.lo;
        t.hi = -t.hi;
    }
    return t;
}
// Single-threaded add (host code and the host emulator).  A zero contributes nothing, so it is not written at all.
RB_HD void exact_add_serial(long long* acc, float v) {
    if (v == 0.f) return;
    const ExactTerm t = exact_term(v);
    acc[RB_EXACT_LIMBS] |= (long long)t.flag;
    acc[t.limb] += t.lo;
    acc[t.limb + 1] += t.hi;
}
// Carry propagation: limbs 0..8 into [0, 2^32), the rest into limb 9.  The value is unchanged.
RB_HD void exact_normalise(long long* acc) {
    for (int k = 0; k < RB_EXACT_LIMBS - 1; k++) {
        const long long low = (long long)((unsigned long long)acc[k] & 0xffffffffull);
        acc[k + 1] += (acc[k] - low) / 4294967296LL; // exact: acc[k] - low is a multiple of 2^32
        acc[k] = low;
    }
}
// An accumulator that received a non-zero sum or a non-finite value; the others are left alone by the finalisation.
RB_HD bool exact_touched(const long long* acc) {
    for (int k = 0; k < RB_EXACT_WORDS; k++)
        if (acc[k] != 0) return true;
    return false;
}
// Round the exact value to PREC significant bits, to nearest with ties to even.  Returns the sign, the integer significand
// m < 2^PREC and the exponent: value = (-1)^neg * m * 2^(e - 149).  m == 0 for a zero sum.  Non-finite flags are the caller's.
template <int PREC>
RB_HD void exact_round(const long long* acc_in, bool& neg, unsigned long long& m, int& e) {
    long long a[RB_EXACT_LIMBS];
    for (int k = 0; k < RB_EXACT_LIMBS; k++) a[k] = acc_in[k];
    exact_normalise(a);
    // two's complement words of 32 bits, low first: limbs 0..8, then the 64 bits of limb 9 and its sign extension
    unsigned w[RB_EXACT_LIMBS + 4];
    for (int k = 0; k < RB_EXACT_LIMBS - 1; k++) w[k] = (unsigned)a[k];
    const unsigned long long top = (unsigned long long)a[RB_EXACT_LIMBS - 1];
    neg = a[RB_EXACT_LIMBS - 1] < 0;
    w[RB_EXACT_LIMBS - 1] = (unsigned)top;
    w[RB_EXACT_LIMBS] = (unsigned)(top >> 32);
    w[RB_EXACT_LIMBS + 1] = w[RB_EXACT_LIMBS + 2] = w[RB_EXACT_LIMBS + 3] = neg ? 0xffffffffu : 0u;
    const int nw = RB_EXACT_LIMBS + 4;
    if (neg) { // magnitude: invert and add one
        unsigned carry = 1;
        for (int k = 0; k < nw; k++) {
            const unsigned long long s = (unsigned long long)(~w[k]) + carry;
            w[k] = (unsigned)s;
            carry = (unsigned)(s >> 32);
        }
    }
    int h = -1; // highest set bit
    for (int k = nw - 1; k >= 0 && h < 0; k--)
        if (w[k]) {
            int b = 31;
            while (!((w[k] >> b) & 1u)) b--;
            h = 32 * k + b;
        }
    m = 0;
    e = 0;
    if (h < 0) return;
    const int shift = h < PREC ? 0 : h - PREC + 1; // lowest kept bit
    // PREC bits from `shift` (PREC + 31 <= 84 bits span at most three words)
    const int q = shift >> 5, r = shift & 31;
    const unsigned long long w0 = w[q], w1 = q + 1 < nw ? w[q + 1] : 0u, w2 = q + 2 < nw ? w[q + 2] : 0u;
    unsigned long long bits = ((w0 | (w1 << 32)) >> r) | (r ? (w2 << (64 - r)) : 0ull);
    m = bits & ((1ull << PREC) - 1ull);
    if (shift > 0) {
        const int rb = shift - 1;
        const bool round = (w[rb >> 5] >> (rb & 31)) & 1u;
        bool sticky = false;
        for (int k = 0; k < (rb >> 5) && !sticky; k++) sticky = w[k] != 0;
        if (!sticky && (rb & 31)) sticky = (w[rb >> 5] & ((1u << (rb & 31)) - 1u)) != 0;
        if (round && (sticky || (m & 1ull))) m++;
    }
    e = shift;
    if (m >> PREC) { // rounding carried into a new bit
        m >>= 1;
        e++;
    }
}
// The correctly rounded float of the exact sum (+-inf beyond the float range), with the flags' non-finite rules.
RB_HD float exact_to_float(const long long* acc) {
    const unsigned f = (unsigned)acc[RB_EXACT_LIMBS];
    if ((f & RB_EXACT_NAN) || (f & (RB_EXACT_POS_INF | RB_EXACT_NEG_INF)) == (RB_EXACT_POS_INF | RB_EXACT_NEG_INF)) return exact_float(0x7fc00000u);
    if (f & RB_EXACT_POS_INF) return exact_float(0x7f800000u);
    if (f & RB_EXACT_NEG_INF) return exact_float(0xff800000u);
    bool neg;
    unsigned long long m;
    int e;
    exact_round<24>(acc, neg, m, e);
    // m * 2^(e - 149) with m < 2^24: for e == 0 the bit pattern is m itself (a subnormal, or the smallest normals when bit 23 is set);
    // otherwise m has bit 23 set and (e << 23) + m puts biased exponent e + 1 above the 23 stored bits
    const unsigned long long pattern = ((unsigned long long)e << 23) + m;
    const unsigned mag = pattern >= 0x7f800000ull ? 0x7f800000u : (unsigned)pattern;
    return exact_float(mag | (neg ? 0x80000000u : 0u));
}
// The correctly rounded double of the exact sum (it cannot overflow a double).
RB_HD double exact_to_double(const long long* acc) {
    const unsigned f = (unsigned)acc[RB_EXACT_LIMBS];
    if ((f & RB_EXACT_NAN) || (f & (RB_EXACT_POS_INF | RB_EXACT_NEG_INF)) == (RB_EXACT_POS_INF | RB_EXACT_NEG_INF)) return (double)exact_float(0x7fc00000u);
    if (f & RB_EXACT_POS_INF) return (double)exact_float(0x7f800000u);
    if (f & RB_EXACT_NEG_INF) return (double)exact_float(0xff800000u);
    bool neg;
    unsigned long long m;
    int e;
    exact_round<53>(acc, neg, m, e);
    const double v = ldexp((double)m, e - 149); // exact: m < 2^53 and the exponent stays inside the double range
    return neg ? -v : v;
}
// The range of accumulator i: the last of `ranges` (sorted by `first`) with first <= i.
RB_HD int exact_range_of(long long i, const ExactRange* ranges, int num_ranges) {
    int lo = 0, hi = num_ranges - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (ranges[mid].first <= i) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}
// Finalisation of accumulator i of a backward pass (the CUDA kernel k_exact_finalise and the host emulator): nothing if it received
// nothing; the first `num_cam` accumulators are the camera scalars and become doubles in cam_accum; any other is rounded to float
// and added once into the caller's element it stands for (`ranges` sorted by `first`).
RB_HD void exact_finalise(const long long* acc_all, long long i, const ExactRange* ranges, int num_ranges, double* cam_accum, int num_cam) {
    const long long* a = acc_all + i * RB_EXACT_WORDS;
    if (!exact_touched(a)) return;
    if (i < num_cam) {
        cam_accum[i] = exact_to_double(a);
        return;
    }
    const int r = exact_range_of(i, ranges, num_ranges);
    ranges[r].dst[i - ranges[r].first] += exact_to_float(a);
}

// Records: the form in which the accumulators of a backward pass leave one call (rb_render_exact) and come back to another
// (rb_exact_round), possibly summed over calls, devices and processes in between.  One record is RB_EXACT_RECORD_WORDS signed 64-bit
// words: the RB_EXACT_LIMBS limbs, then three COUNTS of non-finite contributions (+inf, -inf, NaN).  A sum of records, word by word, is
// the record of the summed contributions: the limbs because integer addition is associative, the counts because a count stays
// non-zero once set -- unlike the OR-ed flag bits of an accumulator, which a sum would turn into other bits (two +inf flags would add
// up to the -inf flag).  Records are handed out normalised (exact_normalise), so N summed records have limbs below N * 2^32; an import
// normalises again before anything looks at them.  Where a record sits depends on the structure of the gradient descriptor only
// (ExactLayout::rec_first), not on where its buffers are.
#define RB_EXACT_RECORD_WORDS (RB_EXACT_LIMBS + 3)
// Record of accumulator i: the camera's first (record i), then rec_first[r] + (i - ranges[r].first) in range r.
RB_HD long long exact_record_of(long long i, const ExactRange* ranges, const long long* rec_first, int num_ranges, int num_cam) {
    if (i < num_cam) return i;
    const int r = exact_range_of(i, ranges, num_ranges);
    return rec_first[r] + (i - ranges[r].first);
}
// Adds accumulator `acc` into record `rec` and leaves the record normalised.
RB_HD void exact_export(const long long* acc, long long* rec) {
    long long a[RB_EXACT_LIMBS];
    for (int k = 0; k < RB_EXACT_LIMBS; k++) a[k] = acc[k] + rec[k];
    exact_normalise(a);
    for (int k = 0; k < RB_EXACT_LIMBS; k++) rec[k] = a[k];
    const long long f = acc[RB_EXACT_LIMBS];
    rec[RB_EXACT_LIMBS] += (f & RB_EXACT_POS_INF) ? 1 : 0;
    rec[RB_EXACT_LIMBS + 1] += (f & RB_EXACT_NEG_INF) ? 1 : 0;
    rec[RB_EXACT_LIMBS + 2] += (f & RB_EXACT_NAN) ? 1 : 0;
}
// Accumulator `acc` from record `rec` (a sum of records, maybe): normalised limbs and the flag bits of the non-zero counts.  A record
// whose value is zero and whose counts are zero gives an untouched accumulator, whatever its raw words were.
RB_HD void exact_import(const long long* rec, long long* acc) {
    long long a[RB_EXACT_LIMBS];
    for (int k = 0; k < RB_EXACT_LIMBS; k++) a[k] = rec[k];
    exact_normalise(a);
    for (int k = 0; k < RB_EXACT_LIMBS; k++) acc[k] = a[k];
    acc[RB_EXACT_LIMBS] = (rec[RB_EXACT_LIMBS] ? RB_EXACT_POS_INF : 0) | (rec[RB_EXACT_LIMBS + 1] ? RB_EXACT_NEG_INF : 0) | (rec[RB_EXACT_LIMBS + 2] ? RB_EXACT_NAN : 0);
}
