// pcd_codec.h -- exact per-token arithmetic of the ASCII PCD codec (DESIGN.md section 12), compiled for the device by
// pcd_kernels.cu and for the host by host_selftest.cpp, so that the CPU test-suite checks the very code the kernels run.
//
// Parse: a token of numpy's loadtxt grammar (optional sign; digits with an optional '.'; an optional e/E exponent with an optional
// sign; or nan / inf / infinity in any case with an optional sign) becomes the correctly rounded double (round-half-even), then
// (float) of that double.  Both host readers (np.loadtxt + astype(float32), istream >> double + (float)) round twice this way;
// a direct decimal -> float rounding differs near float midpoints.
//   - fast path (Clinger): at most 19 significant digits whose integer w is <= 2^53, and w * 10^e with |e| <= 22 (or w * 10^(e-22)
//     still <= 2^53): one IEEE multiplication or division of two exact doubles is the correctly rounded result;
//   - everything else is the slow path (parse_slow_abs): exact big-integer arithmetic in 32-bit limbs, no approximation decides.
// Format: exactly glibc's printf("%.8g", (double)f), which Python's "%.8g" % f equals; NaN is written "nan" whatever its sign.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define PCD_HD __host__ __device__ __forceinline__
#define PCD_HDN __host__ __device__ __noinline__
#else
#define PCD_HD inline
#define PCD_HDN inline
#endif

namespace pcd {

enum { TOK_OK = 0, TOK_SLOW = 1, TOK_INVALID = 2 };

PCD_HD bool is_ws(uint8_t c) { return c == ' ' || c == '\t' || c == '\r' || c == '\v' || c == '\f'; }
PCD_HD bool is_digit(uint8_t c) { return c >= '0' && c <= '9'; }
PCD_HD uint8_t lower(uint8_t c) { return (c >= 'A' && c <= 'Z') ? (uint8_t)(c + 32) : c; }

PCD_HD double bits_to_double(uint64_t b) {
    union { uint64_t u; double d; } v; v.u = b; return v.d;
}
PCD_HD uint64_t double_to_bits(double d) {
    union { uint64_t u; double d; } v; v.d = d; return v.u;
}
PCD_HD uint32_t float_to_bits(float f) {
    union { uint32_t u; float f; } v; v.f = f; return v.u;
}

// 10^k for 0 <= k <= 22: every partial product is an exactly representable double, so the loop is exact
PCD_HD double pow10_exact(int k) {
    double p = 1.0;
    for (int i = 0; i < k; ++i) p *= 10.0;
    return p;
}

// What the grammar scan learns about a token [s, s + n).
struct TokenScan {
    int kind;            // TOK_OK (value set), TOK_SLOW (needs parse_slow_abs), TOK_INVALID
    bool neg;
    double value;        // the correctly rounded double when kind == TOK_OK
};

// The grammar scan plus the fast path.  want_value = false only validates (a column that is not kept).
PCD_HD TokenScan scan_token(const uint8_t* s, uint64_t n, bool want_value) {
    TokenScan r{TOK_INVALID, false, 0.0};
    uint64_t i = 0;
    if (i < n && (s[i] == '+' || s[i] == '-')) { r.neg = s[i] == '-'; ++i; }
    if (i < n && !is_digit(s[i]) && s[i] != '.') {
        // nan / inf / infinity, any case
        const uint64_t m = n - i;
        const uint8_t* t = s + i;
        if (m == 3 && lower(t[0]) == 'n' && lower(t[1]) == 'a' && lower(t[2]) == 'n') {
            r.kind = TOK_OK;
            r.value = bits_to_double(r.neg ? 0xFFF8000000000000ull : 0x7FF8000000000000ull);
            return r;
        }
        bool inf = m == 3 || m == 8;
        const char* word = "infinity";
        for (uint64_t k = 0; inf && k < m; ++k) inf = lower(t[k]) == (uint8_t)word[k];
        if (inf) {
            r.kind = TOK_OK;
            r.value = bits_to_double(r.neg ? 0xFFF0000000000000ull : 0x7FF0000000000000ull);
        }
        return r;
    }
    // mantissa: the first 19 significant digits in w, the decimal exponent of w's last digit in e10
    uint64_t w = 0;
    int nsig = 0;                 // significant digits taken into w
    bool trunc = false;           // a nonzero digit was dropped after the 19th
    int64_t dropped = 0;          // integer-part digits dropped (each raises the exponent by one)
    int64_t frac_taken = 0;       // fraction digits that went into w (or were leading zeros)
    int ndig = 0;
    bool dot = false;
    for (; i < n; ++i) {
        const uint8_t c = s[i];
        if (c == '.') {
            if (dot) return r;
            dot = true;
            continue;
        }
        if (!is_digit(c)) break;
        ++ndig;
        const uint32_t d = c - '0';
        if (nsig == 0 && d == 0) {                   // leading zero
            if (dot) ++frac_taken;
            continue;
        }
        if (nsig < 19) {
            w = w * 10 + d;
            ++nsig;
            if (dot) ++frac_taken;
        } else {
            if (d) trunc = true;
            if (!dot) ++dropped;
        }
    }
    if (ndig == 0) return r;                         // "", ".", "e5", "+"
    int64_t ex = 0;
    if (i < n && (s[i] == 'e' || s[i] == 'E')) {
        ++i;
        bool eneg = false;
        if (i < n && (s[i] == '+' || s[i] == '-')) { eneg = s[i] == '-'; ++i; }
        if (i >= n || !is_digit(s[i])) return r;
        for (; i < n && is_digit(s[i]); ++i)
            if (ex < 100000000) ex = ex * 10 + (s[i] - '0');
        if (eneg) ex = -ex;
    }
    if (i != n) return r;
    r.kind = TOK_OK;
    if (!want_value) return r;
    if (w == 0) {                                    // every digit zero: a signed zero
        r.value = r.neg ? -0.0 : 0.0;
        return r;
    }
    if (trunc) { r.kind = TOK_SLOW; return r; }
    int64_t e10 = ex + dropped - frac_taken;
    while (w % 10 == 0) { w /= 10; ++e10; }         // trailing zeros only widen the fast path's reach
    const uint64_t two53 = 1ull << 53;
    if (w <= two53) {
        double v;
        if (e10 >= 0 && e10 <= 22) {
            v = (double)w * pow10_exact((int)e10);
        } else if (e10 < 0 && e10 >= -22) {
            v = (double)w / pow10_exact((int)-e10);
        } else if (e10 > 22 && e10 <= 22 + 15) {
            uint64_t ww = w;
            bool ok = true;
            for (int64_t k = 0; k < e10 - 22 && ok; ++k) { ww *= 10; ok = ww <= two53; }
            if (!ok) { r.kind = TOK_SLOW; return r; }
            v = (double)ww * 1e22;
        } else {
            r.kind = TOK_SLOW;
            return r;
        }
        r.value = r.neg ? -v : v;
        return r;
    }
    r.kind = TOK_SLOW;
    return r;
}

// ---- the slow path: exact big integers in 32-bit limbs --------------------------------------------------------------------
// At most kMaxDigits significant digits are kept; a longer token with a nonzero digit after them keeps kMaxDigits and appends a
// '1'.  No midpoint between two doubles has more than 767 significant digits, so a midpoint cannot lie strictly between the kept
// prefix and the prefix plus one unit of its last digit, and the appended digit leaves every comparison with a midpoint as it was.
constexpr int kMaxDigits = 780;
constexpr int kLimbs = 96;        // 3072 bits: D < 10^781 < 2^2595 and H 5^t < 2^55 5^1105 < 2^2622, aligned within one shift

struct Big {
    uint32_t w[kLimbs];
    int n;                        // limbs in use; w[n - 1] != 0 unless n == 0
};

PCD_HD void big_set(Big& a, uint64_t v) {
    a.n = 0;
    while (v) { a.w[a.n++] = (uint32_t)v; v >>= 32; }
}
PCD_HD void big_mul_add(Big& a, uint32_t m, uint32_t add) {
    uint64_t carry = add;
    for (int i = 0; i < a.n; ++i) {
        const uint64_t t = (uint64_t)a.w[i] * m + carry;
        a.w[i] = (uint32_t)t;
        carry = t >> 32;
    }
    if (carry && a.n < kLimbs) a.w[a.n++] = (uint32_t)carry;
}
// a *= 5^k
PCD_HD void big_mul_pow5(Big& a, int k) {
    while (k >= 13) { big_mul_add(a, 1220703125u, 0); k -= 13; }     // 5^13
    uint32_t m = 1;
    while (k-- > 0) m *= 5;
    if (m != 1) big_mul_add(a, m, 0);
}
PCD_HD void big_shl(Big& a, int k) {
    if (!a.n || k <= 0) return;
    const int limbs = k >> 5, bits = k & 31;
    int n = a.n + limbs + 1;
    if (n > kLimbs) n = kLimbs;
    for (int i = n - 1; i >= 0; --i) {
        const int src = i - limbs;
        uint32_t v = 0;
        if (src >= 0 && src < a.n) v = bits ? (a.w[src] << bits) : a.w[src];
        if (bits && src - 1 >= 0 && src - 1 < a.n) v |= a.w[src - 1] >> (32 - bits);
        a.w[i] = v;
    }
    a.n = n;
    while (a.n && !a.w[a.n - 1]) --a.n;
}
PCD_HD int big_bits(const Big& a) {
    if (!a.n) return 0;
    uint32_t t = a.w[a.n - 1];
    int b = 0;
    while (t) { ++b; t >>= 1; }
    return 32 * (a.n - 1) + b;
}
PCD_HD int big_cmp(const Big& a, const Big& b) {
    if (a.n != b.n) return a.n < b.n ? -1 : 1;
    for (int i = a.n - 1; i >= 0; --i)
        if (a.w[i] != b.w[i]) return a.w[i] < b.w[i] ? -1 : 1;
    return 0;
}
// bit k of a
PCD_HD uint32_t big_bit(const Big& a, int k) { return (k >> 5) < a.n ? (a.w[k >> 5] >> (k & 31)) & 1u : 0u; }
// the top 64 bits of a (a != 0) as an integer, and whether any bit below them is set
PCD_HD uint64_t big_top64(const Big& a, int nbits, bool& sticky) {
    uint64_t v = 0;
    const int lo = nbits > 64 ? nbits - 64 : 0;
    for (int k = nbits - 1; k >= lo; --k) v = (v << 1) | big_bit(a, k);
    sticky = false;
    for (int k = 0; k < lo && !sticky; ++k) sticky = big_bit(a, k) != 0;
    return v;
}

// sign(D * 10^-t - H * 2^K) for t > 0: D 2^-t 5^-t vs H 2^K  <=>  D 2^(-t-K) vs H 5^t
PCD_HD int cmp_dec_bin(const Big& D, int t, uint64_t H, int K, Big& tmpA, Big& tmpB) {
    tmpA = D;
    big_set(tmpB, H);
    big_mul_pow5(tmpB, t);
    const int sh = -t - K;
    if (sh >= 0) big_shl(tmpA, sh); else big_shl(tmpB, -sh);
    return big_cmp(tmpA, tmpB);
}

// m * 2^k with m an integer: the double b > 0 (finite) as (m, k)
PCD_HD void decompose(double b, uint64_t& m, int& k) {
    const uint64_t u = double_to_bits(b);
    const int be = (int)((u >> 52) & 0x7FF);
    const uint64_t f = u & ((1ull << 52) - 1);
    if (be == 0) { m = f; k = -1074; }
    else { m = f | (1ull << 52); k = be - 1075; }
}

// The correctly rounded double of a token the fast path sent here (positive magnitude; the caller applies the sign).  The token
// has passed scan_token.  Scratch: three Bigs (about 1.2 KB) in local memory on the device.
PCD_HDN double parse_slow_abs(const uint8_t* s, uint64_t n, Big& D, Big& A, Big& B) {
    uint64_t i = 0;
    if (i < n && (s[i] == '+' || s[i] == '-')) ++i;
    // D = the first kMaxDigits significant digits (+ a sticky '1'), e10 = the exponent of D's last digit
    D.n = 0;
    int nsig = 0;
    bool dot = false, trunc = false;
    int64_t dropped = 0, frac_taken = 0;
    uint32_t chunk = 0, chunk_mul = 1;
    for (; i < n; ++i) {
        const uint8_t c = s[i];
        if (c == '.') { dot = true; continue; }
        if (!is_digit(c)) break;
        const uint32_t d = c - '0';
        if (nsig == 0 && d == 0) { if (dot) ++frac_taken; continue; }
        if (nsig < kMaxDigits) {
            chunk = chunk * 10 + d;
            chunk_mul *= 10;
            if (chunk_mul == 1000000000u) { big_mul_add(D, chunk_mul, chunk); chunk = 0; chunk_mul = 1; }
            ++nsig;
            if (dot) ++frac_taken;
        } else {
            if (d) trunc = true;
            if (!dot) ++dropped;
        }
    }
    if (trunc) {
        chunk = chunk * 10 + 1;
        chunk_mul *= 10;
        if (chunk_mul == 1000000000u) { big_mul_add(D, chunk_mul, chunk); chunk = 0; chunk_mul = 1; }
        ++frac_taken;                                 // the appended digit sits one place below the last kept one
        ++nsig;
    }
    if (chunk_mul != 1) big_mul_add(D, chunk_mul, chunk);
    int64_t ex = 0;
    if (i < n && (s[i] == 'e' || s[i] == 'E')) {
        ++i;
        bool eneg = false;
        if (i < n && (s[i] == '+' || s[i] == '-')) { eneg = s[i] == '-'; ++i; }
        for (; i < n && is_digit(s[i]); ++i)
            if (ex < 100000000) ex = ex * 10 + (s[i] - '0');
        if (eneg) ex = -ex;
    }
    if (!D.n) return 0.0;
    const int64_t e10 = ex + dropped - frac_taken;
    // 10^(nsig + e10 - 1) <= value < 10^(nsig + e10)
    if (nsig + e10 - 1 >= 309) return bits_to_double(0x7FF0000000000000ull);     // >= 1e309 > DBL_MAX + ulp/2
    if (nsig + e10 <= -324) return 0.0;                                          // < 1e-324 < min subnormal / 2
    if (e10 >= 0) {
        // value = D 5^e10 2^e10, an integer: round its top 53 bits, half to even
        big_mul_pow5(D, (int)e10);
        const int nb = big_bits(D);
        uint64_t m;
        int sh = 0;
        if (nb <= 53) {
            bool st;
            m = big_top64(D, nb, st);
        } else {
            sh = nb - 53;
            uint64_t v = 0;
            for (int k = nb - 1; k >= sh; --k) v = (v << 1) | big_bit(D, k);
            const uint32_t rb = big_bit(D, sh - 1);
            bool sticky = false;
            for (int k = 0; k < sh - 1 && !sticky; ++k) sticky = big_bit(D, k) != 0;
            m = v;
            if (rb && (sticky || (m & 1))) ++m;
            if (m == (1ull << 53)) { m >>= 1; ++sh; }
        }
        const int be = (int)e10 + sh;                 // value = m 2^be
        if (be + 53 > 1024) return bits_to_double(0x7FF0000000000000ull);
        double r = (double)m;                         // exact (m < 2^53 + 1 and even when it is 2^53)
        for (int k = 0; k < be; ++k) r *= 2.0;        // exact scaling up to the overflow checked above
        return r;
    }
    // e10 < 0: value = D / 10^t.  A candidate from the top 64 bits of D and of 5^t, then exact comparisons with the midpoints.
    const int t = (int)-e10;
    big_set(A, 1);
    big_mul_pow5(A, t);
    bool st;
    const int nbD = big_bits(D), nbP = big_bits(A);
    const double dq = (double)big_top64(D, nbD, st) / (double)big_top64(A, nbP, st);
    int sc = (nbD > 64 ? nbD - 64 : 0) - (nbP > 64 ? nbP - 64 : 0) - t;   // value ~= dq 2^sc
    double b = dq;
    while (sc > 0) { b *= 2.0; --sc; }
    while (sc < -600) { b *= 0x1p-600; sc += 600; }
    if (sc < 0) b *= bits_to_double((uint64_t)(1023 + sc) << 52);            // 2^sc, exact for sc >= -1022
    if (!(b < bits_to_double(0x7FF0000000000000ull))) b = bits_to_double(0x7FEFFFFFFFFFFFFFull);
    for (int iter = 0; iter < 64; ++iter) {
        uint64_t m;
        int k;
        decompose(b, m, k);
        // upper midpoint (2m + 1) 2^(k - 1)
        const int cu = cmp_dec_bin(D, t, 2 * m + 1, k - 1, A, B);
        if (cu > 0 || (cu == 0 && (m & 1))) {
            if (b == bits_to_double(0x7FEFFFFFFFFFFFFFull)) return bits_to_double(0x7FF0000000000000ull);
            b = bits_to_double(double_to_bits(b) + 1);
            if (cu == 0) return b;
            continue;
        }
        if (m == 0) return b;
        // lower midpoint: (2m - 1) 2^(k - 1), or (4m - 1) 2^(k - 2) where the binade starts (m = 2^52 of a normal)
        const bool edge = m == (1ull << 52) && k > -1074;
        const int cl = edge ? cmp_dec_bin(D, t, 4 * m - 1, k - 2, A, B) : cmp_dec_bin(D, t, 2 * m - 1, k - 1, A, B);
        if (cl < 0 || (cl == 0 && (m & 1))) {
            b = bits_to_double(double_to_bits(b) - 1);
            if (cl == 0) return b;
            continue;
        }
        return b;
    }
    return b;
}

// ---- format: printf("%.8g", (double)f) ----------------------------------------------------------------------------------
// |f| = M 2^E exactly (M < 2^24, -149 <= E <= 104).  The decimal exponent X (10^X <= |f| < 10^(X+1)) and the rounded eight-digit
// q = round_half_even(|f| / 10^(X-7)) are found from double estimates corrected by exact comparisons of M 2^E with H 10^s
// (H < 2^28, -52 <= s <= 39) in 192-bit integers: 5^52 < 2^121, so M 5^52 < 2^145 and the two sides, of like size, fit once aligned
// (a shift that would overflow decides the comparison by itself).
struct U192 { uint64_t w[3]; };

PCD_HD void mul64(uint64_t a, uint64_t b, uint64_t& hi, uint64_t& lo) {
#if defined(__CUDA_ARCH__)
    lo = a * b;
    hi = __umul64hi(a, b);
#else
    const unsigned __int128 p = (unsigned __int128)a * b;
    lo = (uint64_t)p;
    hi = (uint64_t)(p >> 64);
#endif
}
PCD_HD void u_mul(U192& a, uint64_t m) {
    uint64_t carry = 0;
    for (int i = 0; i < 3; ++i) {
        uint64_t hi, lo;
        mul64(a.w[i], m, hi, lo);
        lo += carry;
        hi += lo < carry;
        a.w[i] = lo;
        carry = hi;
    }
}
PCD_HD void u_pow5(U192& a, int k) {
    while (k >= 27) { u_mul(a, 7450580596923828125ull); k -= 27; }   // 5^27
    uint64_t m = 1;
    while (k-- > 0) m *= 5;
    u_mul(a, m);
}
PCD_HD int u_bits(const U192& a) {
    for (int i = 2; i >= 0; --i)
        if (a.w[i]) {
            int b = 0;
            uint64_t t = a.w[i];
            while (t) { ++b; t >>= 1; }
            return 64 * i + b;
        }
    return 0;
}
// a <<= k; false when bits would be lost
PCD_HD bool u_shl(U192& a, int k) {
    if (k <= 0) return true;
    if (u_bits(a) + k > 192) return false;
    while (k >= 64) { a.w[2] = a.w[1]; a.w[1] = a.w[0]; a.w[0] = 0; k -= 64; }
    if (k) {
        a.w[2] = (a.w[2] << k) | (a.w[1] >> (64 - k));
        a.w[1] = (a.w[1] << k) | (a.w[0] >> (64 - k));
        a.w[0] <<= k;
    }
    return true;
}
PCD_HD int u_cmp(const U192& a, const U192& b) {
    for (int i = 2; i >= 0; --i)
        if (a.w[i] != b.w[i]) return a.w[i] < b.w[i] ? -1 : 1;
    return 0;
}
// sign(M 2^E - H 10^s), all positive
PCD_HD int cmp_bin_dec(uint64_t M, int E, uint64_t H, int s) {
    U192 a{{M, 0, 0}}, b{{H, 0, 0}};
    int ea = E, eb = 0;
    if (s >= 0) { u_pow5(b, s); eb = s; }           // H 5^s 2^s
    else { u_pow5(a, -s); eb = s; }                 // M 5^-s 2^E vs H 2^s
    if (ea >= eb) { if (!u_shl(a, ea - eb)) return 1; }
    else { if (!u_shl(b, eb - ea)) return -1; }
    return u_cmp(a, b);
}

// printf("%.8g") of f into out (at most 15 bytes); returns the length
PCD_HD int format_g8(float f, char* out) {
    const uint32_t u = float_to_bits(f);
    const bool neg = u >> 31;
    const uint32_t be = (u >> 23) & 0xFF, fr = u & 0x7FFFFF;
    int p = 0;
    if (be == 0xFF) {
        if (fr) { out[0] = 'n'; out[1] = 'a'; out[2] = 'n'; return 3; }
        if (neg) out[p++] = '-';
        out[p++] = 'i'; out[p++] = 'n'; out[p++] = 'f';
        return p;
    }
    if (neg) out[p++] = '-';
    if (be == 0 && fr == 0) { out[p++] = '0'; return p; }
    const uint64_t M = be ? (fr | 0x800000u) : fr;
    const int E = be ? (int)be - 150 : -149;
    const double av = neg ? -(double)f : (double)f;   // |f|, exact
    // X: estimate from the binary exponent, then exact corrections
    int bl = 0;
    { uint64_t t = M; while (t) { ++bl; t >>= 1; } }
    int X = (int)((double)(bl - 1 + E) * 0.30102999566398120);
    if ((bl - 1 + E) < 0 && (double)X != (double)(bl - 1 + E) * 0.30102999566398120) --X;   // floor for negatives
    while (cmp_bin_dec(M, E, 1, X) < 0) --X;
    while (cmp_bin_dec(M, E, 1, X + 1) >= 0) ++X;
    // q: nearest integer to |f| / 10^(X - 7), half to even
    const int s = X - 7;
    double sc = av;
    if (s > 0) { for (int k = 0; k < s; ++k) sc /= 10.0; }
    else { for (int k = 0; k < -s; ++k) sc *= 10.0; }
    uint64_t q = (uint64_t)(sc + 0.5);
    if (q < 10000000ull) q = 10000000ull;
    if (q > 100000000ull) q = 100000000ull;
    for (int it = 0; it < 8; ++it) {
        // 2|f| vs (2q + 1) 10^s and (2q - 1) 10^s
        const int cu = cmp_bin_dec(M, E + 1, 2 * q + 1, s);
        if (cu > 0 || (cu == 0 && (q & 1))) { ++q; if (cu == 0) break; continue; }
        const int cl = cmp_bin_dec(M, E + 1, 2 * q - 1, s);
        if (cl < 0 || (cl == 0 && (q & 1))) { --q; if (cl == 0) break; continue; }
        break;
    }
    if (q == 100000000ull) { q = 10000000ull; ++X; }
    char dg[8];
    for (int k = 7; k >= 0; --k) { dg[k] = (char)('0' + q % 10); q /= 10; }
    int nd = 8;
    while (nd > 1 && dg[nd - 1] == '0') --nd;       // significant digits left after stripping trailing zeros
    if (X < -4 || X >= 8) {
        out[p++] = dg[0];
        if (nd > 1) {
            out[p++] = '.';
            for (int k = 1; k < nd; ++k) out[p++] = dg[k];
        }
        out[p++] = 'e';
        int ax = X;
        out[p++] = ax < 0 ? '-' : '+';
        if (ax < 0) ax = -ax;
        if (ax >= 100) { out[p++] = (char)('0' + ax / 100); ax %= 100; out[p++] = (char)('0' + ax / 10); out[p++] = (char)('0' + ax % 10); }
        else { out[p++] = (char)('0' + ax / 10); out[p++] = (char)('0' + ax % 10); }
        return p;
    }
    if (X >= 0) {
        for (int k = 0; k <= X; ++k) out[p++] = dg[k];
        if (nd > X + 1) {
            out[p++] = '.';
            for (int k = X + 1; k < nd; ++k) out[p++] = dg[k];
        }
        return p;
    }
    out[p++] = '0';
    out[p++] = '.';
    for (int k = 0; k < -X - 1; ++k) out[p++] = '0';
    for (int k = 0; k < nd; ++k) out[p++] = dg[k];
    return p;
}

}  // namespace pcd
