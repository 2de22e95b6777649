// chain.h — the re-quantising descent ("chain") arithmetic, shared by the CUDA kernels and the host
// orchestration.  Every operation is IEEE-754 binary64 in the reference's exact order; this header
// must be compiled with FMA contraction OFF (nvcc -fmad=false, g++ -ffp-contract=off): the only fused
// operations are the two explicit fma() calls that restate `mul_add` in the reference's decode.
//
// Reference semantics (file:line relative to the reference checkout):
//   child index      src/octree/node.rs:34-42      strict `>` against Cube::center (aabb.rs:184-192)
//   child cube       src/octree/node.rs:157-172    e /= 2; min += bit * e
//   encode           src/read_write/codec.rs:102-121,142-148  clamp((v-min)/edge,0,1) * MAX -> `as` cast
//   decode           src/read_write/codec.rs:124-139  (v / MAX).mul_add(edge, min)
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define PCV_HD __host__ __device__ __forceinline__
#else
#define PCV_HD inline
#include <cmath>
#include <cstring>
#endif

namespace pcv {

enum : int { ENC_U8 = 1, ENC_U16 = 2, ENC_F32 = 3, ENC_F64 = 4 };
constexpr int kMaxLevels = 41;  // NodeId holds a 120-bit octal path: levels 0..40 (node.rs:152-154)

PCV_HD int enc_bytes(int enc) { return enc == ENC_U8 ? 1 : enc == ENC_U16 ? 2 : enc == ENC_F32 ? 4 : 8; }

PCV_HD double bits_to_f64(uint64_t b) {
#if defined(__CUDA_ARCH__)
    return __longlong_as_double((long long)b);
#else
    double d;
    memcpy(&d, &b, 8);
    return d;
#endif
}
PCV_HD uint64_t f64_to_bits(double d) {
#if defined(__CUDA_ARCH__)
    return (uint64_t)__double_as_longlong(d);
#else
    uint64_t b;
    memcpy(&b, &d, 8);
    return b;
#endif
}
PCV_HD float bits_to_f32(uint32_t b) {
#if defined(__CUDA_ARCH__)
    return __uint_as_float(b);
#else
    float f;
    memcpy(&f, &b, 4);
    return f;
#endif
}
PCV_HD uint32_t f32_to_bits(float f) {
#if defined(__CUDA_ARCH__)
    return __float_as_uint(f);
#else
    uint32_t b;
    memcpy(&b, &f, 4);
    return b;
#endif
}

// num::clamp (num 0.3.0): NaN passes through.
PCV_HD double clamp01(double x) {
    if (x < 0.0) return 0.0;
    if (x > 1.0) return 1.0;
    return x;
}

// Rust `f64 as u16/u8` as the callers need it (they cap the result at 255 / 65535): truncate toward zero, NaN -> 0,
// negative -> 0, huge -> saturated.  On the GPU this goes through the SIGNED conversion:
// cvt.rzi.u32.f64 returns 0x80000000 for NaN (not 0), while cvt.rzi.s32.f64 gives INT_MIN for NaN / -inf and INT_MAX
// for +inf / huge, so max(v, 0) has exactly the semantics of the Rust cast below 2^31.
PCV_HD uint32_t trunc_u32(double s) {
#if defined(__CUDA_ARCH__)
    const int v = __double2int_rz(s);
    return (uint32_t)(v < 0 ? 0 : v);
#else
    if (!(s == s)) return 0u;
    if (s <= 0.0) return 0u;
    if (s >= 4294967295.0) return 4294967295u;
    return (uint32_t)s;
#endif
}

// One coordinate -> code bits (u8/u16 value, f32 bits or f64 bits, in a u64).
PCV_HD uint64_t encode1(double value, double mn, double edge, int enc) {
    double t = clamp01((value - mn) / edge);
    if (enc == ENC_U8) return (uint64_t)trunc_u32(255.0 * t);
    if (enc == ENC_U16) return (uint64_t)trunc_u32(65535.0 * t);
    if (enc == ENC_F32) return (uint64_t)f32_to_bits((float)t);
    return f64_to_bits(t);
}

PCV_HD double decode1(uint64_t bits, double mn, double edge, int enc) {
    if (enc == ENC_U8) return fma((double)(uint32_t)bits / 255.0, edge, mn);
    if (enc == ENC_U16) return fma((double)(uint32_t)bits / 65535.0, edge, mn);
    if (enc == ENC_F32) return fma((double)bits_to_f32((uint32_t)bits), edge, mn);
    return fma(bits_to_f64(bits), edge, mn);
}

// ------------------------------------------------------------------------------------------------
// Exact fast paths.  The descent is bound by the FP64 pipe (two IEEE divisions per axis per level),
// so the two divisions are replaced by sequences that are *proven* to return the same correctly
// rounded result, with a guard that falls back to the IEEE operator outside the proven range.
// tests/test_chain_exact.py checks them exhaustively (unit fractions) and on 10^7..10^9 random and
// adversarial operands (division) against the plain operators, on the host and on the GPU.
// ------------------------------------------------------------------------------------------------

// RN(v / (2^k - 1)) for k = 8 or 16 and 0 <= v <= 2^k - 1, built with integer instructions only.
// v/(2^k-1) = 0.(v)(v)(v)... in binary (the k-bit pattern of v repeated for ever), so the 53-bit
// significand is read off the repeated pattern; the discarded tail is periodic and non-zero, hence
// never an exact tie: round up iff the first discarded bit is set.
template <int K>
PCV_HD double unit_frac_int(uint32_t v) {
    const uint32_t M = (1u << K) - 1u;
    if (v == 0u) return 0.0;
    if (v >= M) return 1.0;
    const uint64_t rep = K == 8 ? 0x0101010101010101ull : 0x0001000100010001ull;
    const uint64_t P = (uint64_t)v * rep;  // first 64 fraction bits; the pattern continues with period K | 64
#if defined(__CUDA_ARCH__)
    const int lz = __clzll((long long)P);
#else
    const int lz = __builtin_clzll(P);
#endif
    const uint64_t S = lz ? ((P << lz) | (P >> (64 - lz))) : P;  // rotate == shift in the periodic tail
    const uint64_t mant = (S >> 11) + ((S >> 10) & 1ull);        // 53 bits incl. the leading one (may carry to 2^53)
    // value = 1.f * 2^-(lz+1): biased exponent 1022 - lz; adding `mant` (bit 52 set) bumps the field by one
    return bits_to_f64(((uint64_t)(1021 - lz) << 52) + mant);
}

// Same value with three FP64 instructions: q0 = RN(v*y), q = RN(q0 + (v - q0*M)*y) with y = RN(1/M).  For the two
// divisors that occur (255, 65535) this is verified EXHAUSTIVELY against v / M for every code v (tests/test_chain_exact.py),
// so no proof obligation remains.  int -> f64 is the exact magic-number conversion (no I2F on the XU pipe).
template <int K>
PCV_HD double unit_frac(uint32_t v) {
    const double M = K == 8 ? 255.0 : 65535.0;
    const double y = K == 8 ? (1.0 / 255.0) : (1.0 / 65535.0);
#if defined(__CUDA_ARCH__)
    const double a = __hiloint2double(0x43300000, (int)v) - 4503599627370496.0;
#else
    const double a = (double)v;
#endif
    const double q0 = a * y;
    return fma(fma(-q0, M, a), y, q0);
}

// a / b, correctly rounded, given y = RN(1/b) computed once per divisor on the host.
//   q0 = RN(a*y)                      relative error <= 2^-52
//   q1 = RN(q0 + (a - b*q0)*y)        faithful (error of the correction term ~2^-105)
//   q2 = RN(q1 + (a - b*q1)*y)        = RN(a/b) by Markstein's theorem (y = RN(1/b), q1 faithful, the residuals
//                                     a - b*q are exact in an FMA, significand of b not all ones - checked on the host)
// valid while nothing under/overflows: guarded to 2^-500 < |a| < 2^500 (the host guarantees the same for b);
// everything else (0, tiny, inf, NaN) takes the IEEE operator.
PCV_HD double div_known(double a, double b, double y) {
    const uint32_t hi = (uint32_t)(f64_to_bits(a) >> 32) & 0x7fffffffu;
    if (hi - 0x20b00000u < 0x3e800000u) {  // biased exponent in [523, 1523)
        const double q0 = a * y;
        const double q1 = fma(fma(-q0, b, a), y, q0);
        return fma(fma(-q1, b, a), y, q1);
    }
    return a / b;
}

// Host-side admissibility of a divisor for div_known: normal range with head-room and significand not all ones.
PCV_HD bool div_known_ok(double b) {
    const uint64_t bits = f64_to_bits(b);
    const uint32_t ex = (uint32_t)(bits >> 52) & 0x7ffu;
    const uint64_t frac = bits & 0xFFFFFFFFFFFFFull;
    return b > 0.0 && ex > 523u && ex < 1523u && frac != 0xFFFFFFFFFFFFFull;
}

// encode1 / decode1 with the exact fast paths (ry = RN(1/edge)).  For the integer encodings the clamp is
// dropped: `as u8/u16` saturates and maps NaN to 0, so trunc(MAX * t) capped at MAX equals the clamped form
// for every t (t < 0 -> 0, t > 1 -> MAX, NaN -> 0).
PCV_HD uint64_t encode1_fast(double value, double mn, double edge, double ry, int enc) {
    const double t = div_known(value - mn, edge, ry);
    if (enc == ENC_U8) {
        const uint32_t v = trunc_u32(255.0 * t);
        return v > 255u ? 255u : v;
    }
    if (enc == ENC_U16) {
        const uint32_t v = trunc_u32(65535.0 * t);
        return v > 65535u ? 65535u : v;
    }
    const double c = clamp01(t);
    if (enc == ENC_F32) return (uint64_t)f32_to_bits((float)c);
    return f64_to_bits(c);
}
PCV_HD double decode1_fast(uint64_t bits, double mn, double edge, int enc) {
    if (enc == ENC_U8) return fma(unit_frac<8>((uint32_t)bits), edge, mn);
    if (enc == ENC_U16) return fma(unit_frac<16>((uint32_t)bits), edge, mn);
    if (enc == ENC_F32) return fma((double)bits_to_f32((uint32_t)bits), edge, mn);
    return fma(bits_to_f64(bits), edge, mn);
}

// Per-level constants, computed once on the host exactly like the reference does per node:
// edge[L] by repeated `/= 2` from the root edge (node.rs:161), enc[L] = PositionEncoding::new
// (codec.rs:31-40, log2 evaluated on the host only).
struct LevelTable {
    double edge[kMaxLevels];
    double ry[kMaxLevels];  // RN(1 / edge[L]) for div_known
    int8_t enc[kMaxLevels];
    int32_t last_level;  // deepest level a node can have (nodes there are never split)
    int32_t fast;        // 1 if every edge is admissible for the exact fast paths (div_known_ok)
};

// One descent step: point at decoded position q inside the cube (m, e_cur) of a node at level L.
// Computes the child digit, advances m to the child's min, encodes q into the child cube and
// replaces q by the decoded value — i.e. exactly what the child's node file would hand to the next
// split (generation.rs:78-101 then raw.rs:127-216).
struct Step {
    uint64_t code[3];
    unsigned digit;
};
PCV_HD Step descend(double q[3], double m[3], double e_cur, double e_half, int enc_child) {
    Step s;
    unsigned d = 0;
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (int a = 0; a < 3; ++a) {
        double c = (m[a] + (m[a] + e_cur)) / 2.0;  // Cube::center
        unsigned bit = q[a] > c ? 1u : 0u;
        d = (d << 1) | bit;
        if (bit) m[a] = m[a] + e_half;  // min += 1.0 * edge (bit 0 adds 0.0: unchanged)
        uint64_t code = encode1(q[a], m[a], e_half, enc_child);
        s.code[a] = code;
        q[a] = decode1(code, m[a], e_half, enc_child);
    }
    s.digit = d;  // (x>cx)<<2 | (y>cy)<<1 | (z>cz)
    return s;
}

// Same step through the exact fast paths (identical results, ~2.5x fewer FP64-pipe instructions).
PCV_HD Step descend_fast(double q[3], double m[3], double e_cur, double e_half, double ry_half, int enc_child) {
    Step s;
    unsigned d = 0;
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (int a = 0; a < 3; ++a) {
        double c = (m[a] + (m[a] + e_cur)) / 2.0;
        unsigned bit = q[a] > c ? 1u : 0u;
        d = (d << 1) | bit;
        if (bit) m[a] = m[a] + e_half;
        uint64_t code = encode1_fast(q[a], m[a], e_half, ry_half, enc_child);
        s.code[a] = code;
        q[a] = decode1_fast(code, m[a], e_half, enc_child);
    }
    s.digit = d;
    return s;
}

}  // namespace pcv
