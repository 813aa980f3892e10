// bazuka_b200 — carry-free ("unsaturated limb") Fp for the MSM inner loops on sm_90a.
//
// Why: the carry forms of the integer multiply (IMAD.WIDE.U32.X, carry-in/out IADD3.X) cost more
// issue slots than plain IMAD-class instructions — imad.cu times them, ff.cuh counts them per
// product.  A saturated 12 x 32-bit Montgomery
// product needs a carry on every one of its 288 partial products.  With 13 limbs of 30 bits the
// partial products are < 2^60, so a 64-bit column accumulator absorbs 14 of them without any carry:
// the product becomes 338 plain IMAD.WIDE.U32 (t[j] += a[j]*b[i]) + 13 IMAD, carries are handled by
// a handful of shifts/masks on the otherwise idle ALU pipe.
//
// Representation: value v < p as limbs l[0..12], each < 2^30, in Montgomery form with radix
// R' = 2^390 (NOT the wire format's 2^384).  Conversion to/from the wire image `Fp` (ff.cuh) costs
// one product each way and happens once per resident base (at upload) and once per result.
// All functions are plain C (no PTX), identical on host and device; tests/test_abi.py checks the host
// build against the oracle.
#pragma once
#include "ff.cuh"

namespace bzk {

struct FpU {
    static constexpr int N = 13;
    static constexpr uint32_t W = 30;
    static constexpr uint32_t M = (1u << 30) - 1;
    uint32_t l[N];

    BZK_TABLE(p, 0x3fffaaabu, 0x27fbffffu, 0x153ffffbu, 0x2affffacu, 0x30f6241eu, 0x034a83dau, 0x112bf673u, 0x12e13ce1u,
              0x2cd76477u, 0x1ed90d2eu, 0x29a4b1bau, 0x3a8e5ff9u, 0x001a0111u)
    BZK_TABLE(onel, 0x00d1ff2eu, 0x19d80000u, 0x34800ac4u, 0x2e00cde6u, 0x02431c84u, 0x269f83a2u, 0x3dcf80ddu, 0x09b42da0u,
              0x25eec26cu, 0x15d98f12u, 0x04b29f14u, 0x259fcfa0u, 0x00015de9u)
    // 2^396 mod p and 2^384 mod p as plain 30-bit-limb integers: Montgomery factors for the domain change
    BZK_TABLE(to_u, 0x3480cb7fu, 0x3e0c0000u, 0x2042b126u, 0x3f337aafu, 0x3de4b4d1u, 0x1e015cf1u, 0x005c540du, 0x3467b19au,
              0x352a6da3u, 0x19d89d19u, 0x2fb9afe6u, 0x3848c817u, 0x0009772fu)
    BZK_TABLE(from_u, 0x0002fffdu, 0x18240000u, 0x00c00027u, 0x3d0002f1u, 0x0758baebu, 0x22615d4fu, 0x257455f4u, 0x1614dc14u,
              0x2c6d77ceu, 0x2a5e895bu, 0x0935c071u, 0x30fea039u, 0x0015f65eu)
    BZK_HD static constexpr uint32_t inv() { return 0x3ffcfffdu; }  // -p^-1 mod 2^30

    BZK_HD static FpU zero() {
        FpU r;
#pragma unroll
        for (int i = 0; i < N; i++) r.l[i] = 0;
        return r;
    }
    BZK_HD static FpU one() {
        FpU r;
#pragma unroll
        for (int i = 0; i < N; i++) r.l[i] = onel(i);
        return r;
    }
    BZK_HD bool is_zero() const {
        uint32_t t = 0;
#pragma unroll
        for (int i = 0; i < N; i++) t |= l[i];
        return t == 0;
    }
    BZK_HD bool operator==(const FpU &o) const {
        uint32_t t = 0;
#pragma unroll
        for (int i = 0; i < N; i++) t |= l[i] ^ o.l[i];
        return t == 0;
    }
    BZK_HD bool operator!=(const FpU &o) const { return !(*this == o); }

    // v (limbs < 2^31, value < 2p) -> v mod p, normalised
    BZK_HD static FpU reduce_norm(const uint32_t s[N]) {
        FpU a, d;
        int32_t c = 0, bw = 0;
#pragma unroll
        for (int j = 0; j < N; j++) {
            int32_t v = (int32_t)s[j] + c;            // < 2^31 + 1: fits (s[j] < 2^31 - 1)
            a.l[j] = (uint32_t)v & M;
            c = v >> 30;
            int32_t e = (int32_t)a.l[j] - (int32_t)p(j) + bw;
            d.l[j] = (uint32_t)e & M;
            bw = e >> 30;                              // 0 or -1 (arithmetic)
        }
        // value >= p  <=>  no final borrow (the carry c out of the top limb is zero: v < 2p < 2^390)
        FpU r;
#pragma unroll
        for (int j = 0; j < N; j++) r.l[j] = bw ? a.l[j] : d.l[j];
        return r;
    }
    BZK_HD friend FpU operator+(const FpU &a, const FpU &b) {
        uint32_t s[N];
#pragma unroll
        for (int j = 0; j < N; j++) s[j] = a.l[j] + b.l[j];
        return reduce_norm(s);
    }
    BZK_HD friend FpU operator-(const FpU &a, const FpU &b) {
        // a - b + p, limb-wise (each limb in (-2^30, 2^31)), then one normalising reduction
        FpU t, u;
        int32_t c = 0, c2 = 0;
#pragma unroll
        for (int j = 0; j < N; j++) {
            int32_t v = (int32_t)a.l[j] - (int32_t)b.l[j] + c;
            t.l[j] = (uint32_t)v & M;
            c = v >> 30;
            int32_t w2 = (int32_t)t.l[j] + (int32_t)p(j) + c2;
            u.l[j] = (uint32_t)w2 & M;
            c2 = w2 >> 30;
        }
        FpU r;
#pragma unroll
        for (int j = 0; j < N; j++) r.l[j] = c ? u.l[j] : t.l[j];  // c == -1: a < b, take a - b + p
        return r;
    }
    BZK_HD FpU neg() const { return zero() - *this; }
    BZK_HD FpU dbl() const { return *this + *this; }

    // Montgomery product a*b/2^390 mod p, normalised and fully reduced.
    BZK_HD friend FpU operator*(const FpU &a, const FpU &b) {
        uint64_t t[N];
#pragma unroll
        for (int j = 0; j < N; j++) t[j] = 0;
#pragma unroll
        for (int i = 0; i < N; i++) {
            const uint32_t bi = b.l[i];
#pragma unroll
            for (int j = 0; j < N; j++) t[j] += (uint64_t)a.l[j] * bi;
            const uint32_t m = ((uint32_t)t[0] * inv()) & M;
#pragma unroll
            for (int j = 0; j < N; j++) t[j] += (uint64_t)m * p(j);
            const uint64_t carry = t[0] >> W;  // t[0] is now divisible by 2^30
#pragma unroll
            for (int j = 0; j < N - 1; j++) t[j] = t[j + 1];
            t[N - 1] = 0;
            t[0] += carry;
            if (i == 6) {  // keep every column below 2^64: <= 7 rows of 2 products (< 2^60 each) between normalisations
#pragma unroll
                for (int j = 0; j < N - 1; j++) {
                    t[j + 1] += t[j] >> W;
                    t[j] &= M;
                }
            }
        }
        uint32_t s[N];
        uint64_t c = 0;
#pragma unroll
        for (int j = 0; j < N; j++) {
            uint64_t v = t[j] + c;
            s[j] = (uint32_t)v & M;
            c = v >> W;
        }
        return reduce_norm(s);  // value < 2p
    }
    BZK_HD FpU sqr() const { return (*this) * (*this); }

    // wire image (12 x 32-bit saturated limbs, Montgomery radix 2^384) <-> internal
    BZK_HD static FpU from_fp(const Fp &x) {
        FpU r;
#pragma unroll
        for (int j = 0; j < N; j++) {
            const int bit = 30 * j, w = bit >> 5, sh = bit & 31;
            uint64_t two = x.l[w];
            if (w + 1 < 12) two |= (uint64_t)x.l[w + 1] << 32;
            r.l[j] = (uint32_t)(two >> sh) & M;
        }
        FpU c;
#pragma unroll
        for (int j = 0; j < N; j++) c.l[j] = to_u(j);
        return r * c;  // x*2^384 * 2^396 / 2^390 = x * 2^390
    }
    BZK_HD Fp to_fp() const {
        FpU c;
#pragma unroll
        for (int j = 0; j < N; j++) c.l[j] = from_u(j);
        const FpU v = (*this) * c;  // x*2^390 * 2^384 / 2^390 = x * 2^384, as a plain integer < p
        Fp r;
#pragma unroll
        for (int k = 0; k < 12; k++) {
            // bits [32k, 32k+32) of the 30-bit-limb integer
            const int bit = 32 * k, j = bit / 30, sh = bit % 30;
            uint64_t acc = (uint64_t)v.l[j] >> sh;
            if (j + 1 < N) acc |= (uint64_t)v.l[j + 1] << (30 - sh);
            if (j + 2 < N) acc |= (uint64_t)v.l[j + 2] << (60 - sh);
            r.l[k] = (uint32_t)acc;
        }
        return r;
    }
};

}  // namespace bzk
