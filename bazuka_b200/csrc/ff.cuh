// bazuka_b200 — Montgomery prime-field arithmetic for sm_90a (and a bit-identical host path).
//
// Replaces, on the GPU, what the reference obtains from un-vendored crates:
//   Fr  = `ZkScalar([u64;4])`            /root/reference/src/zk/mod.rs:202-206   (ff 0.13 derive)
//   Fp  = `groth16::Fp([u64;6])`         /root/reference/src/zk/groth16/mod.rs:19-20 (bls12_381 0.8.0)
// Memory image = the reference's: little-endian 64-bit limbs in Montgomery form (R = 2^256 / 2^384),
// always fully reduced, so device results can be memcmp'd against the CPU prover's.
//
// Hopper has no 64-bit integer multiplier; the native wide op is IMAD.WIDE.U32 (32x32+64 with
// carry-in/out predicates).  The product is therefore organised on 32-bit limbs as two interleaved
// accumulators — one holding the 64-bit partial products that start on even columns, one those
// that start on odd columns — so that every 32x32 product is ONE `mad.lo.cc/madc.hi.cc` pair
// (fused by ptxas into one IMAD.WIDE) in a gap-free carry chain, and Montgomery reduction is
// interleaved row by row (CIOS).  ~2N^2+6N integer instructions per N-limb product.
//
// The same algorithm text compiles for the host with an explicit carry variable standing in for
// the PTX condition code; tests run it on the CPU against the oracle, so the carry-chain logic is
// verified without a GPU.
#pragma once
#include <stdint.h>
#include <string.h>

#if defined(__CUDACC__)
#define BZK_HD __host__ __device__ __forceinline__
#define BZK_D __device__ __forceinline__
#else
#define BZK_HD inline
#define BZK_D inline
#endif

#if defined(__CUDACC__)
#define BZK_HD_POW __host__ __device__ __noinline__
#else
#define BZK_HD_POW
#endif

namespace bzk {

// ---------------------------------------------------------------------------------------------
// carry-chain primitives.  Device: PTX condition code (the CC argument is dead).  Host: explicit.
// ---------------------------------------------------------------------------------------------
struct CC {
    uint32_t c;
};

#if defined(__CUDA_ARCH__)
#define BZK_ASM asm volatile
BZK_D uint32_t add_cc(uint32_t a, uint32_t b, CC &) { uint32_t r; BZK_ASM("add.cc.u32 %0,%1,%2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
BZK_D uint32_t addc_cc(uint32_t a, uint32_t b, CC &) { uint32_t r; BZK_ASM("addc.cc.u32 %0,%1,%2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
BZK_D uint32_t addc(uint32_t a, uint32_t b, CC &) { uint32_t r; BZK_ASM("addc.u32 %0,%1,%2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
BZK_D uint32_t sub_cc(uint32_t a, uint32_t b, CC &) { uint32_t r; BZK_ASM("sub.cc.u32 %0,%1,%2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
BZK_D uint32_t subc_cc(uint32_t a, uint32_t b, CC &) { uint32_t r; BZK_ASM("subc.cc.u32 %0,%1,%2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
BZK_D uint32_t subc(uint32_t a, uint32_t b, CC &) { uint32_t r; BZK_ASM("subc.u32 %0,%1,%2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
BZK_D uint32_t mad_lo_cc(uint32_t a, uint32_t b, uint32_t c, CC &) { uint32_t r; BZK_ASM("mad.lo.cc.u32 %0,%1,%2,%3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
BZK_D uint32_t madc_lo_cc(uint32_t a, uint32_t b, uint32_t c, CC &) { uint32_t r; BZK_ASM("madc.lo.cc.u32 %0,%1,%2,%3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
BZK_D uint32_t madc_hi_cc(uint32_t a, uint32_t b, uint32_t c, CC &) { uint32_t r; BZK_ASM("madc.hi.cc.u32 %0,%1,%2,%3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
BZK_D uint32_t mul_lo(uint32_t a, uint32_t b) { return a * b; }
BZK_D uint32_t mul_hi(uint32_t a, uint32_t b) { return __umulhi(a, b); }
// (hi:lo) += a*b with the carry chained through, as ONE asm statement so that ptxas emits a single
// IMAD.WIDE.U32.X per product (as separate statements it splits register-register products into
// IMAD + IMAD.HI + 2 IADD3.X).  Per 384-bit product that is 301 heavy instructions fused (this),
// 433 heavy + 295 IADD3.X split, or 310 heavy + 575 IADD3.X with carry-less IMAD.WIDE: carries,
// not multiplies, dominate the instruction count.  tools/microbench/imad.cu times the three forms.
#ifndef BZK_MUL_WIDE_ADD
BZK_D void mad_pair_first(uint32_t &lo, uint32_t &hi, uint32_t a, uint32_t b, CC &) {
    BZK_ASM("mad.lo.cc.u32 %0,%2,%3,%0; madc.hi.cc.u32 %1,%2,%3,%1;" : "+r"(lo), "+r"(hi) : "r"(a), "r"(b));
}
BZK_D void mad_pair_next(uint32_t &lo, uint32_t &hi, uint32_t a, uint32_t b, CC &) {
    BZK_ASM("madc.lo.cc.u32 %0,%2,%3,%0; madc.hi.cc.u32 %1,%2,%3,%1;" : "+r"(lo), "+r"(hi) : "r"(a), "r"(b));
}
#else  // carry-less IMAD.WIDE.U32 into a temporary + two IADD3.X (microbenchmark comparison only)
BZK_D void mad_pair_first(uint32_t &lo, uint32_t &hi, uint32_t a, uint32_t b, CC &) {
    BZK_ASM("{ .reg .u64 t; .reg .u32 tl, th; mul.wide.u32 t,%2,%3; mov.b64 {tl,th}, t; add.cc.u32 %0,%0,tl; addc.cc.u32 %1,%1,th; }"
            : "+r"(lo), "+r"(hi) : "r"(a), "r"(b));
}
BZK_D void mad_pair_next(uint32_t &lo, uint32_t &hi, uint32_t a, uint32_t b, CC &) {
    BZK_ASM("{ .reg .u64 t; .reg .u32 tl, th; mul.wide.u32 t,%2,%3; mov.b64 {tl,th}, t; addc.cc.u32 %0,%0,tl; addc.cc.u32 %1,%1,th; }"
            : "+r"(lo), "+r"(hi) : "r"(a), "r"(b));
}
#endif
#else
BZK_HD uint32_t add_cc(uint32_t a, uint32_t b, CC &cc) { uint64_t t = (uint64_t)a + b; cc.c = (uint32_t)(t >> 32); return (uint32_t)t; }
BZK_HD uint32_t addc_cc(uint32_t a, uint32_t b, CC &cc) { uint64_t t = (uint64_t)a + b + cc.c; cc.c = (uint32_t)(t >> 32); return (uint32_t)t; }
BZK_HD uint32_t addc(uint32_t a, uint32_t b, CC &cc) { return a + b + cc.c; }
BZK_HD uint32_t sub_cc(uint32_t a, uint32_t b, CC &cc) { uint64_t t = (uint64_t)a - b; cc.c = (uint32_t)(t >> 63); return (uint32_t)t; }
BZK_HD uint32_t subc_cc(uint32_t a, uint32_t b, CC &cc) { uint64_t t = (uint64_t)a - b - cc.c; cc.c = (uint32_t)(t >> 63); return (uint32_t)t; }
BZK_HD uint32_t subc(uint32_t a, uint32_t b, CC &cc) { return a - b - cc.c; }
BZK_HD uint32_t mad_lo_cc(uint32_t a, uint32_t b, uint32_t c, CC &cc) { uint64_t t = (uint64_t)(uint32_t)((uint64_t)a * b) + c; cc.c = (uint32_t)(t >> 32); return (uint32_t)t; }
BZK_HD uint32_t madc_lo_cc(uint32_t a, uint32_t b, uint32_t c, CC &cc) { uint64_t t = (uint64_t)(uint32_t)((uint64_t)a * b) + c + cc.c; cc.c = (uint32_t)(t >> 32); return (uint32_t)t; }
BZK_HD uint32_t madc_hi_cc(uint32_t a, uint32_t b, uint32_t c, CC &cc) { uint64_t t = (((uint64_t)a * b) >> 32) + c + cc.c; cc.c = (uint32_t)(t >> 32); return (uint32_t)t; }
BZK_HD uint32_t mul_lo(uint32_t a, uint32_t b) { return a * b; }
BZK_HD uint32_t mul_hi(uint32_t a, uint32_t b) { return (uint32_t)(((uint64_t)a * b) >> 32); }
BZK_HD void mad_pair_first(uint32_t &lo, uint32_t &hi, uint32_t a, uint32_t b, CC &cc) {
    lo = mad_lo_cc(a, b, lo, cc);
    hi = madc_hi_cc(a, b, hi, cc);
}
BZK_HD void mad_pair_next(uint32_t &lo, uint32_t &hi, uint32_t a, uint32_t b, CC &cc) {
    lo = madc_lo_cc(a, b, lo, cc);
    hi = madc_hi_cc(a, b, hi, cc);
}
#endif

// ---------------------------------------------------------------------------------------------
// Field element: N 32-bit limbs, little-endian (identical bytes to N/2 little-endian u64 limbs).
// P supplies: static constexpr int N; modulus p[N]; inv = -p^-1 mod 2^32; one[N] = R mod p;
//             r2[N] = R^2 mod p   (as functions returning the k-th limb so that they constant-fold)
// ---------------------------------------------------------------------------------------------
template <class P>
struct Fe {
    static constexpr int N = P::N;
    uint32_t l[N];

    BZK_HD static Fe zero() {
        Fe r;
#pragma unroll
        for (int i = 0; i < N; i++) r.l[i] = 0;
        return r;
    }
    BZK_HD static Fe one() {
        Fe r;
#pragma unroll
        for (int i = 0; i < N; i++) r.l[i] = P::one(i);
        return r;
    }
    BZK_HD static Fe r2() {
        Fe r;
#pragma unroll
        for (int i = 0; i < N; i++) r.l[i] = P::r2(i);
        return r;
    }
    BZK_HD bool is_zero() const {
        uint32_t t = 0;
#pragma unroll
        for (int i = 0; i < N; i++) t |= l[i];
        return t == 0;
    }
    BZK_HD bool operator==(const Fe &o) const {
        uint32_t t = 0;
#pragma unroll
        for (int i = 0; i < N; i++) t |= l[i] ^ o.l[i];
        return t == 0;
    }
    BZK_HD bool operator!=(const Fe &o) const { return !(*this == o); }

    // r = a - p if a >= p else a        (a < 2p)
    BZK_HD static Fe reduce_once(const Fe &a) {
        Fe t;
        CC cc{0};
        t.l[0] = sub_cc(a.l[0], P::p(0), cc);
#pragma unroll
        for (int i = 1; i < N; i++) t.l[i] = subc_cc(a.l[i], P::p(i), cc);
        uint32_t borrow = subc(0, 0, cc);  // 0 or 0xffffffff
        Fe r;
#pragma unroll
        for (int i = 0; i < N; i++) r.l[i] = borrow ? a.l[i] : t.l[i];
        return r;
    }
    // BZK_HOST_DEVICE_TEXT (tests only) makes a host build run the device text everywhere, so that sqr, inv, pow and the
    // group law are checked on the CPU through add_limbs32 / sub_limbs32 / mul_evenodd as well
    BZK_HD friend Fe operator+(const Fe &a, const Fe &b) {
#if defined(__CUDA_ARCH__) || defined(BZK_HOST_DEVICE_TEXT)
        return add_limbs32(a, b);
#else
        return add_host64(a, b);
#endif
    }
    BZK_HD friend Fe operator-(const Fe &a, const Fe &b) {
#if defined(__CUDA_ARCH__) || defined(BZK_HOST_DEVICE_TEXT)
        return sub_limbs32(a, b);
#else
        return sub_host64(a, b);
#endif
    }
    // host constants as 64-bit limbs, built once (the constexpr limb tables would otherwise be re-materialised on
    // the stack at every call with a runtime index)
    struct HostConsts {
        uint64_t p[N / 2];
        uint64_t inv64;  // -p^-1 mod 2^64
    };
    static inline const HostConsts &host_consts() {
        static const HostConsts hc = [] {
            HostConsts c;
            for (int i = 0; i < N / 2; i++) c.p[i] = (uint64_t)P::p(2 * i) | ((uint64_t)P::p(2 * i + 1) << 32);
            uint64_t x = (uint64_t)(0u - P::inv());  // p^-1 mod 2^32
            x *= 2 - c.p[0] * x;                      // one Newton step: p^-1 mod 2^64
            c.inv64 = (uint64_t)0 - x;
            return c;
        }();
        return hc;
    }
    // host fast paths on 64-bit limbs (the 32-bit-limb image is the same bytes on a little-endian host)
    static inline Fe add_host64(const Fe &a, const Fe &b) {
        constexpr int M = N / 2;
        uint64_t A[M], B[M], t[M], s[M];
        memcpy(A, a.l, sizeof A);
        memcpy(B, b.l, sizeof B);
        unsigned __int128 c = 0;
        for (int i = 0; i < M; i++) { c += (unsigned __int128)A[i] + B[i]; t[i] = (uint64_t)c; c >>= 64; }
        uint64_t borrow = 0;
        const uint64_t *Pm = host_consts().p;
        for (int i = 0; i < M; i++) {
            const uint64_t pm = Pm[i];
            const unsigned __int128 d = (unsigned __int128)t[i] - pm - borrow;
            s[i] = (uint64_t)d;
            borrow = (uint64_t)(d >> 64) & 1;
        }
        Fe r;
        memcpy(r.l, borrow ? t : s, sizeof t);
        return r;
    }
    static inline Fe sub_host64(const Fe &a, const Fe &b) {
        constexpr int M = N / 2;
        uint64_t A[M], B[M], t[M];
        memcpy(A, a.l, sizeof A);
        memcpy(B, b.l, sizeof B);
        uint64_t borrow = 0;
        for (int i = 0; i < M; i++) {
            const unsigned __int128 d = (unsigned __int128)A[i] - B[i] - borrow;
            t[i] = (uint64_t)d;
            borrow = (uint64_t)(d >> 64) & 1;
        }
        if (borrow) {
            unsigned __int128 c = 0;
            const uint64_t *Pm = host_consts().p;
            for (int i = 0; i < M; i++) {
                const uint64_t pm = Pm[i];
                c += (unsigned __int128)t[i] + pm;
                t[i] = (uint64_t)c;
                c >>= 64;
            }
        }
        Fe r;
        memcpy(r.l, t, sizeof t);
        return r;
    }
    // the device algorithm (32-bit limbs, carry chain); also compiled for the host so tests can check it
    BZK_HD static Fe add_limbs32(const Fe &a, const Fe &b) {
        Fe t;
        CC cc{0};
        t.l[0] = add_cc(a.l[0], b.l[0], cc);
#pragma unroll
        for (int i = 1; i < N; i++) t.l[i] = addc_cc(a.l[i], b.l[i], cc);
        return reduce_once(t);  // both moduli leave a spare top bit: no carry out of limb N-1
    }
    BZK_HD static Fe sub_limbs32(const Fe &a, const Fe &b) {
        Fe t;
        CC cc{0};
        t.l[0] = sub_cc(a.l[0], b.l[0], cc);
#pragma unroll
        for (int i = 1; i < N; i++) t.l[i] = subc_cc(a.l[i], b.l[i], cc);
        uint32_t borrow = subc(0, 0, cc);
        CC c2{0};
        t.l[0] = add_cc(t.l[0], borrow & P::p(0), c2);
#pragma unroll
        for (int i = 1; i < N; i++) t.l[i] = addc_cc(t.l[i], borrow & P::p(i), c2);
        return t;
    }
    BZK_HD Fe neg() const { return zero() - *this; }
    BZK_HD Fe dbl() const { return *this + *this; }

    // Montgomery product a*b/R mod p, fully reduced.  See the header comment for the layout:
    // E holds 64-bit partial products starting on even absolute columns, O those starting on odd
    // columns; row i adds a*b[i] and m_i*p and retires column i.
    BZK_HD friend Fe operator*(const Fe &a, const Fe &b) {
#if defined(__CUDA_ARCH__) && defined(BZK_MUL_NOINLINE)
        return mul_call(a, b);   // one out-of-line copy per translation unit: code-size experiment (instruction cache)
#elif defined(__CUDA_ARCH__) || defined(BZK_HOST_DEVICE_TEXT)
        return mul_evenodd(a, b);
#else
        return mul_host64(a, b);
#endif
    }
#if defined(__CUDACC__)
    __device__ __noinline__ static Fe mul_call(Fe a, Fe b) { return mul_evenodd(a, b); }
#endif
    // host fast path: plain CIOS on 64-bit limbs (unsigned __int128 products); same result
    static inline Fe mul_host64(const Fe &a, const Fe &b) {
        constexpr int M = N / 2;
        uint64_t A[M], B[M], t[M + 2];
        memcpy(A, a.l, sizeof A);
        memcpy(B, b.l, sizeof B);
        const HostConsts &hc = host_consts();
        const uint64_t *Pm = hc.p;
        const uint64_t inv64 = hc.inv64;
        for (int i = 0; i < M + 2; i++) t[i] = 0;
        for (int i = 0; i < M; i++) {
            unsigned __int128 cur;
            uint64_t carry = 0;
            for (int j = 0; j < M; j++) {
                cur = (unsigned __int128)A[j] * B[i] + t[j] + carry;
                t[j] = (uint64_t)cur;
                carry = (uint64_t)(cur >> 64);
            }
            cur = (unsigned __int128)t[M] + carry;
            t[M] = (uint64_t)cur;
            t[M + 1] = (uint64_t)(cur >> 64);
            const uint64_t m = t[0] * inv64;
            cur = (unsigned __int128)m * Pm[0] + t[0];
            carry = (uint64_t)(cur >> 64);
            for (int j = 1; j < M; j++) {
                cur = (unsigned __int128)m * Pm[j] + t[j] + carry;
                t[j - 1] = (uint64_t)cur;
                carry = (uint64_t)(cur >> 64);
            }
            cur = (unsigned __int128)t[M] + carry;
            t[M - 1] = (uint64_t)cur;
            t[M] = t[M + 1] + (uint64_t)(cur >> 64);
        }
        // t < 2p and 2p < 2^(32N): t[M] == 0; one conditional subtraction
        uint64_t s[M], borrow = 0;
        for (int i = 0; i < M; i++) {
            const unsigned __int128 d = (unsigned __int128)t[i] - Pm[i] - borrow;
            s[i] = (uint64_t)d;
            borrow = (uint64_t)(d >> 64) & 1;
        }
        Fe r;
        memcpy(r.l, borrow ? t : s, M * sizeof(uint64_t));
        return r;
    }
    // the device algorithm (also compiled for the host so tests can check its carry logic)
    BZK_HD static Fe mul_evenodd(const Fe &a, const Fe &b) {
        uint32_t E[2 * N + 2], O[2 * N + 2];
#pragma unroll
        for (int i = 0; i < 2 * N + 2; i++) E[i] = O[i] = 0;
        CC cc{0};
#pragma unroll
        for (int i = 0; i < N; i++) {
            uint32_t *Pp = (i & 1) ? O : E;  // pairs start on column i's parity
            uint32_t *Q = (i & 1) ? E : O;
            const uint32_t bi = b.l[i];
            if (i == 0) {
#pragma unroll
                for (int j = 0; j < N; j += 2) {
                    Pp[j] = mul_lo(a.l[j], bi);
                    Pp[j + 1] = mul_hi(a.l[j], bi);
                    Q[j + 1] = mul_lo(a.l[j + 1], bi);
                    Q[j + 2] = mul_hi(a.l[j + 1], bi);
                }
            } else {
                // retire the high half Q[i] of Q's pair (i-1,i) into column i; its carry enters
                // Q's chain at column i+1
                Pp[i] = add_cc(Pp[i], Q[i], cc);
#pragma unroll
                for (int j = 1; j < N; j += 2) mad_pair_next(Q[i + j], Q[i + j + 1], a.l[j], bi, cc);
                Q[i + N + 1] = addc(0, 0, cc);
                mad_pair_first(Pp[i], Pp[i + 1], a.l[0], bi, cc);
#pragma unroll
                for (int j = 2; j < N; j += 2) mad_pair_next(Pp[i + j], Pp[i + j + 1], a.l[j], bi, cc);
                Pp[i + N] = addc(Pp[i + N], 0, cc);
            }
            const uint32_t m = mul_lo(Pp[i], P::inv());
            mad_pair_first(Pp[i], Pp[i + 1], m, P::p(0), cc);
#pragma unroll
            for (int j = 2; j < N; j += 2) mad_pair_next(Pp[i + j], Pp[i + j + 1], m, P::p(j), cc);
            Pp[i + N] = addc(Pp[i + N], 0, cc);
            mad_pair_first(Q[i + 1], Q[i + 2], m, P::p(1), cc);
#pragma unroll
            for (int j = 3; j < N; j += 2) mad_pair_next(Q[i + j], Q[i + j + 1], m, P::p(j), cc);
            Q[i + N + 1] = addc(Q[i + N + 1], 0, cc);
        }
        // columns N .. 2N-1 of E + O  (column 2N is provably zero: the result is < 2p < 2^(32N))
        Fe r;
        r.l[0] = add_cc(E[N], O[N], cc);
#pragma unroll
        for (int k = 1; k < N; k++) r.l[k] = addc_cc(E[N + k], O[N + k], cc);
        return reduce_once(r);
    }
    BZK_HD Fe sqr() const { return (*this) * (*this); }

    // ---- lazy reduction for inner products (Poseidon's MDS rows) --------------------------------
    // out[0..2N) = a*b as a plain 2N-limb integer: the even/odd IMAD.WIDE chains of mul_evenodd without
    // the interleaved reduction rows (half the multiply work of a Montgomery product).
    BZK_HD static void mul_wide(uint32_t out[2 * N], const Fe &a, const Fe &b) {
        uint32_t E[2 * N + 2], O[2 * N + 2];
#pragma unroll
        for (int i = 0; i < 2 * N + 2; i++) E[i] = O[i] = 0;
        CC cc{0};
#pragma unroll
        for (int i = 0; i < N; i++) {
            uint32_t *Pp = (i & 1) ? O : E;
            uint32_t *Q = (i & 1) ? E : O;
            const uint32_t bi = b.l[i];
            if (i == 0) {
#pragma unroll
                for (int j = 0; j < N; j += 2) {
                    Pp[j] = mul_lo(a.l[j], bi);
                    Pp[j + 1] = mul_hi(a.l[j], bi);
                    Q[j + 1] = mul_lo(a.l[j + 1], bi);
                    Q[j + 2] = mul_hi(a.l[j + 1], bi);
                }
            } else {
                mad_pair_first(Q[i + 1], Q[i + 2], a.l[1], bi, cc);
#pragma unroll
                for (int j = 3; j < N; j += 2) mad_pair_next(Q[i + j], Q[i + j + 1], a.l[j], bi, cc);
                Q[i + N + 1] = addc(0, 0, cc);
                mad_pair_first(Pp[i], Pp[i + 1], a.l[0], bi, cc);
#pragma unroll
                for (int j = 2; j < N; j += 2) mad_pair_next(Pp[i + j], Pp[i + j + 1], a.l[j], bi, cc);
                Pp[i + N] = addc(Pp[i + N], 0, cc);
            }
        }
        out[0] = add_cc(E[0], O[0], cc);
#pragma unroll
        for (int k = 1; k < 2 * N; k++) out[k] = addc_cc(E[k], O[k], cc);
    }
    // acc[0..2N] += w[0..2N)   (acc has 2N+1 limbs)
    BZK_HD static void wide_accumulate(uint32_t acc[2 * N + 1], const uint32_t w[2 * N]) {
        CC cc{0};
        acc[0] = add_cc(acc[0], w[0], cc);
#pragma unroll
        for (int k = 1; k < 2 * N; k++) acc[k] = addc_cc(acc[k], w[k], cc);
        acc[2 * N] = addc(acc[2 * N], 0, cc);
    }
    // Montgomery reduction of a (2N+1)-limb value T < p * 2^(32(N+1)) by N+1 limbs:
    // returns T / 2^(32(N+1)) mod p, fully reduced.  Runs once per inner product, so it is written as
    // plain operand scanning with 64-bit carries.
    BZK_HD static Fe redc_wide(const uint32_t T[2 * N + 1]) {
        uint32_t t[2 * N + 2];
#pragma unroll
        for (int k = 0; k < 2 * N + 1; k++) t[k] = T[k];
        t[2 * N + 1] = 0;
#pragma unroll
        for (int i = 0; i < N + 1; i++) {
            const uint32_t m = t[i] * P::inv();
            uint64_t carry = 0;
#pragma unroll
            for (int j = 0; j < N; j++) {
                uint64_t cur = (uint64_t)m * P::p(j) + t[i + j] + carry;
                t[i + j] = (uint32_t)cur;
                carry = cur >> 32;
            }
#pragma unroll
            for (int k = i + N; k < 2 * N + 2; k++) {
                uint64_t cur = (uint64_t)t[k] + carry;
                t[k] = (uint32_t)cur;
                carry = cur >> 32;
            }
        }
        Fe r;
#pragma unroll
        for (int k = 0; k < N; k++) r.l[k] = t[N + 1 + k];
        return reduce_once(r);  // < 2p and t[2N+1] == 0 by the bound on T
    }

    BZK_HD Fe to_mont() const { return (*this) * r2(); }
    BZK_HD Fe from_mont() const {
        Fe o = zero();
        o.l[0] = 1;
        return (*this) * o;
    }
    BZK_HD static Fe from_u32(uint32_t v) {
        Fe o = zero();
        o.l[0] = v;
        return o.to_mont();
    }
    // a^e for a plain little-endian exponent of `nw` 32-bit words (not constant time; not needed)
    BZK_HD_POW Fe pow(const uint32_t *e, int nw) const {
        Fe acc = one();
        for (int i = nw * 32 - 1; i >= 0; i--) {
            acc = acc.sqr();
            if ((e[i >> 5] >> (i & 31)) & 1) acc = acc * (*this);
        }
        return acc;
    }
    // Fermat inverse (0 -> 0)
    BZK_HD Fe inv() const {
        uint32_t e[N];
#pragma unroll
        for (int i = 0; i < N; i++) e[i] = P::p(i);
        // e = p - 2 with borrow propagation (r's low 32-bit limb is 1)
        uint32_t borrow = 2;
        for (int i = 0; i < N && borrow; i++) {
            uint32_t before = e[i];
            e[i] = before - borrow;
            borrow = before < borrow ? 1 : 0;
        }
        return pow(e, N);
    }
    // Inverse by the binary extended Euclid (0 -> 0): ~1.4*bits halvings and ~0.7*bits subtractions on N-limb integers,
    // no multiplications until the two that restore the Montgomery form.  For a LONE thread (the witness interpreter's
    // EdDSA ladders: one dependent affine addition after another) it is several times shorter than the 380 dependent
    // products of the Fermat power; the throughput kernels batch their inversions and keep inv().
    // Invariants: x1 * a = u, x2 * a = v (mod p); u, v odd after the halving loops; ends at u == 1 or v == 1.
    BZK_HD_POW Fe inv_gcd() const {
        if (is_zero()) return zero();
        uint32_t u[N], v[N], x1[N], x2[N];
#pragma unroll
        for (int i = 0; i < N; i++) { u[i] = l[i]; v[i] = P::p(i); x1[i] = 0; x2[i] = 0; }
        x1[0] = 1;
        auto is_one = [](const uint32_t *a) {
            uint32_t t = a[0] ^ 1u;
#pragma unroll
            for (int i = 1; i < N; i++) t |= a[i];
            return t == 0;
        };
        // a >>= 1 ; x = x / 2 mod p
        auto halve = [](uint32_t *a, uint32_t *x) {
#pragma unroll
            for (int i = 0; i < N - 1; i++) a[i] = (a[i] >> 1) | (a[i + 1] << 31);
            a[N - 1] >>= 1;
            uint32_t top = 0;
            if (x[0] & 1u) {
                CC cc{0};
                x[0] = add_cc(x[0], P::p(0), cc);
#pragma unroll
                for (int i = 1; i < N; i++) x[i] = addc_cc(x[i], P::p(i), cc);
                top = addc(0, 0, cc);
            }
#pragma unroll
            for (int i = 0; i < N - 1; i++) x[i] = (x[i] >> 1) | (x[i + 1] << 31);
            x[N - 1] = (x[N - 1] >> 1) | (top << 31);
        };
        // x -= y mod p   (x, y < p)
        auto sub_mod = [](uint32_t *x, const uint32_t *y) {
            CC cc{0};
            x[0] = sub_cc(x[0], y[0], cc);
#pragma unroll
            for (int i = 1; i < N; i++) x[i] = subc_cc(x[i], y[i], cc);
            if (subc(0, 0, cc)) {
                CC c2{0};
                x[0] = add_cc(x[0], P::p(0), c2);
#pragma unroll
                for (int i = 1; i < N - 1; i++) x[i] = addc_cc(x[i], P::p(i), c2);
                x[N - 1] = addc(x[N - 1], P::p(N - 1), c2);
            }
        };
        while (!is_one(u) && !is_one(v)) {
            while (!(u[0] & 1u)) halve(u, x1);
            while (!(v[0] & 1u)) halve(v, x2);
            uint32_t d[N];
            CC cc{0};
            d[0] = sub_cc(u[0], v[0], cc);
#pragma unroll
            for (int i = 1; i < N; i++) d[i] = subc_cc(u[i], v[i], cc);
            if (!subc(0, 0, cc)) {  // u >= v
#pragma unroll
                for (int i = 0; i < N; i++) u[i] = d[i];
                sub_mod(x1, x2);
            } else {
                CC c2{0};
                v[0] = sub_cc(v[0], u[0], c2);
#pragma unroll
                for (int i = 1; i < N - 1; i++) v[i] = subc_cc(v[i], u[i], c2);
                v[N - 1] = subc(v[N - 1], u[N - 1], c2);
                sub_mod(x2, x1);
            }
        }
        Fe r;
        const bool first = is_one(u);
#pragma unroll
        for (int i = 0; i < N; i++) r.l[i] = first ? x1[i] : x2[i];
        // r = (aR)^-1 = a^-1 R^-1  ->  a^-1 R
        const Fe rr = r2();
        return (r * rr) * rr;
    }
};

// ---------------------------------------------------------------------------------------------
// BLS12-381 parameter packs.  Limbs as constexpr switch tables so that they fold to immediates.
// (p, R, R^2 and inv are checked against big-integer arithmetic in tests/test_arith_edges_cpu.py.)
// ---------------------------------------------------------------------------------------------
#define BZK_TABLE(name, ...)                                   \
    BZK_HD static constexpr uint32_t name(int i) {             \
        constexpr uint32_t t[] = {__VA_ARGS__};                \
        return t[i];                                           \
    }

struct FrParams {  // r = 0x73eda753299d7d483339d80809a1d80553bda402fffe5bfeffffffff00000001
    static constexpr int N = 8;
    BZK_TABLE(p, 0x00000001u, 0xffffffffu, 0xfffe5bfeu, 0x53bda402u, 0x09a1d805u, 0x3339d808u, 0x299d7d48u, 0x73eda753u)
    BZK_TABLE(one, 0xfffffffeu, 0x00000001u, 0x00034802u, 0x5884b7fau, 0xecbc4ff5u, 0x998c4fefu, 0xacc5056fu, 0x1824b159u)
    BZK_TABLE(r2, 0xf3f29c6du, 0xc999e990u, 0x87925c23u, 0x2b6cedcbu, 0x7254398fu, 0x05d31496u, 0x9f59ff11u, 0x0748d9d9u)
    BZK_HD static constexpr uint32_t inv() { return 0xffffffffu; }
};

struct FpParams {  // p = 0x1a0111ea...ffffaaab
    static constexpr int N = 12;
    BZK_TABLE(p, 0xffffaaabu, 0xb9feffffu, 0xb153ffffu, 0x1eabfffeu, 0xf6b0f624u, 0x6730d2a0u, 0xf38512bfu, 0x64774b84u,
              0x434bacd7u, 0x4b1ba7b6u, 0x397fe69au, 0x1a0111eau)
    BZK_TABLE(one, 0x0002fffdu, 0x76090000u, 0xc40c0002u, 0xebf4000bu, 0x53c758bau, 0x5f489857u, 0x70525745u, 0x77ce5853u,
              0xa256ec6du, 0x5c071a97u, 0xfa80e493u, 0x15f65ec3u)
    BZK_TABLE(r2, 0x1c341746u, 0xf4df1f34u, 0x09d104f1u, 0x0a76e6a6u, 0x4c95b6d5u, 0x8de5476cu, 0x939d83c0u, 0x67eb88a9u,
              0xb519952du, 0x9a793e85u, 0x92cae3aau, 0x11988fe5u)
    BZK_HD static constexpr uint32_t inv() { return 0xfffcfffdu; }
};

typedef Fe<FrParams> Fr;
typedef Fe<FpParams> Fp;

}  // namespace bzk
