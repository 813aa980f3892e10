// bazuka_b200 — one point of bellman's `Parameters` file: the uncompressed encodings of bls12_381 0.8 and the
// prime-order subgroup tests (device + host; see params_io.cu for the file layout and the pipeline around them).
//
//   G1 = 96 bytes:  x | y, each 48 bytes big-endian canonical (not Montgomery)
//   G2 = 192 bytes: x.c1 | x.c0 | y.c1 | y.c0
//   byte 0 carries the flags: bit 7 compression (must be 0), bit 6 infinity, bit 5 sort (must be 0); x is read with
//   them masked off.  The identity is the infinity bit alone, every other bit zero.
//
// `from_uncompressed_unchecked` refuses bad flags, a coordinate >= p and an infinity bit with coordinate bits set;
// `from_uncompressed` also requires the curve equation and membership of the prime-order subgroup.  The subgroup
// tests are the endomorphism tests bls12_381 0.8 uses (eprint 2021/1130, correctness 2022/352):
//   G1: sigma(P) = (beta x, y) == -[x^2] P          G2: psi(P) == [x] P          x = -0xd201000000010000
// with beta a primitive cube root of unity and psi = untwist-Frobenius-twist; the constants are derived from their
// definitions (derive_endo_consts, run once per process) and the CPU tier holds these tests to the definition [r]P = O
// of the oracle (oracle/py/bellman_params.py) on this header compiled for the host.
#pragma once
#include "ec.cuh"

namespace bzk {

// why a point was refused; ordered as the decoder tests them
enum PointFault : uint32_t {
    kPointOk = 0,
    kCompressionFlag = 1,
    kSortFlag = 2,
    kXNotCanonical = 3,
    kYNotCanonical = 4,
    kInfinityWithBits = 5,
    kPointAtInfinity = 6,
    kNotOnCurve = 7,
    kNotInSubgroup = 8,
};

struct EndoConsts {
    Fp beta;          // sigma(x, y) = (beta x, y) acts on G1 as [-x^2]
    Fp2 psi_x, psi_y; // psi(x, y) = (conj(x) psi_x, conj(y) psi_y) acts on G2 as [x]
};

BZK_HD uint32_t bswap32(uint32_t v) {
#if defined(__CUDA_ARCH__)
    return __byte_perm(v, 0, 0x0123);
#else
    return __builtin_bswap32(v);
#endif
}

// 48 big-endian bytes, read as 12 little-endian words -> canonical limbs (and back)
BZK_HD Fp fp_from_be_words(const uint32_t *w) {
    Fp r;
#pragma unroll
    for (int i = 0; i < 12; i++) r.l[11 - i] = bswap32(w[i]);
    return r;
}
BZK_HD void fp_to_be_words(const Fp &v, uint32_t *w) {
#pragma unroll
    for (int i = 0; i < 12; i++) w[i] = bswap32(v.l[11 - i]);
}

// [|x|] q, |x| = 0xd201000000010000: 63 doublings and 5 additions
template <class F>
BZK_HD Xyzz<F> mul_by_abs_x(const Xyzz<F> &q) {
    constexpr uint64_t kAbsX = 0xd201000000010000ull;
    Xyzz<F> acc = q;
    for (int i = 62; i >= 0; i--) {
        acc = acc.dbl();
        if ((kAbsX >> i) & 1) acc.add(q);
    }
    return acc;
}

// a == (x, y) for an affine point that is not the identity
template <class F>
BZK_HD bool xyzz_equals(const Xyzz<F> &a, const F &x, const F &y) {
    return !a.is_inf() && a.X == x * a.ZZ && a.Y == y * a.ZZZ;
}

// -[x^2] P == sigma(P)  <=>  [|x|]([|x|] P) == (beta x, -y)
BZK_HD bool torsion_free(const G1Affine &p, const EndoConsts &k) {
    if (p.is_inf()) return true;
    const G1Xyzz q = mul_by_abs_x(mul_by_abs_x(G1Xyzz::from_affine(p)));
    return xyzz_equals(q, k.beta * p.x, p.y.neg());
}
// psi(P) == [x] P = -[|x|] P  <=>  [|x|] P == -psi(P)
BZK_HD bool torsion_free(const G2Affine &p, const EndoConsts &k) {
    if (p.is_inf()) return true;
    const G2Xyzz q = mul_by_abs_x(G2Xyzz::from_affine(p));
    const Fp2 cx{p.x.c0, p.x.c1.neg()}, cy{p.y.c0, p.y.c1.neg()};
    return xyzz_equals(q, cx * k.psi_x, (cy * k.psi_y).neg());
}

// ---- host: the constants from their definitions, checked on the generators and on the 3-torsion point (0, 2) -------
inline void exponent_div(uint32_t d, uint32_t e[12]) {  // e = (p - 1) / d
    uint64_t rem = 0;
    for (int i = 11; i >= 0; i--) {
        const uint64_t cur = (rem << 32) | (FpParams::p(i) - (i == 0 ? 1u : 0u));
        e[i] = (uint32_t)(cur / d);
        rem = cur % d;
    }
}
inline Fp2 fp2_pow(const Fp2 &a, const uint32_t e[12]) {
    Fp2 acc = Fp2::one();
    for (int i = 383; i >= 0; i--) {
        acc = acc.sqr();
        if ((e[i >> 5] >> (i & 31)) & 1) acc = acc * a;
    }
    return acc;
}
inline bool derive_endo_consts(EndoConsts *c) {
    uint32_t e3[12], e2[12];
    exponent_div(3, e3);
    exponent_div(2, e2);
    // beta: the primitive cube root of unity for which sigma acts as [-x^2] on G1 (the other one acts as [x^2 - 1])
    Fp w = Fp::one();
    for (uint32_t g = 2; w == Fp::one(); g++) w = Fp::from_u32(g).pow(e3, 12);
    const G1Affine g1 = g1_generator();
    c->beta = w;
    if (!torsion_free(g1, *c)) c->beta = w.sqr();
    // psi = untwist-Frobenius-twist: conj(x) / (u+1)^((p-1)/3), conj(y) / (u+1)^((p-1)/2)
    const Fp2 xi{Fp::one(), Fp::one()};
    c->psi_x = fp2_pow(xi, e3).inv();
    c->psi_y = fp2_pow(xi, e2).inv();
    const G1Affine t3{Fp::zero(), Fp::from_u32(2)};
    G1Xyzz gt = G1Xyzz::from_affine(g1);
    gt.madd(t3);
    return torsion_free(g1, *c) && torsion_free(g2_generator(), *c) && !torsion_free(t3, *c) && !torsion_free(gt.to_affine(), *c);
}

// One encoded point -> Montgomery affine (identity = x = y = 0).  w: the image as little-endian words (24 for G1, 48 for
// G2).  checked: curve + subgroup; allow_inf: the identity is accepted (the verifying key's single points).
BZK_HD uint32_t decode_point(const uint32_t *w, bool checked, bool allow_inf, const EndoConsts &k, G1Affine &p) {
    const uint32_t flags = w[0] & 0xffu;  // byte 0 of the image
    Fp x = fp_from_be_words(w), y = fp_from_be_words(w + 12);
    x.l[11] &= 0x1fffffffu;
    if (flags & 0x80u) return kCompressionFlag;
    if (flags & 0x20u) return kSortFlag;
    if (Fp::reduce_once(x) != x) return kXNotCanonical;
    if (Fp::reduce_once(y) != y) return kYNotCanonical;
    if (flags & 0x40u) {
        if (!x.is_zero() || !y.is_zero()) return kInfinityWithBits;
        if (!allow_inf) return kPointAtInfinity;
        p = G1Affine::inf();
        return kPointOk;
    }
    p = G1Affine{x.to_mont(), y.to_mont()};
    if (!checked) return kPointOk;
    if (!on_curve(p)) return kNotOnCurve;
    if (!torsion_free(p, k)) return kNotInSubgroup;
    return kPointOk;
}
BZK_HD uint32_t decode_point(const uint32_t *w, bool checked, bool allow_inf, const EndoConsts &k, G2Affine &p) {
    const uint32_t flags = w[0] & 0xffu;
    Fp x1 = fp_from_be_words(w), x0 = fp_from_be_words(w + 12), y1 = fp_from_be_words(w + 24), y0 = fp_from_be_words(w + 36);
    x1.l[11] &= 0x1fffffffu;
    if (flags & 0x80u) return kCompressionFlag;
    if (flags & 0x20u) return kSortFlag;
    if (Fp::reduce_once(x1) != x1 || Fp::reduce_once(x0) != x0) return kXNotCanonical;
    if (Fp::reduce_once(y1) != y1 || Fp::reduce_once(y0) != y0) return kYNotCanonical;
    if (flags & 0x40u) {
        if (!x1.is_zero() || !x0.is_zero() || !y1.is_zero() || !y0.is_zero()) return kInfinityWithBits;
        if (!allow_inf) return kPointAtInfinity;
        p = G2Affine::inf();
        return kPointOk;
    }
    p = G2Affine{Fp2{x0.to_mont(), x1.to_mont()}, Fp2{y0.to_mont(), y1.to_mont()}};
    if (!checked) return kPointOk;
    if (!on_curve(p)) return kNotOnCurve;
    if (!torsion_free(p, k)) return kNotInSubgroup;
    return kPointOk;
}

// Montgomery affine -> `to_uncompressed` (the identity: the infinity bit alone)
BZK_HD void encode_point(const G1Affine &p, uint32_t *w) {
    if (p.is_inf()) {
#pragma unroll
        for (int i = 0; i < 24; i++) w[i] = 0;
        w[0] = 0x40u;
        return;
    }
    fp_to_be_words(p.x.from_mont(), w);
    fp_to_be_words(p.y.from_mont(), w + 12);
}
BZK_HD void encode_point(const G2Affine &p, uint32_t *w) {
    if (p.is_inf()) {
#pragma unroll
        for (int i = 0; i < 48; i++) w[i] = 0;
        w[0] = 0x40u;
        return;
    }
    fp_to_be_words(p.x.c1.from_mont(), w);
    fp_to_be_words(p.x.c0.from_mont(), w + 12);
    fp_to_be_words(p.y.c1.from_mont(), w + 24);
    fp_to_be_words(p.y.c0.from_mont(), w + 36);
}

}  // namespace bzk
