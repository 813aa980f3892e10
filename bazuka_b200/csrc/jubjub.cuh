// bazuka_b200 — JubJub (twisted Edwards, a = -1, over BLS12-381 Fr) and the EdDSA-Poseidon check, as BZK_HD code shared by
// the batch kernels (jubjub.cu), the host calls (mpn_host.cu: bzk_jubjub_eddsa_verify, bzk_jubjub_decompress, the withdraw
// builder) and the CPU test shim (tests/hostshim/jubjub_shim.cpp).
//
// The reference (src/crypto/jubjub/curve.rs) adds projective points with special cases for its zero encoding and for equal
// points.  On JubJub a = -1 is a square and d is not, so the unified addition of Hisil, Wong, Carter and Dawson (2008) in
// extended coordinates is complete: one branch-free formula gives the same group element for every pair of curve points, and
// so does the dedicated doubling.  Scalars are used as full 256-bit integers (no reduction modulo the prime order, no cofactor
// clearing), as `PointAffine::multiply` uses them: the verdict on points with small-order components depends on that.
#pragma once
#include <vector>

#include "ff.cuh"

namespace bzk {

// y^2 - x^2 == 1 + d x^2 y^2  (`PointAffine::is_on_curve`, curve.rs:40-47)
BZK_HD bool jj_on_curve(const Fr &x, const Fr &y, const Fr &d) {
    Fr x2 = x.sqr(), y2 = y.sqr();
    return (y2 - x2) == (Fr::one() + d * x2 * y2);
}

// The group law below is written once over the field F of any twisted Edwards curve with a = -1 and a non-square d, where it
// is complete: JubJub (F = Fr) here, Ed25519 (F = Fe<P25519Params>) in ed25519.cuh.
// extended coordinates: x = X/Z, y = Y/Z, xy = T/Z (Z never vanishes on the curve: the formulas below are complete)
template <class F> struct EdExt { F x, y, t, z; };
// an addend in the form the addition consumes: (Y - X, Y + X, 2d T, 2Z)
template <class F> struct EdCached { F ymx, ypx, t2d, z2; };
// an affine addend (Z = 1): (y - x, y + x, 2d x y) — the fixed-base tables' entries
template <class F> struct EdNiels { F ymx, ypx, t2d; };
using JJ = EdExt<Fr>;
using JJCached = EdCached<Fr>;
using JJNiels = EdNiels<Fr>;

template <class F> BZK_HD EdExt<F> jj_identity() { return EdExt<F>{F::zero(), F::one(), F::zero(), F::one()}; }
template <class F> BZK_HD EdExt<F> jj_from_affine(const F &x, const F &y) { return EdExt<F>{x, y, x * y, F::one()}; }
template <class F> BZK_HD EdCached<F> jj_cached(const EdExt<F> &p, const F &d2) { return EdCached<F>{p.y - p.x, p.y + p.x, p.t * d2, p.z.dbl()}; }

// unified addition, a = -1 ("add-2008-hwcd-3"): 9 products
template <class F> BZK_HD EdExt<F> jj_add(const EdExt<F> &p, const EdCached<F> &q) {
    const F a = (p.y - p.x) * q.ymx, b = (p.y + p.x) * q.ypx, c = p.t * q.t2d, d = p.z * q.z2;
    const F e = b - a, f = d - c, g = d + c, h = b + a;
    return EdExt<F>{e * f, g * h, e * h, f * g};
}
// the same with Z2 = 1: 7 products
template <class F> BZK_HD EdExt<F> jj_add(const EdExt<F> &p, const EdNiels<F> &q) {
    const F a = (p.y - p.x) * q.ymx, b = (p.y + p.x) * q.ypx, c = p.t * q.t2d, d = p.z.dbl();
    const F e = b - a, f = d - c, g = d + c, h = b + a;
    return EdExt<F>{e * f, g * h, e * h, f * g};
}
// doubling, a = -1 ("dbl-2008-hwcd"): 8 products
template <class F> BZK_HD EdExt<F> jj_dbl(const EdExt<F> &p) {
    const F a = p.x.sqr(), b = p.y.sqr(), c = p.z.sqr().dbl();
    const F e = (p.x + p.y).sqr() - a - b, g = b - a, f = g - c, h = (a + b).neg();
    return EdExt<F>{e * f, g * h, e * h, f * g};
}
// the same group element (projective equality of X/Z and Y/Z)
template <class F> BZK_HD bool jj_equal(const EdExt<F> &p, const EdExt<F> &q) { return p.x * q.z == q.x * p.z && p.y * q.z == q.y * p.z; }

// [k] P for a plain 256-bit little-endian k (any k: no reduction; K is any 8-limb Fe, only its limbs are read), 4-bit unsigned
// windows MSB first: 256 doublings and 64 additions of a per-call table of [0..15] P
template <class F, class K> BZK_HD EdExt<F> jj_mul(const EdExt<F> &p, const K &k, const F &d2) {
    EdCached<F> tab[16];
    tab[0] = jj_cached(jj_identity<F>(), d2);
    tab[1] = jj_cached(p, d2);
    EdExt<F> cur = p;
#pragma unroll 1
    for (int i = 2; i < 16; i++) {
        cur = jj_add(cur, tab[1]);
        tab[i] = jj_cached(cur, d2);
    }
    EdExt<F> acc = jj_identity<F>();
#pragma unroll 1
    for (int w = 63; w >= 0; w--) {
        acc = jj_dbl(jj_dbl(jj_dbl(jj_dbl(acc))));
        acc = jj_add(acc, tab[(k.l[w >> 3] >> (4 * (w & 7))) & 15u]);
    }
    return acc;
}

// A fixed-base table: kJJFixedWindows windows of 8 bits, entry [j][v] = [v * 2^(8j)] G (v = 0: the identity), so that [k] G is
// one mixed addition per byte of k.  786 KB on the device, built once per context (jubjub.cu: G = BASE, ed25519.cu: G = B).
constexpr int kJJFixedWindows = 32;
constexpr int kJJFixedEntries = kJJFixedWindows * 256;
template <class F, class K> BZK_HD EdExt<F> jj_mul_fixed(const EdNiels<F> *tab, const K &k) {
    EdExt<F> acc = jj_identity<F>();
#pragma unroll 1
    for (int j = 0; j < kJJFixedWindows; j++) acc = jj_add(acc, tab[j * 256 + ((k.l[j >> 2] >> (8 * (j & 3))) & 255u)]);
    return acc;
}

// host: the fixed-base table of the affine point (gx, gy) on the curve with this d (Montgomery); entries normalised to affine
// with one batched inversion
template <class F> inline std::vector<EdNiels<F>> ed_fixed_base_table(const F &gx, const F &gy, const F &d) {
    const F d2 = d.dbl();
    std::vector<EdExt<F>> pts(kJJFixedEntries);
    EdExt<F> row = jj_from_affine(gx, gy);   // [2^(8j)] G
    for (int j = 0; j < kJJFixedWindows; j++) {
        const EdCached<F> step = jj_cached(row, d2);
        EdExt<F> cur = jj_identity<F>();
        for (int v = 0; v < 256; v++) {
            pts[j * 256 + v] = cur;
            cur = jj_add(cur, step);
        }
        row = cur;
    }
    std::vector<F> prefix(kJJFixedEntries);
    F acc = F::one();
    for (int i = 0; i < kJJFixedEntries; i++) { prefix[i] = acc; acc = acc * pts[i].z; }
    F inv = acc.inv_gcd();
    std::vector<EdNiels<F>> out(kJJFixedEntries);
    for (int i = kJJFixedEntries - 1; i >= 0; i--) {
        const F zi = inv * prefix[i];
        inv = inv * pts[i].z;
        const F x = pts[i].x * zi, y = pts[i].y * zi;
        out[i] = EdNiels<F>{y - x, y + x, x * y * d2};
    }
    return out;
}

// BASE (curve.rs:146-164), Montgomery
BZK_HD void jj_base(Fr *x, Fr *y) {
    Fr c;
    c.l[0] = 0xec7beacau; c.l[1] = 0x4df7b7ffu; c.l[2] = 0xfd6c54edu; c.l[3] = 0x2e3ebb21u;
    c.l[4] = 0x0fd6cce6u; c.l[5] = 0xf1fbf02du; c.l[6] = 0x43ac65a6u; c.l[7] = 0x3fd2814cu;
    *x = c.to_mont();
    *y = Fr::from_u32(18);
}

// host: the fixed-base table of BASE for the curve with this d (Montgomery)
inline std::vector<JJNiels> jj_fixed_base_table(const Fr &d) {
    Fr bx, by;
    jj_base(&bx, &by);
    return ed_fixed_base_table(bx, by, d);
}

// Fr square root (Tonelli-Shanks, r - 1 = 2^32 q with q odd, 7 a non-residue); false when none exists.  One 223-bit power:
// w = a^((q-1)/2) gives both x = a w = a^((q+1)/2) and t = x w = a^q; the loop then corrects x by powers of c = 7^q; a
// non-residue is recognised at the end (x^2 != a) instead of by a separate Legendre power.
BZK_HD bool fr_sqrt(const Fr &a, Fr *out) {
    if (a.is_zero()) { *out = a; return true; }
    uint32_t e[8];   // (q - 1) / 2 = (r - 1) >> 33, as 32-bit words
#pragma unroll
    for (int i = 0; i < 8; i++) e[i] = i < 7 ? (FrParams::p(i + 1) >> 1) | (i < 6 ? FrParams::p(i + 2) << 31 : 0u) : 0u;
    Fr c;   // 7^q, Montgomery: a generator of the 2^32-torsion
    c.l[0] = 0x5f0e466au; c.l[1] = 0xb9b58d8cu; c.l[2] = 0x1819d7ecu; c.l[3] = 0x5b1b4c80u;
    c.l[4] = 0x52a31e64u; c.l[5] = 0x0af53ae3u; c.l[6] = 0x19e9b27bu; c.l[7] = 0x5bf3addau;
    const Fr w = a.pow(e, 8);
    Fr x = a * w, t = x * w;
    uint32_t m = 32;
    while (!(t == Fr::one())) {
        uint32_t i = 0;
        Fr t2 = t;
        while (!(t2 == Fr::one())) {
            t2 = t2.sqr();
            if (++i == m) return false;   // t has order 2^m: a is not a square
        }
        Fr b = c;
        for (uint32_t k = 0; k + i + 1 < m; k++) b = b.sqr();
        m = i;
        c = b.sqr();
        t = t * c;
        x = x * b;
    }
    if (!(x * x == a)) return false;
    *out = x;
    return true;
}

// `PointCompressed::decompress` (curve.rs:78-88) before the parity rule: a root y of (1 + x^2) / (1 - d x^2), or false where
// the reference's `.sqrt().unwrap()` (or `.invert().unwrap()`) would panic.  Montgomery in and out.
BZK_HD bool jj_decompress_root(const Fr &x, const Fr &d, Fr *y) {
    const Fr x2 = x.sqr(), den = Fr::one() - d * x2;
    if (den.is_zero()) return false;
    return fr_sqrt((Fr::one() + x2) * den.inv_gcd(), y);   // a = -1
}
// the parity rule: y or -y, whichever has the flag's parity as a canonical integer
BZK_HD Fr jj_with_parity(const Fr &y, bool odd) {
    const bool y_odd = (y.from_mont().l[0] & 1u) != 0;
    return y_odd != odd ? y.neg() : y;
}

// `JubJub::verify` (src/crypto/jubjub/mod.rs:151-167) once h = Poseidon(R.x, R.y, A.x, A.y, msg) is known: A and R on the
// curve and [h] A + R == sB, where sB = [s] BASE (the caller's fixed-base product).  Points Montgomery, h a plain integer.
BZK_HD bool jj_eddsa_check(const Fr &d, const Fr &ax, const Fr &ay, const Fr &rx, const Fr &ry, const Fr &h, const JJ &sB) {
    if (!jj_on_curve(ax, ay, d) || !jj_on_curve(rx, ry, d)) return false;
    const Fr d2 = d.dbl();
    const JJ lhs = jj_add(jj_mul(jj_from_affine(ax, ay), h, d2), jj_cached(jj_from_affine(rx, ry), d2));
    return jj_equal(lhs, sB);
}

}  // namespace bzk
