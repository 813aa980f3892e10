// bazuka_b200 — BLS12-381 G1/G2 group arithmetic for the MSM kernels (device + host).
//
// GPU-side replacement for bls12_381 0.8.0 `G1Affine/G1Projective/G2Affine/G2Projective`
// (un-vendored crate; the reference sees them only through the transmuted wire tuples
//  `(Fp,Fp,bool)` / `((Fp,Fp),(Fp,Fp),bool)`, /root/reference/src/zk/groth16/mod.rs:21-38, and through
//  bellman's multiexp inside create_proof, call sites /root/reference/src/mpn/circuits/test.rs:135,175,215).
//
// Representation choices (GPU-first, not the crate's):
//   * bases in HBM:  packed affine {x,y}, 96 B (G1) / 192 B (G2), 16-byte aligned so a point is
//     6 / 12 LDG.128;  identity is encoded as x = y = 0 (not on the curve, b != 0).  The 104 / 200-byte
//     crate images (x | y | infinity byte | pad) are converted at the C-ABI boundary.
//   * accumulators:  extended Jacobian "XYZZ" (x = X/ZZ, y = Y/ZZZ, ZZ^3 = ZZZ^2); mixed addition
//     is 8M+2S with no inversion and no field doubling chains; identity is ZZ = 0.
// Every exceptional case (P+P, P-P, identity operands) is handled, so results are exact group
// elements for adversarial inputs too (repeated bases, zero scalars), which the parity tests use.
#pragma once
#include "ff.cuh"

// Cold group operations (full additions, doublings, inversions) are kept out of line on the
// device: they are 5-10 k instructions each, and inlining them at every call site (including the
// never-taken exceptional branches of the hot mixed addition) multiplies compile time and I-cache
// footprint for no gain.
#if defined(__CUDACC__)
#define BZK_HD_COLD __host__ __device__ __noinline__
#else
#define BZK_HD_COLD
#endif

namespace bzk {

// ------------------------------------------------------------------------------------------
// Fp2 = Fp[u]/(u^2+1), memory order c0 | c1 (bls12_381 `Fp2 {c0, c1}`).
// ------------------------------------------------------------------------------------------
struct Fp2 {
    Fp c0, c1;
    BZK_HD static Fp2 zero() { return Fp2{Fp::zero(), Fp::zero()}; }
    BZK_HD static Fp2 one() { return Fp2{Fp::one(), Fp::zero()}; }
    BZK_HD bool is_zero() const { return c0.is_zero() && c1.is_zero(); }
    BZK_HD bool operator==(const Fp2 &o) const { return c0 == o.c0 && c1 == o.c1; }
    BZK_HD bool operator!=(const Fp2 &o) const { return !(*this == o); }
    BZK_HD friend Fp2 operator+(const Fp2 &a, const Fp2 &b) { return Fp2{a.c0 + b.c0, a.c1 + b.c1}; }
    BZK_HD friend Fp2 operator-(const Fp2 &a, const Fp2 &b) { return Fp2{a.c0 - b.c0, a.c1 - b.c1}; }
    BZK_HD Fp2 neg() const { return Fp2{c0.neg(), c1.neg()}; }
    BZK_HD Fp2 dbl() const { return Fp2{c0.dbl(), c1.dbl()}; }
    // Karatsuba: 3 base-field products
    BZK_HD friend Fp2 operator*(const Fp2 &a, const Fp2 &b) {
        Fp t0 = a.c0 * b.c0;
        Fp t1 = a.c1 * b.c1;
        Fp t2 = (a.c0 + a.c1) * (b.c0 + b.c1);
        return Fp2{t0 - t1, t2 - t0 - t1};
    }
    // complex squaring: 2 base-field products
    BZK_HD Fp2 sqr() const {
        Fp t = c0 * c1;
        return Fp2{(c0 + c1) * (c0 - c1), t.dbl()};
    }
    BZK_HD Fp2 inv() const {
        Fp n = (c0.sqr() + c1.sqr()).inv();
        return Fp2{c0 * n, (c1 * n).neg()};
    }
};

// ------------------------------------------------------------------------------------------
// Points.  F = Fp (G1) or Fp2 (G2).
// ------------------------------------------------------------------------------------------
template <class F>
struct Affine {
    F x, y;
    BZK_HD bool is_inf() const { return x.is_zero() && y.is_zero(); }
    BZK_HD static Affine inf() { return Affine{F::zero(), F::zero()}; }
    BZK_HD Affine neg() const { return Affine{x, y.neg()}; }
};

template <class F>
struct Xyzz {
    F X, Y, ZZ, ZZZ;

    BZK_HD static Xyzz inf() { return Xyzz{F::zero(), F::zero(), F::zero(), F::zero()}; }
    BZK_HD bool is_inf() const { return ZZ.is_zero(); }
    BZK_HD static Xyzz from_affine(const Affine<F> &p) {
        if (p.is_inf()) return inf();
        return Xyzz{p.x, p.y, F::one(), F::one()};
    }
    BZK_HD Xyzz neg() const { return Xyzz{X, Y.neg(), ZZ, ZZZ}; }

    // 2*(affine p)  — mdbl-2008-s-1 (a = 0)
    BZK_HD_COLD static Xyzz dbl_affine(const Affine<F> &p) {
        if (p.is_inf() || p.y.is_zero()) return inf();
        F U = p.y.dbl();
        F V = U.sqr();
        F W = U * V;
        F S = p.x * V;
        F M = p.x.sqr();
        M = M.dbl() + M;
        Xyzz r;
        r.X = M.sqr() - S.dbl();
        r.Y = M * (S - r.X) - W * p.y;
        r.ZZ = V;
        r.ZZZ = W;
        return r;
    }
    // 2*this — dbl-2008-s-1 (a = 0)
    BZK_HD_COLD Xyzz dbl() const {
        if (is_inf() || Y.is_zero()) return inf();
        F U = Y.dbl();
        F V = U.sqr();
        F W = U * V;
        F S = X * V;
        F M = X.sqr();
        M = M.dbl() + M;
        Xyzz r;
        r.X = M.sqr() - S.dbl();
        r.Y = M * (S - r.X) - W * Y;
        r.ZZ = V * ZZ;
        r.ZZZ = W * ZZZ;
        return r;
    }
    // this += affine p — madd-2008-s (8M + 2S) with all exceptional cases
    BZK_HD void madd(const Affine<F> &p) {
        if (p.is_inf()) return;
        if (is_inf()) {
            X = p.x; Y = p.y; ZZ = F::one(); ZZZ = F::one();
            return;
        }
        F Pd = p.x * ZZ - X;
        F Rd = p.y * ZZZ - Y;
        if (Pd.is_zero()) {
            if (Rd.is_zero()) *this = dbl_affine(p);
            else *this = inf();
            return;
        }
        F PP = Pd.sqr();
        F PPP = Pd * PP;
        F Q = X * PP;
        F X3 = Rd.sqr() - PPP - Q.dbl();
        Y = Rd * (Q - X3) - Y * PPP;
        X = X3;
        ZZ = ZZ * PP;
        ZZZ = ZZZ * PPP;
    }
    // this += o — add-2008-s (12M + 2S) with all exceptional cases
    BZK_HD_COLD void add(const Xyzz &o) {
        if (o.is_inf()) return;
        if (is_inf()) { *this = o; return; }
        F U1 = X * o.ZZ;
        F U2 = o.X * ZZ;
        F S1 = Y * o.ZZZ;
        F S2 = o.Y * ZZZ;
        F Pd = U2 - U1;
        F Rd = S2 - S1;
        if (Pd.is_zero()) {
            if (Rd.is_zero()) *this = dbl();
            else *this = inf();
            return;
        }
        F PP = Pd.sqr();
        F PPP = Pd * PP;
        F Q = U1 * PP;
        F X3 = Rd.sqr() - PPP - Q.dbl();
        Y = Rd * (Q - X3) - S1 * PPP;
        X = X3;
        ZZ = ZZ * o.ZZ * PP;
        ZZZ = ZZZ * o.ZZZ * PPP;
    }
    BZK_HD_COLD Affine<F> to_affine() const {
        if (is_inf()) return Affine<F>::inf();
        // x = X/ZZ, y = Y/ZZZ with one inversion: i = 1/(ZZ*ZZZ)
        F i = (ZZ * ZZZ).inv();
        return Affine<F>{X * ZZZ * i, Y * ZZ * i};
    }
};

// ------------------------------------------------------------------------------------------
// Affine + affine -> affine with the inversion factored out (batched-affine bucket accumulation, csrc/msm_affine.cuh):
//   den = pair_denominator(a, b);  ... one shared inversion of the product of many den ...;  sum = pair_sum(a, b, 1/den)
// 1 product for the batch's running product + 2 to peel the inverse + 2M + 1S for the sum = 5M + 1S per addition
// against 8M + 2S for the XYZZ mixed addition.  Every exceptional case keeps den = 1 and is resolved in pair_sum:
//   identity operand (x = y = 0) -> the other operand;  a = -b (incl. 2-torsion) -> identity;  a = b -> tangent (den = 2y).
// ------------------------------------------------------------------------------------------
template <class F>
BZK_HD F pair_denominator(const Affine<F> &a, const Affine<F> &b) {
    if (a.is_inf() || b.is_inf()) return F::one();
    const F dx = b.x - a.x;
    if (!dx.is_zero()) return dx;
    if (a.y == b.y && !a.y.is_zero()) return a.y.dbl();
    return F::one();
}
template <class F>
BZK_HD Affine<F> pair_sum(const Affine<F> &a, const Affine<F> &b, const F &dinv) {
    if (a.is_inf()) return b;
    if (b.is_inf()) return a;
    F lam;
    if (a.x != b.x) {
        lam = (b.y - a.y) * dinv;
    } else {
        if (!(a.y == b.y) || a.y.is_zero()) return Affine<F>::inf();
        const F xx = a.x.sqr();
        lam = (xx.dbl() + xx) * dinv;
    }
    Affine<F> r;
    r.x = lam.sqr() - a.x - b.x;
    r.y = lam * (a.x - r.x) - a.y;
    return r;
}

typedef Affine<Fp> G1Affine;
typedef Affine<Fp2> G2Affine;
typedef Xyzz<Fp> G1Xyzz;
typedef Xyzz<Fp2> G2Xyzz;

// [k]p for a canonical (non-Montgomery) 256-bit little-endian scalar; MSB-first double-and-add.
template <class F>
BZK_HD Xyzz<F> scalar_mul(const Affine<F> &p, const uint32_t k[8]) {
    Xyzz<F> acc = Xyzz<F>::inf();
    for (int i = 255; i >= 0; i--) {
        acc = acc.dbl();
        if ((k[i >> 5] >> (i & 31)) & 1) acc.madd(p);
    }
    return acc;
}

// y^2 == x^3 + b for a point that is not the identity: b = 4 on G1, 4(u+1) on G2's twist
BZK_HD bool on_curve(const G1Affine &p) { return p.y.sqr() == p.x.sqr() * p.x + Fp::from_u32(4); }
BZK_HD bool on_curve(const G2Affine &p) {
    const Fp four = Fp::from_u32(4);
    return p.y.sqr() == p.x.sqr() * p.x + Fp2{four, four};
}

// host: generator constants (canonical big-endian hex -> Montgomery)
inline Fp fp_from_hex(const char *hex96) {
    Fp v;
    for (int i = 0; i < 12; i++) {
        uint32_t x = 0;
        for (int k = 0; k < 8; k++) {
            char ch = hex96[(11 - i) * 8 + k];
            x = (x << 4) | (uint32_t)(ch <= '9' ? ch - '0' : (ch | 32) - 'a' + 10);
        }
        v.l[i] = x;
    }
    return v.to_mont();
}
inline G1Affine g1_generator() {
    return G1Affine{
        fp_from_hex("17f1d3a73197d7942695638c4fa9ac0fc3688c4f9774b905a14e3a3f171bac586c55e83ff97a1aeffb3af00adb22c6bb"),
        fp_from_hex("08b3f481e3aaa0f1a09e30ed741d8ae4fcf5e095d5d00af600db18cb2c04b3edd03cc744a2888ae40caa232946c5e7e1")};
}
inline G2Affine g2_generator() {
    return G2Affine{
        Fp2{fp_from_hex("024aa2b2f08f0a91260805272dc51051c6e47ad4fa403b02b4510b647ae3d1770bac0326a805bbefd48056c8c121bdb8"),
            fp_from_hex("13e02b6052719f607dacd3a088274f65596bd0d09920b61ab5da61bbdc7f5049334cf11213945d57e5ac7d055d042b7e")},
        Fp2{fp_from_hex("0ce5d527727d6e118cc9cdc6da2e351aadfd9baa8cbdd3a76d429a695160d12c923ac9cc3baca289e193548608b82801"),
            fp_from_hex("0606c4a02ea734cc32acd2b02bc28b99cb3e287e85a763af267492ab572e99ab3f370d275cec1da1aaa9075ff05f79be")}};
}

}  // namespace bzk
