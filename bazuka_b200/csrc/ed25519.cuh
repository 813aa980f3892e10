// bazuka_b200 — Ed25519 signature verification with the verdict of ed25519-dalek 1.x `PublicKey::verify` (the reference's
// `Ed25519::verify`, src/crypto/ed25519.rs:81-83), as BZK_HD code shared by the batch kernels (ed25519.cu), the host call
// bzk_ed25519_verify and the CPU test shim (tests/hostshim/ed25519_shim.cpp).
//
// The verdict for (pk, sig = R || s, M) is 1 iff
//   s < l (s is never reduced);
//   pk decompresses as curve25519-dalek 3.x `CompressedEdwardsY::decompress` does: y is the low 255 bits, taken mod p (a
//     non-canonical y is accepted), x = sqrt_ratio_i(y^2 - 1, d y^2 + 1) must exist, the non-negative root negated when bit
//     255 is set ("-0" is accepted), no torsion check;
//   k = SHA-512(R || pk || M) as a 512-bit little-endian integer mod l;
//   compress([k](-A) + [s]B) == R as bytes, in the full curve group (no cofactor).  compress writes canonical y and the parity
//     of canonical x, so a non-canonical, off-curve or "-0" R never matches.
// d is not a square mod p, so jubjub.cuh's a = -1 extended-coordinate law, a template over the field, is complete here too.
#pragma once
#include <vector>

#include "jubjub.cuh"

namespace bzk {

struct P25519Params {  // p = 2^255 - 19
    static constexpr int N = 8;
    BZK_TABLE(p, 0xffffffedu, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0x7fffffffu)
    BZK_TABLE(one, 0x00000026u, 0u, 0u, 0u, 0u, 0u, 0u, 0u)
    BZK_TABLE(r2, 0x000005a4u, 0u, 0u, 0u, 0u, 0u, 0u, 0u)
    BZK_HD static constexpr uint32_t inv() { return 0x286bca1bu; }
};
struct L25519Params {  // l = 2^252 + 27742317777372353535851937790883648493, the order of B
    static constexpr int N = 8;
    BZK_TABLE(p, 0x5cf5d3edu, 0x5812631au, 0xa2f79cd6u, 0x14def9deu, 0x00000000u, 0x00000000u, 0x00000000u, 0x10000000u)
    BZK_TABLE(one, 0x8d98951du, 0xd6ec3174u, 0x737dcf70u, 0xc6ef5bf4u, 0xfffffffeu, 0xffffffffu, 0xffffffffu, 0x0fffffffu)
    BZK_TABLE(r2, 0x449c0f01u, 0xa40611e3u, 0x68859347u, 0xd00e1ba7u, 0x17f5be65u, 0xceec73d2u, 0x7c309a3du, 0x0399411bu)
    BZK_TABLE(r3, 0x7b83a2dbu, 0x2a9e4968u, 0xaef7f3ecu, 0x278324e6u, 0x04ec5b65u, 0x8065dc6cu, 0x3599cec7u, 0x0e530b77u)
    BZK_HD static constexpr uint32_t inv() { return 0x12547e1bu; }
};
typedef Fe<P25519Params> Fe25519;   // coordinates, Montgomery
typedef Fe<L25519Params> Sc25519;   // scalars: plain integers below l unless said otherwise
using EdPoint = EdExt<Fe25519>;
using EdNiels25519 = EdNiels<Fe25519>;

template <class F> BZK_HD F fe_from_limbs(uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t a4, uint32_t a5, uint32_t a6, uint32_t a7) {
    F r;
    r.l[0] = a0; r.l[1] = a1; r.l[2] = a2; r.l[3] = a3; r.l[4] = a4; r.l[5] = a5; r.l[6] = a6; r.l[7] = a7;
    return r;
}
// 2d, d = -121665/121666, and sqrt(-1) = 2^((p-1)/4), all Montgomery
BZK_HD Fe25519 ed_d2() {
    return fe_from_limbs<Fe25519>(0xbe8fd3f4u, 0x01db17fdu, 0x5f8c52e7u, 0x21430eefu, 0x78310d20u, 0xcb27240fu, 0xe53f8a4du, 0x590456b4u);
}
BZK_HD Fe25519 ed_d() {
    return fe_from_limbs<Fe25519>(0xdf47e9fau, 0x80ed8bfeu, 0xafc62973u, 0x10a18777u, 0xbc188690u, 0xe5939207u, 0x729fc526u, 0x2c822b5au);
}
BZK_HD Fe25519 ed_sqrt_m1() {
    return fe_from_limbs<Fe25519>(0xfe2bdb04u, 0x3b5807d4u, 0xb51be9edu, 0x03f590fdu, 0x336202d1u, 0x6d6e16bfu, 0xd6c71ba8u, 0x75776b0bu);
}
// B = (x, 4/5) with x even, Montgomery
inline void ed_base(Fe25519 *x, Fe25519 *y) {
    *x = fe_from_limbs<Fe25519>(0x8f25d51au, 0xc9562d60u, 0x9525a7b2u, 0x692cc760u, 0xfdd6dc5cu, 0xc0a4e231u, 0xcd6e53feu, 0x216936d3u).to_mont();
    *y = fe_from_limbs<Fe25519>(0x66666658u, 0x66666666u, 0x66666666u, 0x66666666u, 0x66666666u, 0x66666666u, 0x66666666u, 0x66666666u).to_mont();
}

// 32 little-endian bytes as 8 limbs (any alignment)
template <class F> BZK_HD F fe_load_bytes(const uint8_t *b) {
    F r;
#pragma unroll
    for (int i = 0; i < 8; i++) r.l[i] = (uint32_t)b[4 * i] | (uint32_t)b[4 * i + 1] << 8 | (uint32_t)b[4 * i + 2] << 16 | (uint32_t)b[4 * i + 3] << 24;
    return r;
}
BZK_HD bool fe_is_odd(const Fe25519 &m) { return (m.from_mont().l[0] & 1u) != 0; }

// z^(2^k) by k squarings
BZK_HD Fe25519 fe_sqr_n(Fe25519 z, int k) {
#pragma unroll 1
    for (int i = 0; i < k; i++) z = z.sqr();
    return z;
}
// z^(2^250 - 1) and z^11, the common head of the two power chains below (ref10's): 249 squarings, 11 products
BZK_HD Fe25519 fe_pow_2_250_1(const Fe25519 &z, Fe25519 *z11) {
    const Fe25519 z2 = z.sqr(), z9 = fe_sqr_n(z2, 2) * z;
    *z11 = z9 * z2;
    const Fe25519 z5 = z11->sqr() * z9;                   // 2^5 - 1
    const Fe25519 z10 = fe_sqr_n(z5, 5) * z5;             // 2^10 - 1
    const Fe25519 z20 = fe_sqr_n(z10, 10) * z10;          // 2^20 - 1
    const Fe25519 z40 = fe_sqr_n(z20, 20) * z20;          // 2^40 - 1
    const Fe25519 z50 = fe_sqr_n(z40, 10) * z10;          // 2^50 - 1
    const Fe25519 z100 = fe_sqr_n(z50, 50) * z50;         // 2^100 - 1
    const Fe25519 z200 = fe_sqr_n(z100, 100) * z100;      // 2^200 - 1
    return fe_sqr_n(z200, 50) * z50;                      // 2^250 - 1
}
// z^(p - 2) = z^(2^255 - 21): the inverse (0 -> 0)
BZK_HD Fe25519 fe_invert(const Fe25519 &z) {
    Fe25519 z11;
    const Fe25519 t = fe_pow_2_250_1(z, &z11);
    return fe_sqr_n(t, 5) * z11;
}
// z^((p - 5) / 8) = z^(2^252 - 3)
BZK_HD Fe25519 fe_pow_p58(const Fe25519 &z) {
    Fe25519 z11;
    const Fe25519 t = fe_pow_2_250_1(z, &z11);
    return fe_sqr_n(t, 2) * z;
}

// curve25519-dalek's `FieldElement::sqrt_ratio_i`: r = the non-negative (even) root of u/v when u/v is a square (r = 0 when
// u = 0), else of i u/v; returns whether u/v is a square.  r = (u v^3) (u v^7)^((p-5)/8), corrected by sqrt(-1) when
// v r^2 = -u or -u i.  Montgomery in and out.
BZK_HD bool sqrt_ratio_i(const Fe25519 &u, const Fe25519 &v, Fe25519 *out) {
    const Fe25519 v3 = v.sqr() * v, v7 = v3.sqr() * v;
    Fe25519 r = (u * v3) * fe_pow_p58(u * v7);
    const Fe25519 check = v * r.sqr(), mu = u.neg();
    const bool correct = check == u, flipped = check == mu, flipped_i = check == mu * ed_sqrt_m1();
    if (flipped || flipped_i) r = r * ed_sqrt_m1();
    if (fe_is_odd(r)) r = r.neg();
    *out = r;
    return correct || flipped;
}

// `CompressedEdwardsY::decompress`: false where dalek returns None.  (x, y) Montgomery.
BZK_HD bool ed_decompress(const uint8_t pk[32], Fe25519 *x, Fe25519 *y) {
    Fe25519 yy = fe_load_bytes<Fe25519>(pk);
    yy.l[7] &= 0x7fffffffu;
    yy = Fe25519::reduce_once(yy).to_mont();   // y < 2^255 < 2p: non-canonical y is taken mod p
    const Fe25519 y2 = yy.sqr();
    Fe25519 xx;
    if (!sqrt_ratio_i(y2 - Fe25519::one(), y2 * ed_d() + Fe25519::one(), &xx)) return false;
    if (pk[31] >> 7) xx = xx.neg();
    *x = xx;
    *y = yy;
    return true;
}

// `EdwardsPoint::compress`: canonical y, bit 255 = parity of canonical x.  One inversion.
BZK_HD void ed_compress(const EdPoint &p, uint8_t out[32]) {
    const Fe25519 zi = fe_invert(p.z);
    const Fe25519 x = (p.x * zi).from_mont(), y = (p.y * zi).from_mont();
#pragma unroll
    for (int i = 0; i < 8; i++) {
        out[4 * i] = (uint8_t)y.l[i]; out[4 * i + 1] = (uint8_t)(y.l[i] >> 8);
        out[4 * i + 2] = (uint8_t)(y.l[i] >> 16); out[4 * i + 3] = (uint8_t)(y.l[i] >> 24);
    }
    out[31] |= (uint8_t)((x.l[0] & 1u) << 7);
}

// ---------------------------------------------------------------------------------------------------------------- SHA-512
#define BZK_TABLE64(name, ...)                                 \
    BZK_HD static constexpr uint64_t name(int i) {             \
        constexpr uint64_t t[] = {__VA_ARGS__};                \
        return t[i];                                           \
    }
struct Sha512K {
    BZK_TABLE64(k, 0x428a2f98d728ae22ull, 0x7137449123ef65cdull, 0xb5c0fbcfec4d3b2full, 0xe9b5dba58189dbbcull, 0x3956c25bf348b538ull,
                0x59f111f1b605d019ull, 0x923f82a4af194f9bull, 0xab1c5ed5da6d8118ull, 0xd807aa98a3030242ull, 0x12835b0145706fbeull,
                0x243185be4ee4b28cull, 0x550c7dc3d5ffb4e2ull, 0x72be5d74f27b896full, 0x80deb1fe3b1696b1ull, 0x9bdc06a725c71235ull,
                0xc19bf174cf692694ull, 0xe49b69c19ef14ad2ull, 0xefbe4786384f25e3ull, 0x0fc19dc68b8cd5b5ull, 0x240ca1cc77ac9c65ull,
                0x2de92c6f592b0275ull, 0x4a7484aa6ea6e483ull, 0x5cb0a9dcbd41fbd4ull, 0x76f988da831153b5ull, 0x983e5152ee66dfabull,
                0xa831c66d2db43210ull, 0xb00327c898fb213full, 0xbf597fc7beef0ee4ull, 0xc6e00bf33da88fc2ull, 0xd5a79147930aa725ull,
                0x06ca6351e003826full, 0x142929670a0e6e70ull, 0x27b70a8546d22ffcull, 0x2e1b21385c26c926ull, 0x4d2c6dfc5ac42aedull,
                0x53380d139d95b3dfull, 0x650a73548baf63deull, 0x766a0abb3c77b2a8ull, 0x81c2c92e47edaee6ull, 0x92722c851482353bull,
                0xa2bfe8a14cf10364ull, 0xa81a664bbc423001ull, 0xc24b8b70d0f89791ull, 0xc76c51a30654be30ull, 0xd192e819d6ef5218ull,
                0xd69906245565a910ull, 0xf40e35855771202aull, 0x106aa07032bbd1b8ull, 0x19a4c116b8d2d0c8ull, 0x1e376c085141ab53ull,
                0x2748774cdf8eeb99ull, 0x34b0bcb5e19b48a8ull, 0x391c0cb3c5c95a63ull, 0x4ed8aa4ae3418acbull, 0x5b9cca4f7763e373ull,
                0x682e6ff3d6b2b8a3ull, 0x748f82ee5defb2fcull, 0x78a5636f43172f60ull, 0x84c87814a1f0ab72ull, 0x8cc702081a6439ecull,
                0x90befffa23631e28ull, 0xa4506cebde82bde9ull, 0xbef9a3f7b2c67915ull, 0xc67178f2e372532bull, 0xca273eceea26619cull,
                0xd186b8c721c0c207ull, 0xeada7dd6cde0eb1eull, 0xf57d4f7fee6ed178ull, 0x06f067aa72176fbaull, 0x0a637dc5a2c898a6ull,
                0x113f9804bef90daeull, 0x1b710b35131c471bull, 0x28db77f523047d84ull, 0x32caab7b40c72493ull, 0x3c9ebe0a15c9bebcull,
                0x431d67c49c100d4cull, 0x4cc5d4becb3e42b6ull, 0x597f299cfc657e2aull, 0x5fcb6fab3ad6faecull, 0x6c44198c4a475817ull)
};
BZK_HD uint64_t rotr64(uint64_t x, int n) { return (x >> n) | (x << (64 - n)); }

BZK_HD void sha512_block(uint64_t h[8], uint64_t w[16]) {
    uint64_t a = h[0], b = h[1], c = h[2], d = h[3], e = h[4], f = h[5], g = h[6], hh = h[7];
#pragma unroll
    for (int t = 0; t < 80; t++) {
        if (t >= 16) {
            const uint64_t w15 = w[(t + 1) & 15], w2 = w[(t + 14) & 15];
            w[t & 15] += (rotr64(w15, 1) ^ rotr64(w15, 8) ^ (w15 >> 7)) + w[(t + 9) & 15] + (rotr64(w2, 19) ^ rotr64(w2, 61) ^ (w2 >> 6));
        }
        const uint64_t t1 = hh + (rotr64(e, 14) ^ rotr64(e, 18) ^ rotr64(e, 41)) + ((e & f) ^ (~e & g)) + Sha512K::k(t) + w[t & 15];
        const uint64_t t2 = (rotr64(a, 28) ^ rotr64(a, 34) ^ rotr64(a, 39)) + ((a & b) ^ (a & c) ^ (b & c));
        hh = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + t2;
    }
    h[0] += a; h[1] += b; h[2] += c; h[3] += d; h[4] += e; h[5] += f; h[6] += g; h[7] += hh;
}

// SHA-512 of p0[0..n0) || p1[0..n1) || p2[0..n2) (FIPS 180-4), without copying the pieces: each block's words are gathered
// byte by byte from wherever their bytes lie, padding included.  out: the 64-byte digest.
BZK_HD void sha512_parts(const uint8_t *p0, uint64_t n0, const uint8_t *p1, uint64_t n1, const uint8_t *p2, uint64_t n2, uint8_t out[64]) {
    uint64_t h[8] = {0x6a09e667f3bcc908ull, 0xbb67ae8584caa73bull, 0x3c6ef372fe94f82bull, 0xa54ff53a5f1d36f1ull,
                     0x510e527fade682d1ull, 0x9b05688c2b3e6c1full, 0x1f83d9abfb41bd6bull, 0x5be0cd19137e2179ull};
    const uint64_t total = n0 + n1 + n2, blocks = (total + 17 + 127) / 128, bits = total << 3;
#pragma unroll 1
    for (uint64_t blk = 0; blk < blocks; blk++) {
        uint64_t w[16];
        const uint64_t base = blk * 128;
        if (base + 128 <= total) {
            // a block of data only (every block but the last one or two)
#pragma unroll
            for (int j = 0; j < 16; j++) {
                uint64_t v = 0;
#pragma unroll
                for (int k = 0; k < 8; k++) {
                    const uint64_t pos = base + 8 * j + k;
                    const uint8_t byte = pos < n0 ? p0[pos] : pos < n0 + n1 ? p1[pos - n0] : p2[pos - n0 - n1];
                    v = v << 8 | byte;
                }
                w[j] = v;
            }
        } else {
#pragma unroll 1
            for (int j = 0; j < 16; j++) {
                uint64_t v = 0;
                for (int k = 0; k < 8; k++) {
                    const uint64_t pos = base + 8 * j + k;
                    uint8_t byte;
                    if (pos < n0) byte = p0[pos];
                    else if (pos < n0 + n1) byte = p1[pos - n0];
                    else if (pos < total) byte = p2[pos - n0 - n1];
                    else if (pos == total) byte = 0x80;
                    else if (blk + 1 == blocks && 8 * j + k >= 120) byte = (uint8_t)(bits >> (8 * (127 - (8 * j + k))));
                    else byte = 0;
                    v = v << 8 | byte;
                }
                w[j] = v;
            }
        }
        sha512_block(h, w);
    }
#pragma unroll
    for (int i = 0; i < 8; i++)
#pragma unroll
        for (int k = 0; k < 8; k++) out[8 * i + k] = (uint8_t)(h[i] >> (56 - 8 * k));
}

// `Scalar::from_hash`: the 64 digest bytes as a 512-bit little-endian integer mod l, returned as a plain integer.  With lo, hi
// the two 256-bit halves (unreduced: the Montgomery product of an operand below 2^256 and one below l is still below 2l),
// lo * R^2 / R + hi * R^3 / R = (lo + hi 2^256) R; one more product by 1 removes the R.
BZK_HD Sc25519 sc_from_hash(const uint8_t h[64]) {
    Sc25519 r3;
#pragma unroll
    for (int i = 0; i < 8; i++) r3.l[i] = L25519Params::r3(i);
    const Sc25519 lo = fe_load_bytes<Sc25519>(h), hi = fe_load_bytes<Sc25519>(h + 32);
    return (lo * Sc25519::r2() + hi * r3).from_mont();
}
// s as a plain integer; false unless s < l (bit 255 set is >= l)
BZK_HD bool sc_canonical(const uint8_t b[32], Sc25519 *s) {
    *s = fe_load_bytes<Sc25519>(b);
    return Sc25519::reduce_once(*s) == *s;
}

// The first half of the verdict (the batch's prepare kernel): s < l, A decompressed, k = SHA-512(R || pk || M) mod l.  On false
// the verdict is 0 and the outputs are unspecified.
BZK_HD bool ed25519_prepare(const uint8_t pk[32], const uint8_t sig[64], const uint8_t *msg, uint64_t len, Fe25519 *ax, Fe25519 *ay, Sc25519 *k) {
    Sc25519 s;
    if (!sc_canonical(sig + 32, &s)) return false;
    if (!ed_decompress(pk, ax, ay)) return false;
    uint8_t h[64];
    sha512_parts(sig, 32, pk, 32, msg, len, h);
    *k = sc_from_hash(h);
    return true;
}
// The second half (the verify kernel): compress([k](-A) + [s]B) == R, s < l already checked.  tab: ed_base_table().
BZK_HD bool ed25519_finish(const Fe25519 &ax, const Fe25519 &ay, const Sc25519 &k, const uint8_t sig[64], const EdNiels25519 *tab) {
    const Fe25519 d2 = ed_d2();
    const Sc25519 s = fe_load_bytes<Sc25519>(sig + 32);
    const EdPoint sum = jj_add(jj_mul(jj_from_affine(ax.neg(), ay), k, d2), jj_cached(jj_mul_fixed(tab, s), d2));
    uint8_t c[32];
    ed_compress(sum, c);
    uint32_t diff = 0;
#pragma unroll
    for (int i = 0; i < 32; i++) diff |= c[i] ^ sig[i];
    return diff == 0;
}

// host: the fixed-base table of B (786 KB)
inline std::vector<EdNiels25519> ed_base_table() {
    Fe25519 bx, by;
    ed_base(&bx, &by);
    return ed_fixed_base_table(bx, by, ed_d());
}

}  // namespace bzk
