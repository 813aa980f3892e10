// Conformance harness for csrc/ed25519.cuh and csrc/jubjub.cuh (test infrastructure, not part of libbzk).
//
// The record layout and the three builds of tests/devshim/arith.cu (the BLS12-381 harness), in a library of its own so that
// neither harness's build grows with the other's ops; tests/edwards_cases.py builds it:
//   nvcc, libbzk's sm_90a flags          -> _edwards_dev.so      one thread per record
//   g++ -DBZK_HOST_DEVICE_TEXT           -> _edwards_host_dt.so  the device text with an explicit carry variable
//   g++                                  -> _edwards_host.so     the host fast paths (mul/add/sub_host64)
// A record is an array of 32-bit words: op `op` reads in[0 .. in_w) and writes out[0 .. out_w); edwards_cases.OPS gives every
// op's widths.  Field elements and points are Montgomery limb images, as libbzk stores them.
//
// op = (type << 4) | kind: type 0 the field mod p = 2^255 - 19, 1 the field mod l (Ed25519's group order), 2 Ed25519's group
// law, 3 JubJub's, 4 Ed25519's scalars, points and SHA-512, 5 JubJub's square roots.  JubJub records (types 3 and 5) start
// with d, Montgomery (8 words); the offsets below follow it.  Points are extended (X, Y, T, Z), 32 words; Niels addends
// (y - x, y + x, 2dxy), 24 words.
#include "ed25519.cuh"

using namespace bzk;

#if defined(__CUDACC__)
#define EDW_HD __host__ __device__
#else
#define EDW_HD inline
#endif

enum FieldKind {
    F_ADD, F_SUB, F_MUL,      // a b -> r
    F_NEG, F_DBL, F_SQR,      // a -> r
    F_TO_MONT, F_FROM_MONT,   // a -> r
    F_FROM_U32,               // v (1 word) -> r
    F_POW,                    // a e (8 words, plain) -> r
    F_INV, F_INV_GCD,         // a -> r
    F_MUL_WIDE,               // a b -> a*b (16 words, plain)
    F_REDUCE_ONCE,            // a (any 8 words) -> a - p if a >= p, else a
};
enum EdKind {
    X_ADD,         // Ext p, Ext q -> jj_add(p, jj_cached(q, 2d))
    X_ADD_NIELS,   // Ext p, Niels q -> jj_add(p, q)
    X_DBL,         // Ext p -> jj_dbl(p)
    X_MUL,         // Ext p, k (8 words, plain) -> jj_mul(p, k, 2d)
    X_MUL_FIXED,   // k (8 words, plain) -> jj_mul_fixed(tab, k)
    X_EQUAL,       // Ext p, Ext q -> 1 word
};
enum Ed25519Kind {
    M_SHA512,         // n0 n1 n2 o0 o1 o2, bytes (SHA_WORDS words) -> sha512_parts(b + o0, n0, b + o1, n1, b + o2, n2) (16 words)
    M_SC_FROM_HASH,   // 64 bytes -> sc_from_hash (8 words)
    M_SC_CANONICAL,   // 32 bytes -> flag, s (9 words)
    M_SQRT_RATIO_I,   // u v (Montgomery) -> flag, r (9 words)
    M_DECOMPRESS,     // 32 bytes -> flag, x, y (17 words, Montgomery)
    M_COMPRESS,       // Ext p -> 32 bytes
    M_CONSTS,         // 1 word (unused) -> ed_d, ed_d2, ed_sqrt_m1 (24 words)
};
enum JubJubKind {
    J_FR_SQRT,      // a -> flag, fr_sqrt(a) (9 words)
    J_DECOMPRESS,   // x, odd (1 word) -> flag, jj_decompress_root, jj_with_parity(root, odd) (17 words)
    J_ON_CURVE,     // x y -> 1 word
    J_CONSTS,       // 1 word (unused) -> jj_base x, y (16 words)
};

template <class T>
EDW_HD void ld(T &v, const uint32_t *w) {
    uint32_t *d = (uint32_t *)&v;
    for (int i = 0; i < (int)(sizeof(T) / 4); i++) d[i] = w[i];
}
template <class T>
EDW_HD void st(uint32_t *w, const T &v) {
    const uint32_t *s = (const uint32_t *)&v;
    for (int i = 0; i < (int)(sizeof(T) / 4); i++) w[i] = s[i];
}

template <class F>
EDW_HD void field_op(int k, const uint32_t *in, uint32_t *out) {
    constexpr int N = F::N;
    F a, b, r;
    switch (k) {
        case F_ADD: ld(a, in); ld(b, in + N); r = a + b; break;
        case F_SUB: ld(a, in); ld(b, in + N); r = a - b; break;
        case F_MUL: ld(a, in); ld(b, in + N); r = a * b; break;
        case F_NEG: ld(a, in); r = a.neg(); break;
        case F_DBL: ld(a, in); r = a.dbl(); break;
        case F_SQR: ld(a, in); r = a.sqr(); break;
        case F_TO_MONT: ld(a, in); r = a.to_mont(); break;
        case F_FROM_MONT: ld(a, in); r = a.from_mont(); break;
        case F_FROM_U32: r = F::from_u32(in[0]); break;
        case F_POW: ld(a, in); r = a.pow(in + N, N); break;
        case F_INV: ld(a, in); r = a.inv(); break;
        case F_INV_GCD: ld(a, in); r = a.inv_gcd(); break;
        case F_MUL_WIDE: ld(a, in); ld(b, in + N); F::mul_wide(out, a, b); return;
        case F_REDUCE_ONCE: ld(a, in); r = F::reduce_once(a); break;
        default: r = F::zero(); break;
    }
    st(out, r);
}

// K: the type the product passes scalars in (Sc25519 for Ed25519, Fr for JubJub); only its limbs are read
template <class F, class K>
EDW_HD void edwards_op(int k, const F &d2, const EdNiels<F> *tab, const uint32_t *in, uint32_t *out) {
    constexpr int E = sizeof(EdExt<F>) / 4;
    EdExt<F> p, q;
    EdNiels<F> nq;
    K s;
    switch (k) {
        case X_ADD: ld(p, in); ld(q, in + E); st(out, jj_add(p, jj_cached(q, d2))); break;
        case X_ADD_NIELS: ld(p, in); ld(nq, in + E); st(out, jj_add(p, nq)); break;
        case X_DBL: ld(p, in); st(out, jj_dbl(p)); break;
        case X_MUL: ld(p, in); ld(s, in + E); st(out, jj_mul(p, s, d2)); break;
        case X_MUL_FIXED: ld(s, in); st(out, jj_mul_fixed(tab, s)); break;
        case X_EQUAL: ld(p, in); ld(q, in + E); out[0] = jj_equal(p, q) ? 1u : 0u; break;
        default: break;
    }
}

EDW_HD void ed25519_op(int k, const uint32_t *in, uint32_t *out) {
    const uint8_t *b = (const uint8_t *)in;
    Fe25519 u, v, x, y;
    Sc25519 s;
    EdPoint p;
    switch (k) {
        case M_SHA512: {
            const uint8_t *data = (const uint8_t *)(in + 6);
            sha512_parts(data + in[3], in[0], data + in[4], in[1], data + in[5], in[2], (uint8_t *)out);
            break;
        }
        case M_SC_FROM_HASH: st(out, sc_from_hash(b)); break;
        case M_SC_CANONICAL: out[0] = sc_canonical(b, &s) ? 1u : 0u; st(out + 1, s); break;
        case M_SQRT_RATIO_I: ld(u, in); ld(v, in + 8); out[0] = sqrt_ratio_i(u, v, &x) ? 1u : 0u; st(out + 1, x); break;
        case M_DECOMPRESS:
            x = y = Fe25519::zero();
            out[0] = ed_decompress(b, &x, &y) ? 1u : 0u;
            st(out + 1, x);
            st(out + 9, y);
            break;
        case M_COMPRESS: ld(p, in); ed_compress(p, (uint8_t *)out); break;
        case M_CONSTS: st(out, ed_d()); st(out + 8, ed_d2()); st(out + 16, ed_sqrt_m1()); break;
        default: break;
    }
}

EDW_HD void jubjub_op(int k, const Fr &d, const uint32_t *in, uint32_t *out) {
    Fr a, y;
    switch (k) {
        case J_FR_SQRT: ld(a, in); y = Fr::zero(); out[0] = fr_sqrt(a, &y) ? 1u : 0u; st(out + 1, y); break;
        case J_DECOMPRESS:
            ld(a, in);
            y = Fr::zero();
            out[0] = jj_decompress_root(a, d, &y) ? 1u : 0u;
            st(out + 1, y);
            st(out + 9, jj_with_parity(y, in[8] != 0));
            break;
        case J_ON_CURVE: ld(a, in); ld(y, in + 8); out[0] = jj_on_curve(a, y, d) ? 1u : 0u; break;
        case J_CONSTS: jj_base(&a, &y); st(out, a); st(out + 8, y); break;
        default: break;
    }
}

// tab: the curve's fixed-base table (EdNiels of its field), read by X_MUL_FIXED only
EDW_HD void run_op(int op, const void *tab, const uint32_t *in, uint32_t *out) {
    Fr d;
    switch (op >> 4) {
        case 0: field_op<Fe25519>(op & 15, in, out); break;
        case 1: field_op<Sc25519>(op & 15, in, out); break;
        case 2: edwards_op<Fe25519, Sc25519>(op & 15, ed_d2(), (const EdNiels25519 *)tab, in, out); break;
        case 3: ld(d, in); edwards_op<Fr, Fr>(op & 15, d.dbl(), (const JJNiels *)tab, in + 8, out); break;
        case 4: ed25519_op(op & 15, in, out); break;
        case 5: ld(d, in); jubjub_op(op & 15, d, in + 8, out); break;
        default: break;
    }
}

#if defined(__CUDACC__)
__global__ void k_edwards(int op, const void *tab, const uint32_t *in, int in_w, uint32_t *out, int out_w, size_t n) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) run_op(op, tab, in + i * in_w, out + i * out_w);
}

// in / out / tab are device pointers; returns the cudaError_t of the launch and of the synchronisation after it
extern "C" int edwards_run_dev(int op, const uint32_t *in, int in_w, uint32_t *out, int out_w, size_t n, int block, const void *tab) {
    if (n == 0) return 0;
    k_edwards<<<(unsigned)((n + block - 1) / block), block>>>(op, tab, in, in_w, out, out_w, n);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    return (int)e;
}
#else
extern "C" void edwards_run_host(int op, const uint32_t *in, int in_w, uint32_t *out, int out_w, size_t n, const void *tab) {
    for (size_t i = 0; i < n; i++) run_op(op, tab, in + i * in_w, out + i * out_w);
}

// a parameter pack's tables as compiled: p, one, r2 (8 words each), inv, then (l only) r3
extern "C" void edwards_params(int field, uint32_t *out) {
    for (int i = 0; i < 8; i++) {
        out[i] = field ? L25519Params::p(i) : P25519Params::p(i);
        out[8 + i] = field ? L25519Params::one(i) : P25519Params::one(i);
        out[16 + i] = field ? L25519Params::r2(i) : P25519Params::r2(i);
        if (field) out[25 + i] = L25519Params::r3(i);
    }
    out[24] = field ? L25519Params::inv() : P25519Params::inv();
}
#endif

// Host code in every build (nvcc's host pass in the sm_90a one, where libbzk builds the tables it uploads).
// The two fixed-base tables: curve 0 ed_base_table(), curve 1 jj_fixed_base_table(d) (d Montgomery, 8 words);
// out: kJJFixedEntries Niels entries of 24 words.
extern "C" void edwards_table(int curve, const uint32_t *d, uint32_t *out) {
    if (curve == 0) {
        const std::vector<EdNiels25519> t = ed_base_table();
        memcpy(out, t.data(), t.size() * sizeof(EdNiels25519));
    } else {
        Fr dd;
        ld(dd, d);
        const std::vector<JJNiels> t = jj_fixed_base_table(dd);
        memcpy(out, t.data(), t.size() * sizeof(JJNiels));
    }
}
// the curve constants as the host computes them: ed_d, ed_d2, ed_sqrt_m1, ed_base x, y, jj_base x, y (56 words, Montgomery)
extern "C" void edwards_consts(uint32_t *out) {
    Fe25519 bx, by;
    Fr jx, jy;
    ed_base(&bx, &by);
    jj_base(&jx, &jy);
    st(out, ed_d());
    st(out + 8, ed_d2());
    st(out + 16, ed_sqrt_m1());
    st(out + 24, bx);
    st(out + 32, by);
    st(out + 40, jx);
    st(out + 48, jy);
}
