// Conformance harness for csrc/ff.cuh and csrc/ec.cuh (test infrastructure, not part of libbzk).
//
// One op table and one record layout, compiled three ways by tests/arith_cases.py:
//   nvcc, libbzk's sm_90a flags          -> _arith_dev.so      one thread per record (PTX carry chains, add/sub_limbs32)
//   g++ -DBZK_HOST_DEVICE_TEXT           -> _arith_host_dt.so  the device text with an explicit carry variable
//   g++                                  -> _arith_host.so     the host fast paths (mul/add/sub_host64)
// A record is an array of 32-bit words: op `op` reads in[0 .. in_w) and writes out[0 .. out_w); arith_cases.OPS
// gives every op's widths.  Field elements and points are Montgomery limb images, exactly as libbzk stores them.
//
// op = (type << 4) | kind, type 0 Fr, 1 Fp, 2 Fp2, 3 G1, 4 G2.
#include "ec.cuh"

using namespace bzk;

#if defined(__CUDACC__)
#define ARITH_HD __host__ __device__
#else
#define ARITH_HD inline
#endif

enum FieldKind {  // records, in elements of the field (N words) unless noted
    F_ADD, F_SUB, F_MUL,                 // a b -> r
    F_NEG, F_DBL, F_SQR,                 // a -> r
    F_TO_MONT, F_FROM_MONT,              // a -> r
    F_FROM_U32,                          // v (1 word) -> r
    F_POW,                               // a e (N words, plain) -> r
    F_INV, F_INV_GCD,                    // a -> r
    F_MUL_WIDE,                          // a b -> a*b (2N words, plain)
    F_DOT,                               // t (1 word) m[17] s[17] -> sum_k<t m_k s_k, one reduction (Poseidon's MDS rows)
    F_REDC_WIDE,                         // T (2N+1 words, plain) -> T / 2^(32(N+1)) mod p
    F_REDUCE_ONCE,                       // a (N words, a < 2p) -> a mod p
};
enum Fp2Kind { E_ADD, E_SUB, E_MUL, E_NEG, E_DBL, E_SQR, E_INV };
enum GroupKind {
    G_MADD,        // Xyzz Affine -> Xyzz
    G_ADD,         // Xyzz Xyzz -> Xyzz
    G_DBL,         // Xyzz -> Xyzz
    G_DBL_AFFINE,  // Affine -> Xyzz
    G_TO_AFFINE,   // Xyzz -> Affine
    G_SCALAR_MUL,  // Affine k (8 words, plain) -> Xyzz
    G_PAIR,        // Affine a, Affine b -> den = pair_denominator(a, b), pair_sum(a, b, 1/den)   (F then Affine)
    G_ON_CURVE,    // Affine -> 1 word
};
constexpr int DOT_MAX = 17;

template <class T>
ARITH_HD void ld(T &v, const uint32_t *w) {
    uint32_t *d = (uint32_t *)&v;
    for (int i = 0; i < (int)(sizeof(T) / 4); i++) d[i] = w[i];
}
template <class T>
ARITH_HD void st(uint32_t *w, const T &v) {
    const uint32_t *s = (const uint32_t *)&v;
    for (int i = 0; i < (int)(sizeof(T) / 4); i++) w[i] = s[i];
}

template <class F>
ARITH_HD void field_op(int k, const uint32_t *in, uint32_t *out) {
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
        case F_DOT: {
            // as Poseidon's loader does: m pre-scaled by 2^32 so that one reduction by N+1 limbs lands in Montgomery form
            F two32 = F::zero();
            two32.l[1] = 1;
            two32 = two32.to_mont();
            uint32_t acc[2 * N + 1], w[2 * N];
            for (int i = 0; i < 2 * N + 1; i++) acc[i] = 0;
            for (uint32_t j = 0; j < in[0] && j < (uint32_t)DOT_MAX; j++) {
                ld(a, in + 1 + j * N);
                ld(b, in + 1 + (DOT_MAX + j) * N);
                F::mul_wide(w, a * two32, b);
                F::wide_accumulate(acc, w);
            }
            r = F::redc_wide(acc);
            break;
        }
        case F_REDC_WIDE: r = F::redc_wide(in); break;
        case F_REDUCE_ONCE: ld(a, in); r = F::reduce_once(a); break;
        default: r = F::zero(); break;
    }
    st(out, r);
}

ARITH_HD void fp2_op(int k, const uint32_t *in, uint32_t *out) {
    Fp2 a, b, r;
    ld(a, in);
    if (k <= E_MUL) ld(b, in + 24);
    switch (k) {
        case E_ADD: r = a + b; break;
        case E_SUB: r = a - b; break;
        case E_MUL: r = a * b; break;
        case E_NEG: r = a.neg(); break;
        case E_DBL: r = a.dbl(); break;
        case E_SQR: r = a.sqr(); break;
        case E_INV: r = a.inv(); break;
        default: r = Fp2::zero(); break;
    }
    st(out, r);
}

template <class F>
ARITH_HD void group_op(int k, const uint32_t *in, uint32_t *out) {
    constexpr int A = sizeof(Affine<F>) / 4, X = sizeof(Xyzz<F>) / 4, W = sizeof(F) / 4;
    Affine<F> a, b;
    Xyzz<F> x, y;
    switch (k) {
        case G_MADD: ld(x, in); ld(a, in + X); x.madd(a); st(out, x); break;
        case G_ADD: ld(x, in); ld(y, in + X); x.add(y); st(out, x); break;
        case G_DBL: ld(x, in); st(out, x.dbl()); break;
        case G_DBL_AFFINE: ld(a, in); st(out, Xyzz<F>::dbl_affine(a)); break;
        case G_TO_AFFINE: ld(x, in); st(out, x.to_affine()); break;
        case G_SCALAR_MUL: ld(a, in); st(out, scalar_mul(a, in + A)); break;
        case G_PAIR: {
            ld(a, in);
            ld(b, in + A);
            const F den = pair_denominator(a, b);
            st(out, den);
            st(out + W, pair_sum(a, b, den.inv()));
            break;
        }
        case G_ON_CURVE: ld(a, in); out[0] = on_curve(a) ? 1u : 0u; break;
        default: break;
    }
}

ARITH_HD void run_op(int op, const uint32_t *in, uint32_t *out) {
    switch (op >> 4) {
        case 0: field_op<Fr>(op & 15, in, out); break;
        case 1: field_op<Fp>(op & 15, in, out); break;
        case 2: fp2_op(op & 15, in, out); break;
        case 3: group_op<Fp>(op & 15, in, out); break;
        case 4: group_op<Fp2>(op & 15, in, out); break;
        default: break;
    }
}

#if defined(__CUDACC__)
__global__ void k_arith(int op, const uint32_t *in, int in_w, uint32_t *out, int out_w, size_t n) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) run_op(op, in + i * in_w, out + i * out_w);
}

// in / out are device pointers; returns the cudaError_t of the launch and of the synchronisation after it
extern "C" int arith_run_dev(int op, const uint32_t *in, int in_w, uint32_t *out, int out_w, size_t n, int block) {
    if (n == 0) return 0;
    k_arith<<<(unsigned)((n + block - 1) / block), block>>>(op, in, in_w, out, out_w, n);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    return (int)e;
}
#else
extern "C" void arith_run_host(int op, const uint32_t *in, int in_w, uint32_t *out, int out_w, size_t n) {
    for (size_t i = 0; i < n; i++) run_op(op, in + i * in_w, out + i * out_w);
}

// a parameter pack's tables as compiled: p, one, r2 (N words each), then inv
template <class P>
static void params(uint32_t *out) {
    for (int i = 0; i < P::N; i++) {
        out[i] = P::p(i);
        out[P::N + i] = P::one(i);
        out[2 * P::N + i] = P::r2(i);
    }
    out[3 * P::N] = P::inv();
}
extern "C" void arith_params(int field, uint32_t *out) {
    if (field == 0) params<FrParams>(out);
    else params<FpParams>(out);
}
#endif
