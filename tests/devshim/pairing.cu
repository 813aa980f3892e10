// Conformance harness for the device half of csrc/pairing.cuh and for the per-proof steps of verify.cu's k_verify_miller
// (test infrastructure, not part of libbzk).
//
// One op table and one record layout, compiled three ways by tests/pairing_cases.py, as tests/devshim/arith.cu is:
//   nvcc, libbzk's sm_90a flags          -> _pairing_dev.so      one thread per record
//   g++ -DBZK_HOST_DEVICE_TEXT           -> _pairing_host_dt.so  the device text with an explicit carry variable
//   g++                                  -> _pairing_host.so     the host fast paths
// A record is an array of 32-bit words: op `op` reads in[0 .. in_w) and writes out[0 .. out_w); pairing_cases.OPS gives
// every op's widths.  Field elements and points are Montgomery limb images; an Fp12 is six Fp2 coefficients of w^k.
#include "pairing.cuh"

using namespace bzk;
using namespace bzk::pairing;

#if defined(__CUDACC__)
#define PAIR_HD __host__ __device__
#else
#define PAIR_HD inline
#endif

enum PairingOp {
    P_F12_MUL,         // a b (Fp12) -> a * b
    P_F12_SQR,         // a -> a^2
    P_F12_MUL_SPARSE,  // a (Fp12) l0 l2 l3 (Fp2) -> a * (l0 + l2 w^2 + l3 w^3)
    P_MILLER_XYZZ,     // P (G1 Xyzz) Q (G2 affine) -> miller_one_xyzz(P, Q)
    P_MUL127,          // A (G1 affine) r (8 words, canonical) -> [r mod 2^127] A, as k_verify_miller walks it (Xyzz)
    P_PROOF_CHECK,     // 387-byte proof image (97 words) -> 1 if k_verify_miller would mark it malformed
    // host builds only (heap and static tables): the verifier's host path
    P_MULTI_MILLER,    // P (G1 affine) Q (G2 affine) -> compute_lines(Q) + multi_miller({P, Q})
    P_FINAL_EXP,       // f -> final_exp(f) = f^(3 (p^12 - 1) / r)
};

template <class T>
PAIR_HD void ld(T &v, const uint32_t *w) {
    uint32_t *d = (uint32_t *)&v;
    for (int i = 0; i < (int)(sizeof(T) / 4); i++) d[i] = w[i];
}
template <class T>
PAIR_HD void st(uint32_t *w, const T &v) {
    const uint32_t *s = (const uint32_t *)&v;
    for (int i = 0; i < (int)(sizeof(T) / 4); i++) w[i] = s[i];
}

// k_verify_miller's per-proof predicate, restated over the same header functions: the flag byte of each point selects the
// identity, otherwise every coordinate must be a canonical limb image and the point must satisfy its curve equation
PAIR_HD bool proof_malformed(const uint8_t *p) {
    auto rd_fp = [&](const uint8_t *q, bool &canon) {
        Fp v;
        for (int i = 0; i < 12; i++) v.l[i] = (uint32_t)q[4 * i] | ((uint32_t)q[4 * i + 1] << 8) | ((uint32_t)q[4 * i + 2] << 16) | ((uint32_t)q[4 * i + 3] << 24);
        canon = canon && Fp::reduce_once(v) == v;
        return v;
    };
    bool canon = true;
    const G1Affine A = p[96] ? G1Affine::inf() : G1Affine{rd_fp(p, canon), rd_fp(p + 48, canon)};
    const G2Affine B = p[97 + 192] ? G2Affine::inf() : G2Affine{Fp2{rd_fp(p + 97, canon), rd_fp(p + 145, canon)}, Fp2{rd_fp(p + 193, canon), rd_fp(p + 241, canon)}};
    const G1Affine C = p[290 + 96] ? G1Affine::inf() : G1Affine{rd_fp(p + 290, canon), rd_fp(p + 338, canon)};
    const Fp four = Fp::from_u32(4);
    const bool okA = A.is_inf() || A.y.sqr() == A.x.sqr() * A.x + four, okC = C.is_inf() || C.y.sqr() == C.x.sqr() * C.x + four,
               okB = B.is_inf() || B.y.sqr() == B.x.sqr() * B.x + Fp2{four, four};
    return !(canon && okA && okB && okC);
}

PAIR_HD Xyzz<Fp> mul127(const G1Affine &P, const Fr &r) {
    Xyzz<Fp> acc = Xyzz<Fp>::inf();
    for (int i = 126; i >= 0; i--) {
        acc = acc.dbl();
        if ((r.l[i >> 5] >> (i & 31)) & 1) acc.madd(P);
    }
    return acc;
}

PAIR_HD void run_op(int op, const uint32_t *in, uint32_t *out) {
    Fp12 a, b;
    switch (op) {
        case P_F12_MUL: ld(a, in); ld(b, in + 144); st(out, f12_mul(a, b)); break;
        case P_F12_SQR: ld(a, in); st(out, f12_sqr(a)); break;
        case P_F12_MUL_SPARSE: {
            Fp2 l0, l2, l3;
            ld(a, in); ld(l0, in + 144); ld(l2, in + 168); ld(l3, in + 192);
            st(out, f12_mul_sparse(a, l0, l2, l3));
            break;
        }
        case P_MILLER_XYZZ: {
            Xyzz<Fp> P;
            G2Affine Q;
            ld(P, in); ld(Q, in + 48);
            st(out, miller_one_xyzz(P, Q));
            break;
        }
        case P_MUL127: {
            G1Affine A;
            Fr r;
            ld(A, in); ld(r, in + 24);
            st(out, mul127(A, r));
            break;
        }
        case P_PROOF_CHECK: out[0] = proof_malformed((const uint8_t *)in) ? 1u : 0u; break;
#if !defined(__CUDA_ARCH__)
        case P_MULTI_MILLER: {
            G1Affine P;
            G2Affine Q;
            ld(P, in); ld(Q, in + 24);
            G2Lines L;
            compute_lines(Q, L);
            const MillerPair pr{P, &L};
            st(out, multi_miller(&pr, 1));
            break;
        }
        case P_FINAL_EXP: ld(a, in); st(out, final_exp(a)); break;
#endif
        default: break;
    }
}

#if defined(__CUDACC__)
__global__ void k_pairing(int op, const uint32_t *in, int in_w, uint32_t *out, int out_w, size_t n) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) run_op(op, in + i * in_w, out + i * out_w);
}

// in / out are device pointers; returns the cudaError_t of the launch and of the synchronisation after it
extern "C" int pairing_run_dev(int op, const uint32_t *in, int in_w, uint32_t *out, int out_w, size_t n, int block) {
    if (n == 0) return 0;
    if (op >= P_MULTI_MILLER) return -1;
    k_pairing<<<(unsigned)((n + block - 1) / block), block>>>(op, in, in_w, out, out_w, n);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    return (int)e;
}
#else
extern "C" void pairing_run_host(int op, const uint32_t *in, int in_w, uint32_t *out, int out_w, size_t n) {
    for (size_t i = 0; i < n; i++) run_op(op, in + i * in_w, out + i * out_w);
}
#endif
