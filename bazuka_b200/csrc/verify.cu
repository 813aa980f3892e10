// bazuka_b200 — Groth16 verifier: single proofs, prepared keys, and random-linear-combination batches.
//
// Replaces `zk::groth16::groth16_verify` (/root/reference/src/zk/groth16/mod.rs:67-121), i.e. bellman 0.14.0
// `prepare_verifying_key` + `verify_proof`:  e(A,B) = e(alpha,beta) * e(sum x_i ic_i, gamma) * e(C, delta),
// public inputs [commitment, height, prev_state, aux_data, next_state] in that order
// (`check_proof`, /root/reference/src/zk/mod.rs:157-193).  The reference re-runs `prepare_verifying_key` (one full
// pairing) on every call and verifies under the node's write lock (/root/reference/src/node/api/post_mpn_solution.rs:12);
// here the prepared key — e(alpha,beta) and the Miller-loop line coefficients of gamma and delta — is an explicit
// handle (`bzk_groth16_pvk_*`), and the plain entry points keep the last few prepared keys in a small cache.
//
//   one proof    3-pair Miller loop with shared squarings (B's lines computed inversion-free, gamma/delta's cached),
//                one final exponentiation, comparison with the cached e(alpha,beta)
//   m proofs     prod_j e(r_j A_j, B_j) * e(-sum_j r_j acc_j, gamma) * e(-sum_j r_j C_j, delta) == e(alpha,beta)^(sum r_j)
//                for random 127-bit r_j: m+2 Miller loops split over host threads, ONE final exponentiation; on
//                failure the proofs are checked one by one so that the caller learns which are bad (SURVEY §8f-4)
// Arithmetic: csrc/pairing.cuh.
#include "common.cuh"
#include "pairing.cuh"
#include <algorithm>
#include <memory>
#include <mutex>
#include <thread>

using namespace bzk;
using namespace bzk::pairing;

struct bzk_groth16_pvk {
    G1Affine alpha;
    G2Affine beta, gamma, delta;
    std::vector<G1Affine> ic;
    G2Lines gamma_lines, delta_lines;
    Fp12 alpha_beta;  // final_exp(miller(alpha, beta))
    std::vector<uint8_t> image;  // the bytes it was prepared from (cache key), may be empty
};

namespace {

// a coordinate must be sent as its canonical Montgomery image (< p): x + p still fits in 384 bits and the field
// arithmetic would read it as x, so one proof would have a second byte string (bellman's decoders refuse it too)
BZK_HD bool canonical(const Fp &v) { return Fp::reduce_once(v) == v; }
BZK_HD bool canonical(const G1Affine &p) { return canonical(p.x) && canonical(p.y); }
BZK_HD bool canonical(const G2Affine &p) { return canonical(p.x.c0) && canonical(p.x.c1) && canonical(p.y.c0) && canonical(p.y.c1); }

// a proof's three points are canonically encoded and lie on their curves (the identity counts as on them)
bool on_curves(const G1Affine &A, const G2Affine &B, const G1Affine &C) {
    return (A.is_inf() || (canonical(A) && on_curve(A))) && (B.is_inf() || (canonical(B) && on_curve(B))) &&
           (C.is_inf() || (canonical(C) && on_curve(C)));
}
bzk_g1_affine g1_at(const uint8_t *p) { bzk_g1_affine g; memset(&g, 0, sizeof g); memcpy(&g, p, 97); return g; }
bzk_g2_affine g2_at(const uint8_t *p) { bzk_g2_affine g; memset(&g, 0, sizeof g); memcpy(&g, p, 193); return g; }

bzk_groth16_pvk *prepare(const G1Affine &alpha, const G2Affine &beta, const G2Affine &gamma, const G2Affine &delta,
                         std::vector<G1Affine> &&ic) {
    bzk_groth16_pvk *k = new (std::nothrow) bzk_groth16_pvk();
    if (!k) return nullptr;
    k->alpha = alpha; k->beta = beta; k->gamma = gamma; k->delta = delta;
    k->ic = std::move(ic);
    compute_lines(gamma, k->gamma_lines);
    compute_lines(delta, k->delta_lines);
    G2Lines bl;
    compute_lines(beta, bl);
    MillerPair p{alpha, &bl};
    k->alpha_beta = final_exp(multi_miller(&p, 1));
    return k;
}

// acc = ic[0] + sum x_i ic[i+1]   (x Montgomery images)
G1Affine input_accumulator(const bzk_groth16_pvk *k, const bzk_fr *inputs, size_t n) {
    std::vector<Fr> sc(n);
    for (size_t i = 0; i < n; i++) {
        Fr x;
        memcpy(x.l, &inputs[i], 32);
        sc[i] = x.from_mont();
    }
    G1Xyzz acc = small_msm(k->ic.data() + 1, sc.data(), n);
    acc.madd(k->ic[0]);
    return acc.to_affine();
}

int32_t verify_one(const bzk_groth16_pvk *k, const bzk_fr *inputs, size_t n, const G1Affine &A, const G2Affine &B, const G1Affine &C) {
    if (!on_curves(A, B, C)) return 0;
    G2Lines bl;
    compute_lines(B, bl);
    const MillerPair pairs[3] = {{A, &bl}, {input_accumulator(k, inputs, n).neg(), &k->gamma_lines}, {C.neg(), &k->delta_lines}};
    return f12_eq(final_exp(multi_miller(pairs, 3)), k->alpha_beta) ? 1 : 0;
}

int32_t parse_vk(const uint8_t *vk, size_t vk_len, bzk_groth16_pvk **out) {
    if (!vk || vk_len < 878) return BZK_ERR_BAD_ARG;
    size_t off = 0;
    const bzk_g1_affine alpha = g1_at(vk + off); off += 97;
    off += 97;  // beta_g1 (not used by the verifier)
    const bzk_g2_affine beta = g2_at(vk + off); off += 193;
    const bzk_g2_affine gamma = g2_at(vk + off); off += 193;
    off += 97;  // delta_g1
    const bzk_g2_affine delta = g2_at(vk + off); off += 193;
    uint64_t n_ic;
    memcpy(&n_ic, vk + off, 8); off += 8;
    if (n_ic == 0 || n_ic > 4096 || vk_len != off + 97 * n_ic) return BZK_ERR_BAD_ARG;
    std::vector<G1Affine> ic(n_ic);
    for (uint64_t i = 0; i < n_ic; i++) { bzk_g1_affine g = g1_at(vk + off + 97 * i); ic[i] = from_wire(&g); }
    bzk_groth16_pvk *k = prepare(from_wire(&alpha), from_wire(&beta), from_wire(&gamma), from_wire(&delta), std::move(ic));
    if (!k) return BZK_ERR_OOM;
    k->image.assign(vk, vk + vk_len);
    *out = k;
    return BZK_OK;
}

// the plain (handle-less) entry points keep the most recently used prepared keys: a node verifies against three keys
// (update / deposit / withdraw, /root/reference/src/config/blockchain.rs:32-37) over and over
struct PvkCache {
    std::mutex mu;
    std::vector<std::shared_ptr<bzk_groth16_pvk>> slots;
    std::shared_ptr<bzk_groth16_pvk> get(const uint8_t *vk, size_t len, int32_t *status) {
        std::lock_guard<std::mutex> g(mu);
        for (size_t i = 0; i < slots.size(); i++)
            if (slots[i]->image.size() == len && memcmp(slots[i]->image.data(), vk, len) == 0) {
                auto hit = slots[i];
                slots.erase(slots.begin() + i);
                slots.insert(slots.begin(), hit);
                return hit;
            }
        bzk_groth16_pvk *k = nullptr;
        *status = parse_vk(vk, len, &k);
        if (*status != BZK_OK) return nullptr;
        std::shared_ptr<bzk_groth16_pvk> sp(k);
        slots.insert(slots.begin(), sp);
        if (slots.size() > 8) slots.pop_back();
        return sp;
    }
};
PvkCache &cache() { static PvkCache c; return c; }

// 127-bit multipliers from a 64-bit seed (SplitMix64); the caller may pass its own
void derive_multipliers(uint64_t seed, size_t m, std::vector<Fr> &r) {
    r.resize(m);
    for (size_t j = 0; j < m; j++) {
        Fr v = Fr::zero();
        const uint64_t a = splitmix_at(seed, 2 * j), b = splitmix_at(seed, 2 * j + 1) >> 1;
        v.l[0] = (uint32_t)a; v.l[1] = (uint32_t)(a >> 32); v.l[2] = (uint32_t)b; v.l[3] = (uint32_t)(b >> 32);
        if (v.is_zero()) v.l[0] = 1;
        r[j] = v;  // canonical
    }
}

// the part of a batch check that does not depend on the individual proofs' points:  given  f = prod_j miller(r_j A_j, B_j)
// and  cs = sum_j r_j C_j,  test  f * miller(-sum_j r_j acc_j, gamma) * miller(-cs, delta) == e(alpha,beta)^(sum r_j)
int32_t batch_tail(const bzk_groth16_pvk *k, const bzk_fr *public_inputs, size_t n_inputs, size_t m, const std::vector<Fr> &r, Fp12 f,
                   const G1Xyzz &cs) {
    // sum_j r_j acc_j = (sum r_j) ic_0 + sum_i (sum_j r_j x_ji) ic_i  — scalars combined in Fr first
    std::vector<Fr> comb(n_inputs + 1, Fr::zero());
    for (size_t j = 0; j < m; j++) {
        const Fr rm = r[j].to_mont();
        comb[0] = comb[0] + rm;
        for (size_t i = 0; i < n_inputs; i++) {
            Fr x;
            memcpy(x.l, &public_inputs[j * n_inputs + i], 32);
            comb[i + 1] = comb[i + 1] + rm * x;
        }
    }
    std::vector<Fr> canon(n_inputs + 1);
    for (size_t i = 0; i <= n_inputs; i++) canon[i] = comb[i].from_mont();
    const G1Affine acc = small_msm(k->ic.data(), canon.data(), n_inputs + 1).to_affine();
    const MillerPair tail[2] = {{acc.neg(), &k->gamma_lines}, {cs.to_affine().neg(), &k->delta_lines}};
    f = f12_mul(f, multi_miller(tail, 2));
    // e(alpha,beta)^(sum r_j): the cached value is already in the target group, raise it there
    Fp12 rhs = f12_one();
    const Fr e = canon[0];
    for (int i = 254; i >= 0; i--) {
        rhs = f12_sqr(rhs);
        if ((e.l[i >> 5] >> (i & 31)) & 1) rhs = f12_mul(rhs, k->alpha_beta);
    }
    return f12_eq(final_exp(f), rhs) ? 1 : 0;
}

// one thread per proof: f_j = miller([r_j] A_j, B_j) with the G2 point walked on the fly, c_j = [r_j] C_j
__global__ void __launch_bounds__(64) k_verify_miller(const uint8_t *__restrict__ proofs387, const Fr *__restrict__ r_canon, uint32_t m,
                                                     Fp12 *__restrict__ out_f, G1Xyzz *__restrict__ out_c, uint8_t *__restrict__ malformed) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= m) return;
    const uint8_t *p = proofs387 + (size_t)387 * j;
    auto rd_fp = [&](const uint8_t *q) {
        Fp v;
        for (int i = 0; i < 12; i++) v.l[i] = (uint32_t)q[4 * i] | ((uint32_t)q[4 * i + 1] << 8) | ((uint32_t)q[4 * i + 2] << 16) | ((uint32_t)q[4 * i + 3] << 24);
        return v;
    };
    G1Affine A = p[96] ? G1Affine::inf() : G1Affine{rd_fp(p), rd_fp(p + 48)};
    G2Affine B = p[97 + 192] ? G2Affine::inf() : G2Affine{Fp2{rd_fp(p + 97), rd_fp(p + 145)}, Fp2{rd_fp(p + 193), rd_fp(p + 241)}};
    G1Affine C = p[290 + 96] ? G1Affine::inf() : G1Affine{rd_fp(p + 290), rd_fp(p + 338)};
    const Fp four = Fp::from_u32(4);
    const bool okA = A.is_inf() || (canonical(A) && A.y.sqr() == A.x.sqr() * A.x + four),
               okC = C.is_inf() || (canonical(C) && C.y.sqr() == C.x.sqr() * C.x + four),
               okB = B.is_inf() || (canonical(B) && B.y.sqr() == B.x.sqr() * B.x + Fp2{four, four});
    malformed[j] = (okA && okB && okC) ? 0 : 1;
    Fr r = load_vec(r_canon + j);
    auto mul127 = [&](const G1Affine &P) {
        G1Xyzz acc = G1Xyzz::inf();
        for (int i = 126; i >= 0; i--) {
            acc = acc.dbl();
            if ((r.l[i >> 5] >> (i & 31)) & 1) acc.madd(P);
        }
        return acc;
    };
    if (malformed[j]) {
        out_f[j] = f12_one();
        out_c[j] = G1Xyzz::inf();
        return;
    }
    out_f[j] = miller_one_xyzz(mul127(A), B);
    out_c[j] = mul127(C);
}

}  // namespace

extern "C" {

int32_t bzk_groth16_pvk_create(const bzk_g1_affine *alpha_g1, const bzk_g2_affine *beta_g2, const bzk_g2_affine *gamma_g2,
                               const bzk_g2_affine *delta_g2, const bzk_g1_affine *ic, size_t n_ic, bzk_groth16_pvk **out) {
    if (!alpha_g1 || !beta_g2 || !gamma_g2 || !delta_g2 || !ic || !n_ic || !out) return BZK_ERR_BAD_ARG;
    std::vector<G1Affine> icv(n_ic);
    for (size_t i = 0; i < n_ic; i++) icv[i] = from_wire(&ic[i]);
    bzk_groth16_pvk *k = prepare(from_wire(alpha_g1), from_wire(beta_g2), from_wire(gamma_g2), from_wire(delta_g2), std::move(icv));
    if (!k) return BZK_ERR_OOM;
    *out = k;
    return BZK_OK;
}
int32_t bzk_groth16_pvk_from_bytes(const uint8_t *vk, size_t vk_len, bzk_groth16_pvk **out) {
    if (!out) return BZK_ERR_BAD_ARG;
    return parse_vk(vk, vk_len, out);
}
int32_t bzk_groth16_pvk_free(bzk_groth16_pvk *k) {
    delete k;
    return BZK_OK;
}

/* 1 = accepted, 0 = rejected (including malformed points), <0 = BZK_ERR_BAD_ARG */
int32_t bzk_groth16_verify_prepared(const bzk_groth16_pvk *k, const bzk_fr *public_inputs, size_t n_inputs,
                                    const bzk_g1_affine *proof_a, const bzk_g2_affine *proof_b, const bzk_g1_affine *proof_c) {
    if (!k || !proof_a || !proof_b || !proof_c || k->ic.size() != n_inputs + 1 || (n_inputs && !public_inputs)) return BZK_ERR_BAD_ARG;
    return verify_one(k, public_inputs, n_inputs, from_wire(proof_a), from_wire(proof_b), from_wire(proof_c));
}

int32_t bzk_groth16_verify(const bzk_g1_affine *alpha_g1, const bzk_g2_affine *beta_g2, const bzk_g2_affine *gamma_g2,
                           const bzk_g2_affine *delta_g2, const bzk_g1_affine *ic, size_t n_ic,
                           const bzk_fr *public_inputs, size_t n_inputs,
                           const bzk_g1_affine *proof_a, const bzk_g2_affine *proof_b, const bzk_g1_affine *proof_c) {
    if (!alpha_g1 || !beta_g2 || !gamma_g2 || !delta_g2 || !ic || !proof_a || !proof_b || !proof_c) return BZK_ERR_BAD_ARG;
    if (n_ic != n_inputs + 1 || (n_inputs && !public_inputs)) return BZK_ERR_BAD_ARG;
    // cache key: the bincode image of the key's verifier-relevant points
    std::vector<uint8_t> img(878 + 97 * n_ic, 0);
    memcpy(img.data(), alpha_g1, 97);
    memcpy(img.data() + 194, beta_g2, 193);
    memcpy(img.data() + 387, gamma_g2, 193);
    memcpy(img.data() + 677, delta_g2, 193);
    const uint64_t n64 = n_ic;
    memcpy(img.data() + 870, &n64, 8);
    for (size_t i = 0; i < n_ic; i++) memcpy(img.data() + 878 + 97 * i, &ic[i], 97);
    int32_t st = BZK_OK;
    auto k = cache().get(img.data(), img.size(), &st);
    if (!k) return st;
    return verify_one(k.get(), public_inputs, n_inputs, from_wire(proof_a), from_wire(proof_b), from_wire(proof_c));
}

/* `check_proof` on the reference's byte images (/root/reference/src/zk/mod.rs:157-193): vk = bincode
 * `Groth16VerifyingKey` (878 + 97*len bytes, /root/reference/src/zk/groth16/mod.rs:22-31), proof = 387-byte
 * `Groth16Proof`; inputs = Montgomery scalars. */
int32_t bzk_groth16_verify_bytes(const uint8_t *vk, size_t vk_len, const bzk_fr *public_inputs, size_t n_inputs, const uint8_t *proof387) {
    if (!vk || !proof387 || vk_len < 878) return BZK_ERR_BAD_ARG;
    int32_t st = BZK_OK;
    auto k = cache().get(vk, vk_len, &st);
    if (!k) return st;
    if (k->ic.size() != n_inputs + 1 || (n_inputs && !public_inputs)) return BZK_ERR_BAD_ARG;
    const bzk_g1_affine a = g1_at(proof387), c = g1_at(proof387 + 290);
    const bzk_g2_affine b = g2_at(proof387 + 97);
    return verify_one(k.get(), public_inputs, n_inputs, from_wire(&a), from_wire(&b), from_wire(&c));
}

/* m proofs under one key.  inputs: m rows of n_inputs Montgomery scalars; proofs: m x 387 bytes; seed: randomness for
 * the 127-bit multipliers (draw it fresh per batch: a prover who knows the multipliers can cancel errors);
 * threads <= 0: hardware concurrency.  ok_each (optional, m bytes) receives the per-proof verdicts.
 * Returns 1 when every proof verifies, 0 otherwise. */
int32_t bzk_groth16_verify_batch(const bzk_groth16_pvk *k, const bzk_fr *public_inputs, size_t n_inputs, const uint8_t *proofs387, size_t m,
                                 uint64_t seed, int32_t threads, uint8_t *ok_each) {
    if (!k || (m && !proofs387) || k->ic.size() != n_inputs + 1 || (m && n_inputs && !public_inputs)) return BZK_ERR_BAD_ARG;
    if (m == 0) return 1;
    int nt = threads > 0 ? threads : (int)std::thread::hardware_concurrency();
    if (nt < 1) nt = 1;
    if ((size_t)nt > m) nt = (int)m;
    std::vector<G1Affine> A(m), C(m);
    std::vector<G2Affine> B(m);
    bool well_formed = true;
    for (size_t j = 0; j < m; j++) {
        const uint8_t *p = proofs387 + 387 * j;
        const bzk_g1_affine a = g1_at(p), c = g1_at(p + 290);
        const bzk_g2_affine b = g2_at(p + 97);
        A[j] = from_wire(&a); B[j] = from_wire(&b); C[j] = from_wire(&c);
    }
    std::vector<Fr> r;
    derive_multipliers(seed, m, r);
    // per-thread partial products over a slice of the proofs
    std::vector<Fp12> part(nt, f12_one());
    std::vector<G1Xyzz> c_part(nt, G1Xyzz::inf());
    std::vector<uint8_t> bad(nt, 0);
    auto work = [&](int t) {
        const size_t lo = m * t / nt, hi = m * (t + 1) / nt;
        Fp12 f = f12_one();
        G1Xyzz cs = G1Xyzz::inf();
        for (size_t j = lo; j < hi; j++) {
            if (!on_curves(A[j], B[j], C[j])) { bad[t] = 1; continue; }
            G2Lines bl;
            compute_lines(B[j], bl);
            const MillerPair p{small_msm(&A[j], &r[j], 1, 127).to_affine(), &bl};
            f = f12_mul(f, multi_miller(&p, 1));
            cs.add(small_msm(&C[j], &r[j], 1, 127));
        }
        part[t] = f;
        c_part[t] = cs;
    };
    std::vector<std::thread> th;
    for (int t = 1; t < nt; t++) th.emplace_back(work, t);
    work(0);
    for (auto &x : th) x.join();
    for (int t = 0; t < nt; t++) if (bad[t]) well_formed = false;
    int32_t all_ok = 0;
    if (well_formed) {
        Fp12 f = part[0];
        G1Xyzz cs = c_part[0];
        for (int t = 1; t < nt; t++) { f = f12_mul(f, part[t]); cs.add(c_part[t]); }
        all_ok = batch_tail(k, public_inputs, n_inputs, m, r, f, cs);
    }
    if (ok_each) {
        if (all_ok) {
            memset(ok_each, 1, m);
        } else {  // find the offenders: one by one, still in parallel
            auto each = [&](int t) {
                for (size_t j = m * t / nt; j < m * (t + 1) / nt; j++)
                    ok_each[j] = (uint8_t)verify_one(k, public_inputs + j * n_inputs, n_inputs, A[j], B[j], C[j]);
            };
            std::vector<std::thread> th2;
            for (int t = 1; t < nt; t++) th2.emplace_back(each, t);
            each(0);
            for (auto &x : th2) x.join();
        }
    }
    return all_ok;
}


/* The same batch check with the m proof-dependent Miller loops on the GPU (one thread per proof: [r_j]A_j, the walk of
 * B_j on the twist and the 68 line evaluations, [r_j]C_j), the product of the m values and the two key-dependent loops +
 * final exponentiation on the host.  Verdicts are identical to bzk_groth16_verify_batch's for the same seed. */
int32_t bzk_groth16_verify_batch_dev(bzk_ctx *ctx, const bzk_groth16_pvk *k, const bzk_fr *public_inputs, size_t n_inputs,
                                     const uint8_t *proofs387, size_t m, uint64_t seed, uint8_t *ok_each) {
    if (!ctx || !k || (m && !proofs387) || k->ic.size() != n_inputs + 1 || (m && n_inputs && !public_inputs) || m >= (1u << 24)) return BZK_ERR_BAD_ARG;
    if (m == 0) return 1;
    BZK_CUDA(ctx, cudaSetDevice(ctx->device));
    std::vector<Fr> r;
    derive_multipliers(seed, m, r);
    size_t need = 0;
    {
        Carver cv(nullptr);
        cv.take<uint8_t>(387 * m); cv.take<Fr>(m); cv.take<Fp12>(m); cv.take<G1Xyzz>(m); cv.take<uint8_t>(m);
        need = cv.used();
    }
    BZK_TRY(ensure_ws(ctx, &ctx->stage, &ctx->stage_bytes, need));
    Carver cv(ctx->stage);
    uint8_t *d_proofs = cv.take<uint8_t>(387 * m);
    Fr *d_r = cv.take<Fr>(m);
    Fp12 *d_f = cv.take<Fp12>(m);
    G1Xyzz *d_c = cv.take<G1Xyzz>(m);
    uint8_t *d_bad = cv.take<uint8_t>(m);
    BZK_CUDA(ctx, cudaMemcpyAsync(d_proofs, proofs387, 387 * m, cudaMemcpyHostToDevice, ctx->stream));
    BZK_CUDA(ctx, cudaMemcpyAsync(d_r, r.data(), m * sizeof(Fr), cudaMemcpyHostToDevice, ctx->stream));
    k_verify_miller<<<div_up(m, 64), 64, 0, ctx->stream>>>(d_proofs, d_r, (uint32_t)m, d_f, d_c, d_bad);
    BZK_LAUNCHED(ctx);
    std::vector<Fp12> hf(m);
    std::vector<G1Xyzz> hc(m);
    std::vector<uint8_t> bad(m);
    BZK_CUDA(ctx, cudaMemcpyAsync(hf.data(), d_f, m * sizeof(Fp12), cudaMemcpyDeviceToHost, ctx->stream));
    BZK_CUDA(ctx, cudaMemcpyAsync(hc.data(), d_c, m * sizeof(G1Xyzz), cudaMemcpyDeviceToHost, ctx->stream));
    BZK_CUDA(ctx, cudaMemcpyAsync(bad.data(), d_bad, m, cudaMemcpyDeviceToHost, ctx->stream));
    BZK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    bool well_formed = true;
    for (size_t j = 0; j < m; j++) well_formed = well_formed && !bad[j];
    int32_t all_ok = 0;
    if (well_formed) {
        // product tree over host threads
        int nt = (int)std::thread::hardware_concurrency();
        if (nt < 1) nt = 1;
        if (nt > 16) nt = 16;
        if ((size_t)nt > m) nt = (int)m;
        std::vector<Fp12> part(nt, f12_one());
        std::vector<G1Xyzz> cp(nt, G1Xyzz::inf());
        auto work = [&](int t) {
            Fp12 f = f12_one();
            G1Xyzz cs = G1Xyzz::inf();
            for (size_t j = m * t / nt; j < m * (t + 1) / nt; j++) { f = f12_mul(f, hf[j]); cs.add(hc[j]); }
            part[t] = f;
            cp[t] = cs;
        };
        std::vector<std::thread> th;
        for (int t = 1; t < nt; t++) th.emplace_back(work, t);
        work(0);
        for (auto &x : th) x.join();
        Fp12 f = part[0];
        G1Xyzz cs = cp[0];
        for (int t = 1; t < nt; t++) { f = f12_mul(f, part[t]); cs.add(cp[t]); }
        all_ok = batch_tail(k, public_inputs, n_inputs, m, r, f, cs);
    }
    if (ok_each) {
        if (all_ok) memset(ok_each, 1, m);
        else return bzk_groth16_verify_batch(k, public_inputs, n_inputs, proofs387, m, seed, 0, ok_each);  // locate the offenders on the host
    }
    return all_ok;
}

}  // extern "C"
