// bazuka_b200 — the external prover's whole job as one native call: the bincode image of an `MpnWork` in, the 391-byte
// `ZkProof::Groth16` out (/root/reference/src/mpn/mod.rs:264-295; the role of the `zoro` worker the reference farms works to,
// /root/reference/src/mpn/mod.rs:79-107, /root/reference/src/client/mod.rs:428-464).
//
//   bzk_mpn_prover_create     per circuit (kind, A, T, B): uploads the natively compiled circuit's witness programs and R1CS,
//                             allocates the resident z = inputs ++ aux, borrows the proving key
//   bzk_mpn_prover_prove_work work -> rows (mpn_wire.cu; entering roots and calldata hashes in 2 + A batched launches)
//                             -> witness on the GPU straight into z (bzk_mpn_update_witness / bzk_mpn_dw_witness)
//                             -> bzk_groth16_prove_dev -> proof bytes
// The update circuit may come from either compile: a blocked one (bzk_mpn_update_circuit_compile_blocked, the 2^26 batch of
// BASELINE configs[3]) is uploaded with bzk_r1cs_upload_blocked, so only its stored rows are read and held.
// Nothing here is new arithmetic: it strings together calls that are each checked on their own; the composition is run in the
// CPU tier over the host stand-ins (tests/test_wire_native_cpu.py) and on the GPU in tests/test_gpu_zz_native_worker.py.
#include <chrono>
#include <memory>

#include "mpn_wire.cuh"

using namespace bzk;

extern "C" int32_t bzk_mpn_circuit_kind(const bzk_mpn_circuit *c, uint32_t out[4]);

struct bzk_mpn_prover {
    uint32_t kind = 0, A = 0, T = 0, B = 0;   // circuit kind: 0 update, 1 deposit, 2 withdraw
    uint64_t shape[12] = {0};
    bzk_witness_program *prog[3] = {nullptr, nullptr, nullptr};   // update: slot, epilogue; deposit / withdraw: phase 1, phase 2, reveal
    std::vector<int32_t> ext_src;
    bzk_r1cs *r1cs = nullptr;
    const bzk_groth16_params *params = nullptr;
    bzk_fr jj_d{}, fee_token{};
    void *d_z = nullptr;   // num_inputs + num_aux field elements
};

namespace {
int32_t upload_program(bzk_ctx *ctx, const bzk_mpn_circuit *c, uint32_t which, const bzk_fr *jj_d_mont, bzk_witness_program **out) {
    uint64_t sz[6];
    BZK_TRY(bzk_mpn_circuit_program(c, which, sz, nullptr, nullptr, nullptr, nullptr, nullptr));
    std::vector<int32_t> ops(sz[0] * 6), lc_ptr(sz[1] + 1), lc_slot(sz[2] + 1), lc_coef(sz[2] + 1);
    std::vector<bzk_fr> coefs(sz[3]);
    BZK_TRY(bzk_mpn_circuit_program(c, which, sz, ops.data(), lc_ptr.data(), lc_slot.data(), lc_coef.data(), coefs.data()));
    return bzk_witness_program_upload(ctx, ops.data(), sz[0], lc_ptr.data(), sz[1], lc_slot.data(), lc_coef.data(), sz[2], coefs.data(), sz[3],
                                      (uint32_t)sz[4], (uint32_t)sz[5], jj_d_mont, out);
}
}  // namespace

namespace bzk {
int32_t mpn_prover_prove(bzk_ctx *ctx, bzk_mpn_prover *p, const bzk_mpn_work *work, const uint8_t prover_address[32], const bzk_fr *r, const bzk_fr *s,
                         int32_t check_satisfied, uint8_t zkproof391[391], double *witness_ms) {
    if (!ctx || !p || !work || !prover_address || !r || !s || !zkproof391) return BZK_ERR_BAD_ARG;
    const auto t0 = std::chrono::steady_clock::now();
    bzk_mpn_work_info info;
    BZK_TRY(bzk_mpn_work_get_info(work, &info));
    // MpnWorkData: 0 deposit, 1 withdraw, 2 update; circuit kinds: 0 update, 1 deposit, 2 withdraw
    const uint32_t want_kind = info.kind == 2 ? 0 : info.kind + 1;
    if (want_kind != p->kind || info.log4_tree != p->A || info.log4_token != p->T || info.log4_batch != p->B) return BZK_ERR_BAD_ARG;
    const uint64_t n = 1ull << (2 * p->B);
    bzk_fr commitment, height{};
    BZK_TRY(bzk_mpn_commitment(prover_address, info.reward, &commitment));
    height.l[0] = info.height;
    Fr *z_in = (Fr *)p->d_z, *z_aux = z_in + p->shape[0];
    if (p->kind == 0) {
        const uint32_t n_raw = update_raw_width(p->A, p->T);
        std::vector<bzk_fr> raws(n * n_raw), ext(n * 2);
        BZK_TRY(bzk_mpn_work_update_rows_ctx(ctx, work, &p->jj_d, &p->fee_token, raws.data(), ext.data()));
        const bzk_fr prologue[6] = {commitment, height, info.state, p->fee_token, info.aux_data, info.next_state};
        BZK_TRY(bzk_mpn_update_witness(ctx, p->prog[0], p->prog[1], n, p->T, p->shape[7], p->shape[10], raws.data(), ext.data(), n_raw, prologue, z_in,
                                       z_aux));
    } else {
        const DwWidths w = p->kind == 1 ? deposit_widths(p->A, p->T) : withdraw_widths(p->A, p->T);
        std::vector<bzk_fr> raws1(n * w.raw1), raws2(n * w.raw2), roots(n), reveal(n * w.reveal);
        BZK_TRY(bzk_mpn_work_dw_rows_ctx(ctx, work, &p->jj_d, raws1.data(), raws2.data(), roots.data(), reveal.data()));
        const bzk_fr public5[5] = {commitment, height, info.state, info.aux_data, info.next_state};
        BZK_TRY(bzk_mpn_dw_witness(ctx, p->prog[0], p->prog[1], p->prog[2], n, raws1.data(), raws2.data(), roots.data(), p->ext_src.data(),
                                   (uint32_t)p->ext_src.size(), reveal.data(), public5, z_in, z_aux));
    }
    if (witness_ms) {   // the rows and the witness alone: wait for the witness kernels
        if (cudaStreamSynchronize(ctx->stream) != cudaSuccess) return set_cuda_err(ctx, cudaGetLastError(), "witness", __FILE__, __LINE__);
        *witness_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    }
    bzk_g1_affine pa, pc;
    bzk_g2_affine pb;
    BZK_TRY(bzk_groth16_prove_dev(ctx, p->params, p->r1cs, z_in, z_aux, r, s, check_satisfied, &pa, &pb, &pc));
    memset(zkproof391, 0, 4);   // ZkProof::Groth16 = variant 0 (/root/reference/src/zk/mod.rs:646-651)
    return bzk_groth16_proof_bytes(&pa, &pb, &pc, zkproof391 + 4);
}

int32_t mpn_prover_key_check(const bzk_mpn_prover *p, const bzk_groth16_params *params) {
    if (!p || !params) return BZK_ERR_BAD_ARG;
    uint64_t want[5], have[5];
    BZK_TRY(bzk_r1cs_shape(p->r1cs, want));
    BZK_TRY(bzk_groth16_params_info(params, have, nullptr, nullptr, nullptr, nullptr, nullptr));
    // {h, l, a, b_g1, b_g2} against {m - 1, num_aux, |a|, |b|, |b|}
    const uint64_t need[5] = {want[1], want[2], want[3], want[4], want[4]};
    return memcmp(need, have, sizeof need) ? BZK_ERR_BAD_ARG : BZK_OK;
}
}  // namespace bzk

extern "C" {

int32_t bzk_mpn_prover_free(bzk_ctx *ctx, bzk_mpn_prover *p) {
    if (!p) return BZK_OK;
    if (!ctx) return BZK_ERR_BAD_ARG;
    for (auto *w : p->prog)
        if (w) bzk_witness_program_free(ctx, w);
    if (p->r1cs) bzk_r1cs_free(ctx, p->r1cs);
    if (p->d_z) { cudaSetDevice(ctx->device); cudaFree(p->d_z); }
    delete p;
    return BZK_OK;
}

/* `params` must be the proving key of exactly this circuit (bzk_r1cs_shape of the circuit's R1CS gives the vector lengths) and
 * outlive the prover; the context must have its Poseidon table loaded (bzk_poseidon_load_params: the rows' hashes are batched
 * launches).  jubjub_d, fee_token (UpdateCircuit's `fee_token`, Ziesha = 1): canonical. */
int32_t bzk_mpn_prover_create(bzk_ctx *ctx, const bzk_mpn_circuit *circuit, const bzk_groth16_params *params, const bzk_fr *jubjub_d,
                              const bzk_fr *fee_token, bzk_mpn_prover **out) {
    if (!ctx || !circuit || !params || !jubjub_d || !fee_token || !out) return BZK_ERR_BAD_ARG;
    std::unique_ptr<bzk_mpn_prover> p(new (std::nothrow) bzk_mpn_prover);
    if (!p) return BZK_ERR_OOM;
    uint32_t k4[4];
    BZK_TRY(bzk_mpn_circuit_kind(circuit, k4));
    p->kind = k4[0]; p->A = k4[1]; p->T = k4[2]; p->B = k4[3];
    BZK_TRY(bzk_mpn_circuit_shape(circuit, p->shape));
    p->params = params;
    p->jj_d = *jubjub_d; p->fee_token = *fee_token;
    int32_t st = BZK_OK;
    Fr d;
    memcpy(d.l, jubjub_d, 32);
    d = d.to_mont();
    const uint32_t n_prog = p->kind == 0 ? 2 : 3;
    for (uint32_t w = 0; st == BZK_OK && w < n_prog; w++) st = upload_program(ctx, circuit, w, (const bzk_fr *)&d, &p->prog[w]);
    if (st == BZK_OK && p->kind != 0) {
        uint64_t counts[2];
        st = bzk_mpn_circuit_two_phase_info(circuit, counts, nullptr, nullptr);
        if (st == BZK_OK) {
            std::vector<int32_t> row_local(counts[0] + 1);
            p->ext_src.resize(counts[1]);
            st = bzk_mpn_circuit_two_phase_info(circuit, counts, row_local.data(), p->ext_src.data());
        }
    }
    if (st == BZK_OK) {   // the circuit's R1CS, resident
        // a blocked compile stores fewer entries than the expanded system has (bzk_mpn_circuit_shape counts the expanded one)
        uint64_t blk[9];
        const bool blocked = p->kind == 0 && bzk_mpn_circuit_blocks(circuit, blk) == BZK_OK &&
                             (blk[6] != p->shape[3] || blk[7] != p->shape[4] || blk[8] != p->shape[5]);
        const uint64_t rows = blocked ? blk[0] + blk[1] + blk[3] : p->shape[2];
        std::vector<uint64_t> rp[3];
        std::vector<uint32_t> col[3];
        std::vector<bzk_fr> val[3];
        for (uint32_t s = 0; st == BZK_OK && s < 3; s++) {
            const uint64_t nnz = blocked ? blk[6 + s] : p->shape[3 + s];
            rp[s].resize(rows + 1); col[s].resize(nnz + 1); val[s].resize(nnz + 1);
            st = bzk_mpn_circuit_matrix(circuit, s, rp[s].data(), col[s].data(), val[s].data());
        }
        if (st == BZK_OK && blocked) {
            const uint64_t *rps[3] = {rp[0].data(), rp[1].data(), rp[2].data()};
            const uint32_t *cols[3] = {col[0].data(), col[1].data(), col[2].data()};
            const bzk_fr *vals[3] = {val[0].data(), val[1].data(), val[2].data()};
            st = bzk_r1cs_upload_blocked(ctx, p->shape[0], p->shape[1], blk[0], blk[1], blk[2], blk[3], blk[4], blk[5], rps, cols, vals, &p->r1cs);
        } else if (st == BZK_OK) {
            st = bzk_r1cs_upload(ctx, p->shape[0], p->shape[1], rows, rp[0].data(), col[0].data(), val[0].data(), rp[1].data(), col[1].data(),
                                 val[1].data(), rp[2].data(), col[2].data(), val[2].data(), &p->r1cs);
        }
    }
    if (st == BZK_OK) {
        cudaSetDevice(ctx->device);
        if (cudaMalloc(&p->d_z, (p->shape[0] + p->shape[1]) * sizeof(Fr)) != cudaSuccess) { cudaGetLastError(); st = BZK_ERR_OOM; }
    }
    if (st != BZK_OK) { bzk_mpn_prover_free(ctx, p.release()); return st; }
    *out = p.release();
    return BZK_OK;
}

/* work_bytes = `bincode::serialize(&work)`; prover_address = the worker's ed25519 address (it enters the commitment, so a proof
 * is only good for the address it was made for); r, s: the proof's blinding scalars (Montgomery images, as bzk_groth16_prove
 * takes them).  zkproof391 = `bincode::serialize(&ZkProof::Groth16(..))`.  BZK_ERR_BAD_ARG: the work is not for this circuit
 * (kind or sizes) or malformed; BZK_ERR_UNSAT (check_satisfied != 0): the transitions do not satisfy the circuit. */
int32_t bzk_mpn_prover_prove_work(bzk_ctx *ctx, bzk_mpn_prover *p, const uint8_t *work_bytes, size_t work_len, const uint8_t prover_address[32],
                                  const bzk_fr *r, const bzk_fr *s, int32_t check_satisfied, uint8_t zkproof391[391]) {
    if (!ctx || !p || !work_bytes || !prover_address || !r || !s || !zkproof391) return BZK_ERR_BAD_ARG;
    bzk_mpn_work *raw = nullptr;
    BZK_TRY(bzk_mpn_work_decode(work_bytes, work_len, &raw, nullptr));
    std::unique_ptr<bzk_mpn_work, int32_t (*)(bzk_mpn_work *)> work(raw, bzk_mpn_work_free);
    return mpn_prover_prove(ctx, p, work.get(), prover_address, r, s, check_satisfied, zkproof391, nullptr);
}

}  // extern "C"
