// bazuka_b200 — the extern "C" surface declared in include/bzk.h.
#include "common.cuh"

namespace bzk {
int32_t msm_g1_run(bzk_ctx *ctx, const BasesRef<Fp> &d_bases, const Fr *d_scalars, size_t n, bzk_g1_affine *out);
int32_t msm_g2_run(bzk_ctx *ctx, const BasesRef<Fp2> &d_bases, const Fr *d_scalars, size_t n, bzk_g2_affine *out);
int32_t precompute_g1(bzk_ctx *ctx, bzk_g1_bases *b, uint32_t max_levels);
int32_t precompute_g2(bzk_ctx *ctx, bzk_g2_bases *b, uint32_t max_levels);
int32_t pack_g1(bzk_ctx *ctx, const uint8_t *d_images, size_t n, G1Affine *d_out, uint32_t *d_bad);
int32_t pack_g2(bzk_ctx *ctx, const uint8_t *d_images, size_t n, G2Affine *d_out, uint32_t *d_bad);
int32_t random_g1(bzk_ctx *ctx, uint64_t seed, size_t n, uint8_t *d_out);
int32_t random_g2(bzk_ctx *ctx, uint64_t seed, size_t n, uint8_t *d_out);
int32_t random_fr(bzk_ctx *ctx, uint64_t seed, size_t n, Fr *d_out);
int32_t host_g1_add(const bzk_g1_affine *a, const bzk_g1_affine *b, bzk_g1_affine *out);
int32_t host_g2_add(const bzk_g2_affine *a, const bzk_g2_affine *b, bzk_g2_affine *out);
int32_t divide_by_z_launch(bzk_ctx *ctx, Fr *d, uint32_t log_n);
int32_t merkle4_build(bzk_ctx *ctx, Fr *d_nodes, uint32_t log4);
int32_t merkle4_prove(bzk_ctx *ctx, const Fr *d_nodes, uint32_t log4, const uint64_t *d_idx, size_t m, Fr *d_proofs);
int32_t merkle4_root(bzk_ctx *ctx, uint32_t log4, const uint64_t *d_idx, const Fr *d_leaves, const Fr *d_proofs, size_t m, Fr *d_roots);
int32_t tree4_versioned_update(bzk_ctx *ctx, uint32_t depth, const uint32_t *d_tree_id, const uint64_t *d_idx, size_t n, Fr *d_vals,
                               const Fr *d_init_proofs, Fr *d_out_proofs);
int32_t groth16_h_launch(bzk_ctx *ctx, Fr *a, Fr *b, Fr *c, uint32_t log_n);
int32_t groth16_h_combine_launch(bzk_ctx *ctx, Fr *a, Fr *b, Fr *c, uint32_t log_n);

// out may be a or b (in-place calls): the pointers are not __restrict__, and each element is read, through the
// read-only path, only by the thread that then writes it, so no thread reads a location after it has been written
__global__ void __launch_bounds__(256) k_fr_binop(int op, const Fr *a, const Fr *b, Fr *out, size_t n) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Fr x = load_vec(a + i), y = load_vec(b + i);
    Fr r = op == BZK_FR_ADD ? x + y : (op == BZK_FR_SUB ? x - y : x * y);
    store_vec(out + i, r);
}
__global__ void __launch_bounds__(256) k_fp_mul(const Fp *a, const Fp *b, Fp *out, size_t n) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    store_vec(out + i, load_vec(a + i) * load_vec(b + i));
}
}  // namespace bzk

using namespace bzk;

template <class B, class A>
static int32_t bases_from_dev(bzk_ctx *ctx, const void *d_images, size_t n, int32_t check, B **out,
                              int32_t (*pack)(bzk_ctx *, const uint8_t *, size_t, A *, uint32_t *)) {
    if (!out || (n && !d_images)) return BZK_ERR_BAD_ARG;
    *out = nullptr;
    B *b = new (std::nothrow) B();
    if (!b) return BZK_ERR_OOM;
    b->n = n;
    uint32_t *d_bad = nullptr;
    cudaError_t e = cudaMalloc(&b->d, (n ? n : 1) * sizeof(A));
    if (e == cudaSuccess && check) {
        e = cudaMalloc(&d_bad, sizeof(uint32_t));
        if (e == cudaSuccess) e = cudaMemsetAsync(d_bad, 0, sizeof(uint32_t), ctx->stream);
    }
    if (e != cudaSuccess) {
        if (b->d) cudaFree(b->d);
        if (d_bad) cudaFree(d_bad);
        delete b;
        return set_cuda_err(ctx, e, "cudaMalloc(bases)", __FILE__, __LINE__);
    }
    int32_t s = pack(ctx, (const uint8_t *)d_images, n, b->d, d_bad);
    uint32_t bad = 0;
    if (s == BZK_OK && check) {
        if (cudaMemcpyAsync(&bad, d_bad, sizeof bad, cudaMemcpyDeviceToHost, ctx->stream) != cudaSuccess ||
            cudaStreamSynchronize(ctx->stream) != cudaSuccess)
            s = BZK_ERR_CUDA;
        else if (bad)
            s = BZK_ERR_NOT_ON_CURVE;
    }
    if (d_bad) cudaFree(d_bad);
    if (s != BZK_OK) {
        cudaFree(b->d);
        delete b;
        return s;
    }
    *out = b;
    return BZK_OK;
}

// every stream of the context that may still read a base vector: its own, the side streams and the pipes' copy streams
static int32_t sync_all_streams(bzk_ctx *ctx) {
    BZK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    for (cudaStream_t st : ctx->aux_stream)
        if (st) BZK_CUDA(ctx, cudaStreamSynchronize(st));
    for (const StreamPipe &p : ctx->pipe)
        if (p.copy) BZK_CUDA(ctx, cudaStreamSynchronize(p.copy));
    return BZK_OK;
}

// level 0 of the vector into new storage on the other side, then the old storage is freed (so a vector never exists
// twice on the device); tables are dropped.  On failure the vector stays where it was.
template <class B>
static int32_t bases_move(bzk_ctx *ctx, B *b, bool to_host) {
    if ((b->h != nullptr) == to_host) return BZK_OK;
    BZK_TRY(sync_all_streams(ctx));
    B moved;
    moved.n = b->n;
    BZK_TRY(bases_alloc(ctx, &moved, to_host));
    void *dst = to_host ? (void *)moved.h : (void *)moved.d;
    const void *src = to_host ? (const void *)b->d : (const void *)b->h;
    cudaError_t e = cudaMemcpyAsync(dst, src, b->n * sizeof(*b->d), to_host ? cudaMemcpyDeviceToHost : cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess) {
        if (moved.h) cudaFreeHost(moved.h);
        if (moved.d) cudaFree(moved.d);
        return set_cuda_err(ctx, e, "base vector move", __FILE__, __LINE__);
    }
    if (b->d) cudaFree(b->d);
    if (b->h) cudaFreeHost(b->h);
    b->d = moved.d;
    b->h = moved.h;
    b->tab_c = 0; b->tab_T = 1; b->tab_G = 0;
    return BZK_OK;
}

template <class B, class A, class IMG>
static int32_t bases_upload(bzk_ctx *ctx, const IMG *host, size_t n, int32_t check, B **out,
                            int32_t (*pack)(bzk_ctx *, const uint8_t *, size_t, A *, uint32_t *)) {
    if (!out || (n && !host)) return BZK_ERR_BAD_ARG;
    const size_t bytes = n * sizeof(IMG);
    BZK_TRY(ensure_ws(ctx, &ctx->stage, &ctx->stage_bytes, bytes + 16));
    BZK_CUDA(ctx, cudaMemcpyAsync(ctx->stage, host, bytes, cudaMemcpyHostToDevice, ctx->stream));
    int32_t s = bases_from_dev<B, A>(ctx, ctx->stage, n, check, out, pack);
    // the staging buffer may be reused by the next call: make sure the pack kernel has consumed it
    BZK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return s;
}

extern "C" {

const char *bzk_strerror(int32_t s) {
    switch (s) {
        case BZK_OK: return "ok";
        case BZK_ERR_BAD_ARG: return "bad argument";
        case BZK_ERR_CUDA: return "CUDA error";
        case BZK_ERR_OOM: return "out of memory";
        case BZK_ERR_NOT_ON_CURVE: return "point not on curve";
        case BZK_ERR_NO_PARAMS: return "Poseidon parameters not loaded";
        case BZK_ERR_NO_DEVICE: return "no CUDA device (libbzk has no CPU path)";
        case BZK_ERR_UNSAT: return "unsatisfied constraint system";
        case BZK_ERR_BAD_ENCODING: return "bad key file encoding";
        case BZK_ERR_NOT_IN_SUBGROUP: return "point not in the prime-order subgroup";
        case BZK_ERR_REJECTED: return "proof rejected by its own verifying key";
        default: return "unknown status";
    }
}
const char *bzk_last_error(const bzk_ctx *ctx) { return ctx ? ctx->err : "null ctx"; }
uint32_t bzk_abi_version(void) { return (1u << 16) | 1u; }

int32_t bzk_ctx_create(int32_t device, bzk_ctx **out) {
    if (!out) return BZK_ERR_BAD_ARG;
    *out = nullptr;
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0) return BZK_ERR_NO_DEVICE;
    if (device < 0 || device >= count) return BZK_ERR_BAD_ARG;
    bzk_ctx *ctx = new (std::nothrow) bzk_ctx();
    if (!ctx) return BZK_ERR_OOM;
    ctx->device = device;
    if (cudaSetDevice(device) != cudaSuccess || cudaStreamCreateWithFlags(&ctx->own_stream, cudaStreamNonBlocking) != cudaSuccess) {
        delete ctx;
        return BZK_ERR_CUDA;
    }
    ctx->stream = ctx->own_stream;
    int sms = 0;
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device) == cudaSuccess && sms > 0) ctx->sm_count = sms;
    *out = ctx;
    return BZK_OK;
}

int32_t bzk_ctx_destroy(bzk_ctx *ctx) {
    if (!ctx) return BZK_ERR_BAD_ARG;
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    for (auto &p : ctx->pos) if (p.d_consts) cudaFree(p.d_consts);
    for (auto &t : ctx->ntt) { if (t.d_fwd) cudaFree(t.d_fwd); if (t.d_inv) cudaFree(t.d_inv); }
    if (ctx->d_gpow) cudaFree(ctx->d_gpow);
    if (ctx->d_jj_table) cudaFree(ctx->d_jj_table);
    if (ctx->d_ed_table) cudaFree(ctx->d_ed_table);
    if (ctx->ws) cudaFree(ctx->ws);
    if (ctx->stage) cudaFree(ctx->stage);
    if (ctx->pinned) cudaFreeHost(ctx->pinned);
    for (auto &w : ctx->aux_ws) if (w) cudaFree(w);
    for (auto &p : ctx->pipe) {
        if (p.copy) { cudaStreamSynchronize(p.copy); cudaStreamDestroy(p.copy); }
        if (p.buf) cudaFree(p.buf);
        for (int b = 0; b < 2; b++) {
            if (p.ready[b]) cudaEventDestroy(p.ready[b]);
            if (p.freed[b]) cudaEventDestroy(p.freed[b]);
        }
    }
    for (auto &st : ctx->aux_stream) if (st) cudaStreamDestroy(st);
    for (auto &e : ctx->aux_ev) if (e) cudaEventDestroy(e);
    for (auto &e : ctx->ev) if (e) cudaEventDestroy(e);
    if (ctx->own_stream) cudaStreamDestroy(ctx->own_stream);
    delete ctx;
    return BZK_OK;
}
int32_t bzk_ctx_set_stream(bzk_ctx *ctx, void *s) {
    if (!ctx) return BZK_ERR_BAD_ARG;
    ctx->stream = s ? (cudaStream_t)s : ctx->own_stream;
    return BZK_OK;
}
int32_t bzk_ctx_synchronize(bzk_ctx *ctx) {
    if (!ctx) return BZK_ERR_BAD_ARG;
    BZK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return BZK_OK;
}
uint64_t bzk_ctx_launch_count(const bzk_ctx *ctx) { return ctx ? ctx->launches : 0; }
int32_t bzk_ctx_set_timing(bzk_ctx *ctx, int32_t on) {
    if (!ctx) return BZK_ERR_BAD_ARG;
    ctx->timing = on != 0;
    ctx->stage_runs = 0;
    for (int i = 0; i < bzk_ctx::kMaxStages; i++) { ctx->stage_ms[i] = 0; ctx->stage_ms_sum[i] = 0; }
    return BZK_OK;
}
int32_t bzk_ctx_set_msm_affine_rounds(bzk_ctx *ctx, int32_t g1_rounds, int32_t g2_rounds) {
    if (!ctx || g1_rounds > 6 || g2_rounds > 6) return BZK_ERR_BAD_ARG;
    ctx->affine_rounds[0] = g1_rounds;
    ctx->affine_rounds[1] = g2_rounds;
    return BZK_OK;
}
int32_t bzk_ctx_set_msm_table_window(bzk_ctx *ctx, uint32_t c) {
    if (!ctx || (c != 0 && (c < 8 || c > 23))) return BZK_ERR_BAD_ARG;
    ctx->table_c = c;
    return BZK_OK;
}
int32_t bzk_ctx_set_msm_stream_chunk(bzk_ctx *ctx, uint64_t points) {
    if (!ctx || (points != 0 && points < 256) || points >= (1ull << 31)) return BZK_ERR_BAD_ARG;
    ctx->stream_chunk = points;
    return BZK_OK;
}
int32_t bzk_ctx_last_msm_stream(const bzk_ctx *ctx, uint64_t out[4]) {
    if (!ctx || !out) return BZK_ERR_BAD_ARG;
    memcpy(out, ctx->last_stream, sizeof ctx->last_stream);
    return BZK_OK;
}
int32_t bzk_ctx_last_msm_plan(const bzk_ctx *ctx, uint32_t out[8]) {
    if (!ctx || !out) return BZK_ERR_BAD_ARG;
    memcpy(out, ctx->last_plan, sizeof ctx->last_plan);
    return BZK_OK;
}
uint64_t bzk_ctx_stage_ms(const bzk_ctx *ctx, float *last_ms, double *sum_ms, uint32_t cap) {
    if (!ctx) return 0;
    for (uint32_t i = 0; i < cap && i < (uint32_t)bzk_ctx::kMaxStages; i++) {
        if (last_ms) last_ms[i] = ctx->stage_ms[i];
        if (sum_ms) sum_ms[i] = ctx->stage_ms_sum[i];
    }
    return ctx->stage_runs;
}

#define BZK_ENTER(ctx)                                   \
    if (!(ctx)) return BZK_ERR_BAD_ARG;                  \
    BZK_CUDA((ctx), cudaSetDevice((ctx)->device));

// ------------------------------------------------------------------ Poseidon
int32_t bzk_poseidon_load_params(bzk_ctx *ctx, const uint8_t *blob, size_t len) {
    BZK_ENTER(ctx);
    if (!blob || len < 12 || memcmp(blob, "BZKPOSv1", 8)) return BZK_ERR_BAD_ARG;
    uint32_t nw;
    memcpy(&nw, blob + 8, 4);
    size_t off = 12;
    for (uint32_t i = 0; i < nw; i++) {
        if (off + 16 > len) return BZK_ERR_BAD_ARG;
        uint32_t hdr[4];
        memcpy(hdr, blob + off, 16);
        off += 16;
        const uint32_t t = hdr[0], nrc = hdr[3];
        if (t < 2 || t > 17 || nrc != t * (hdr[1] + hdr[2])) return BZK_ERR_BAD_ARG;
        const size_t cnt = (size_t)nrc + (size_t)t * t;
        if (off + 32 * cnt > len) return BZK_ERR_BAD_ARG;
        // device table: round constants | MDS rows | MDS rows * 2^32 (for the lazily reduced row products)
        std::vector<Fr> host(cnt + (size_t)t * t);
        Fr two32 = Fr::zero();
        two32.l[1] = 1;
        two32 = two32.to_mont();
        for (size_t k = 0; k < cnt; k++) {
            Fr v;
            memcpy(v.l, blob + off + 32 * k, 32);
            // canonical constants must be < r
            if (Fr::reduce_once(v) != v) return BZK_ERR_BAD_ARG;
            host[k] = v.to_mont();
            if (k >= nrc) host[cnt + (k - nrc)] = host[k] * two32;
        }
        off += 32 * cnt;
        PoseidonTable &pt = ctx->pos[t];
        if (pt.d_consts) { BZK_CUDA(ctx, cudaFree(pt.d_consts)); pt.d_consts = nullptr; }
        BZK_CUDA(ctx, cudaMalloc(&pt.d_consts, host.size() * sizeof(Fr)));
        BZK_CUDA(ctx, cudaMemcpy(pt.d_consts, host.data(), host.size() * sizeof(Fr), cudaMemcpyHostToDevice));
        pt.t = t; pt.rf = hdr[1]; pt.rp = hdr[2]; pt.nrc = nrc;
    }
    if (off != len) return BZK_ERR_BAD_ARG;
    ctx->pos_loaded = true;
    return BZK_OK;
}

int32_t bzk_poseidon_hash_dev(bzk_ctx *ctx, uint32_t arity, const void *d_in, size_t n, void *d_out) {
    BZK_ENTER(ctx);
    if (n && (!d_in || !d_out)) return BZK_ERR_BAD_ARG;
    return poseidon_launch(ctx, arity, (const Fr *)d_in, n, (Fr *)d_out);
}

int32_t bzk_poseidon_hash(bzk_ctx *ctx, uint32_t arity, const bzk_fr *in, size_t n, bzk_fr *out) {
    BZK_ENTER(ctx);
    if (arity < 1 || arity > 16) return BZK_ERR_BAD_ARG;
    if (!ctx->pos_loaded) return BZK_ERR_NO_PARAMS;
    if (n == 0) return BZK_OK;
    if (!in || !out) return BZK_ERR_BAD_ARG;
    const size_t in_bytes = n * arity * sizeof(Fr), out_bytes = n * sizeof(Fr);
    BZK_TRY(ensure_ws(ctx, &ctx->stage, &ctx->stage_bytes, in_bytes + out_bytes + 256));
    Fr *d_in = (Fr *)ctx->stage;
    Fr *d_out = (Fr *)((char *)ctx->stage + ((in_bytes + 255) & ~(size_t)255));
    BZK_CUDA(ctx, cudaMemcpyAsync(d_in, in, in_bytes, cudaMemcpyHostToDevice, ctx->stream));
    BZK_TRY(poseidon_launch(ctx, arity, d_in, n, d_out));
    BZK_CUDA(ctx, cudaMemcpyAsync(out, d_out, out_bytes, cudaMemcpyDeviceToHost, ctx->stream));
    BZK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return BZK_OK;
}

int32_t bzk_merkle4_build_dev(bzk_ctx *ctx, void *d_nodes, uint32_t log4_size) {
    BZK_ENTER(ctx);
    return merkle4_build(ctx, (Fr *)d_nodes, log4_size);
}
int32_t bzk_merkle4_prove_dev(bzk_ctx *ctx, const void *d_nodes, uint32_t log4_size, const void *d_indices, size_t m, void *d_proofs) {
    BZK_ENTER(ctx);
    return merkle4_prove(ctx, (const Fr *)d_nodes, log4_size, (const uint64_t *)d_indices, m, (Fr *)d_proofs);
}
int32_t bzk_merkle4_root_dev(bzk_ctx *ctx, uint32_t log4_size, const void *d_indices, const void *d_leaves, const void *d_proofs, size_t m, void *d_roots) {
    BZK_ENTER(ctx);
    return merkle4_root(ctx, log4_size, (const uint64_t *)d_indices, (const Fr *)d_leaves, (const Fr *)d_proofs, m, (Fr *)d_roots);
}
int32_t bzk_tree4_versioned_update_dev(bzk_ctx *ctx, uint32_t depth, const void *d_tree_id, const void *d_indices, size_t n, void *d_vals,
                                       const void *d_init_proofs, void *d_out_proofs) {
    BZK_ENTER(ctx);
    return tree4_versioned_update(ctx, depth, (const uint32_t *)d_tree_id, (const uint64_t *)d_indices, n, (Fr *)d_vals, (const Fr *)d_init_proofs,
                                  (Fr *)d_out_proofs);
}

// ------------------------------------------------------------------ NTT
int32_t bzk_ntt_dev(bzk_ctx *ctx, void *d_data, uint32_t log_n, int32_t op) {
    BZK_ENTER(ctx);
    return ntt_launch(ctx, (Fr *)d_data, log_n, op);
}
int32_t bzk_ntt(bzk_ctx *ctx, bzk_fr *data, uint32_t log_n, int32_t op) {
    BZK_ENTER(ctx);
    if (!data || log_n > 28 || op < 0 || op > 3) return BZK_ERR_BAD_ARG;
    const size_t bytes = ((size_t)1 << log_n) * sizeof(Fr);
    BZK_TRY(ensure_ws(ctx, &ctx->stage, &ctx->stage_bytes, bytes));
    BZK_CUDA(ctx, cudaMemcpyAsync(ctx->stage, data, bytes, cudaMemcpyHostToDevice, ctx->stream));
    BZK_TRY(ntt_launch(ctx, (Fr *)ctx->stage, log_n, op));
    BZK_CUDA(ctx, cudaMemcpyAsync(data, ctx->stage, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    BZK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return BZK_OK;
}
int32_t bzk_divide_by_z_on_coset_dev(bzk_ctx *ctx, void *d_data, uint32_t log_n) {
    BZK_ENTER(ctx);
    return divide_by_z_launch(ctx, (Fr *)d_data, log_n);
}
int32_t bzk_groth16_h_dev(bzk_ctx *ctx, void *d_a, void *d_b, void *d_c, uint32_t log_n) {
    BZK_ENTER(ctx);
    return groth16_h_launch(ctx, (Fr *)d_a, (Fr *)d_b, (Fr *)d_c, log_n);
}
int32_t bzk_groth16_h_combine_dev(bzk_ctx *ctx, void *d_a, void *d_b, void *d_c, uint32_t log_n) {
    BZK_ENTER(ctx);
    return groth16_h_combine_launch(ctx, (Fr *)d_a, (Fr *)d_b, (Fr *)d_c, log_n);
}

// ------------------------------------------------------------------ bases
int32_t bzk_g1_bases_upload(bzk_ctx *ctx, const bzk_g1_affine *bases, size_t n, int32_t check, bzk_g1_bases **out) {
    BZK_ENTER(ctx);
    return bases_upload<bzk_g1_bases, G1Affine>(ctx, bases, n, check, out, pack_g1);
}
int32_t bzk_g2_bases_upload(bzk_ctx *ctx, const bzk_g2_affine *bases, size_t n, int32_t check, bzk_g2_bases **out) {
    BZK_ENTER(ctx);
    return bases_upload<bzk_g2_bases, G2Affine>(ctx, bases, n, check, out, pack_g2);
}
int32_t bzk_g1_bases_from_dev(bzk_ctx *ctx, const void *d_images, size_t n, bzk_g1_bases **out) {
    BZK_ENTER(ctx);
    return bases_from_dev<bzk_g1_bases, G1Affine>(ctx, d_images, n, 0, out, pack_g1);
}
int32_t bzk_g2_bases_from_dev(bzk_ctx *ctx, const void *d_images, size_t n, bzk_g2_bases **out) {
    BZK_ENTER(ctx);
    return bases_from_dev<bzk_g2_bases, G2Affine>(ctx, d_images, n, 0, out, pack_g2);
}
int32_t bzk_g1_bases_free(bzk_ctx *ctx, bzk_g1_bases *b) {
    BZK_ENTER(ctx);
    if (!b) return BZK_OK;
    BZK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    bases_release(b);
    return BZK_OK;
}
int32_t bzk_g2_bases_free(bzk_ctx *ctx, bzk_g2_bases *b) {
    BZK_ENTER(ctx);
    if (!b) return BZK_OK;
    BZK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    bases_release(b);
    return BZK_OK;
}
int32_t bzk_g1_bases_precompute(bzk_ctx *ctx, bzk_g1_bases *b, uint32_t max_levels) {
    BZK_ENTER(ctx);
    if (!b || b->h) return BZK_ERR_BAD_ARG;
    return precompute_g1(ctx, b, max_levels);
}
int32_t bzk_g2_bases_precompute(bzk_ctx *ctx, bzk_g2_bases *b, uint32_t max_levels) {
    BZK_ENTER(ctx);
    if (!b || b->h) return BZK_ERR_BAD_ARG;
    return precompute_g2(ctx, b, max_levels);
}
int32_t bzk_g1_bases_move(bzk_ctx *ctx, bzk_g1_bases *b, int32_t to_host) {
    BZK_ENTER(ctx);
    if (!b) return BZK_ERR_BAD_ARG;
    return bases_move(ctx, b, to_host != 0);
}
int32_t bzk_g2_bases_move(bzk_ctx *ctx, bzk_g2_bases *b, int32_t to_host) {
    BZK_ENTER(ctx);
    if (!b) return BZK_ERR_BAD_ARG;
    return bases_move(ctx, b, to_host != 0);
}
int32_t bzk_g1_bases_on_host(const bzk_g1_bases *b) { return b && b->h ? 1 : 0; }
int32_t bzk_g2_bases_on_host(const bzk_g2_bases *b) { return b && b->h ? 1 : 0; }
uint32_t bzk_g1_bases_levels(const bzk_g1_bases *b) { return b ? b->tab_T : 0; }
uint32_t bzk_g2_bases_levels(const bzk_g2_bases *b) { return b ? b->tab_T : 0; }
size_t bzk_g1_bases_len(const bzk_g1_bases *b) { return b ? b->n : 0; }
size_t bzk_g2_bases_len(const bzk_g2_bases *b) { return b ? b->n : 0; }

// ------------------------------------------------------------------ MSM
static int32_t stage_scalars(bzk_ctx *ctx, const bzk_fr *scalars, size_t n, Fr **d_out) {
    const size_t bytes = (n ? n : 1) * sizeof(Fr);
    BZK_TRY(ensure_ws(ctx, &ctx->stage, &ctx->stage_bytes, bytes));
    BZK_CUDA(ctx, cudaMemcpyAsync(ctx->stage, scalars, n * sizeof(Fr), cudaMemcpyHostToDevice, ctx->stream));
    *d_out = (Fr *)ctx->stage;
    return BZK_OK;
}

int32_t bzk_msm_g1_resident_dev(bzk_ctx *ctx, const bzk_g1_bases *b, size_t offset, const void *d_scalars, size_t n, bzk_g1_affine *out) {
    BZK_ENTER(ctx);
    if (!b || !out || offset > b->n || n > b->n - offset || (n && !d_scalars)) return BZK_ERR_BAD_ARG;
    return msm_g1_run(ctx, bases_ref(b, offset), (const Fr *)d_scalars, n, out);
}
int32_t bzk_msm_g2_resident_dev(bzk_ctx *ctx, const bzk_g2_bases *b, size_t offset, const void *d_scalars, size_t n, bzk_g2_affine *out) {
    BZK_ENTER(ctx);
    if (!b || !out || offset > b->n || n > b->n - offset || (n && !d_scalars)) return BZK_ERR_BAD_ARG;
    return msm_g2_run(ctx, bases_ref(b, offset), (const Fr *)d_scalars, n, out);
}
int32_t bzk_msm_g1_resident(bzk_ctx *ctx, const bzk_g1_bases *b, size_t offset, const bzk_fr *scalars, size_t n, bzk_g1_affine *out) {
    BZK_ENTER(ctx);
    if (!b || !out || offset > b->n || n > b->n - offset || (n && !scalars)) return BZK_ERR_BAD_ARG;
    Fr *d_s = nullptr;
    BZK_TRY(stage_scalars(ctx, scalars, n, &d_s));
    return msm_g1_run(ctx, bases_ref(b, offset), d_s, n, out);
}
int32_t bzk_msm_g2_resident(bzk_ctx *ctx, const bzk_g2_bases *b, size_t offset, const bzk_fr *scalars, size_t n, bzk_g2_affine *out) {
    BZK_ENTER(ctx);
    if (!b || !out || offset > b->n || n > b->n - offset || (n && !scalars)) return BZK_ERR_BAD_ARG;
    Fr *d_s = nullptr;
    BZK_TRY(stage_scalars(ctx, scalars, n, &d_s));
    return msm_g2_run(ctx, bases_ref(b, offset), d_s, n, out);
}
int32_t bzk_msm_g1(bzk_ctx *ctx, const bzk_g1_affine *bases, const bzk_fr *scalars, size_t n, bzk_g1_affine *out) {
    BZK_ENTER(ctx);
    if (!out || (n && (!bases || !scalars))) return BZK_ERR_BAD_ARG;
    bzk_g1_bases *b = nullptr;
    BZK_TRY(bzk_g1_bases_upload(ctx, bases, n, 0, &b));
    int32_t s = bzk_msm_g1_resident(ctx, b, 0, scalars, n, out);
    bzk_g1_bases_free(ctx, b);
    return s;
}
int32_t bzk_msm_g2(bzk_ctx *ctx, const bzk_g2_affine *bases, const bzk_fr *scalars, size_t n, bzk_g2_affine *out) {
    BZK_ENTER(ctx);
    if (!out || (n && (!bases || !scalars))) return BZK_ERR_BAD_ARG;
    bzk_g2_bases *b = nullptr;
    BZK_TRY(bzk_g2_bases_upload(ctx, bases, n, 0, &b));
    int32_t s = bzk_msm_g2_resident(ctx, b, 0, scalars, n, out);
    bzk_g2_bases_free(ctx, b);
    return s;
}

int32_t bzk_g1_add(const bzk_g1_affine *a, const bzk_g1_affine *b, bzk_g1_affine *out) {
    if (!a || !b || !out) return BZK_ERR_BAD_ARG;
    return host_g1_add(a, b, out);
}
int32_t bzk_g2_add(const bzk_g2_affine *a, const bzk_g2_affine *b, bzk_g2_affine *out) {
    if (!a || !b || !out) return BZK_ERR_BAD_ARG;
    return host_g2_add(a, b, out);
}

// ------------------------------------------------------------------ synthetic inputs, elementwise
int32_t bzk_g1_random_bases_dev(bzk_ctx *ctx, uint64_t seed, size_t n, void *d_out) {
    BZK_ENTER(ctx);
    if (n && !d_out) return BZK_ERR_BAD_ARG;
    return random_g1(ctx, seed, n, (uint8_t *)d_out);
}
int32_t bzk_g2_random_bases_dev(bzk_ctx *ctx, uint64_t seed, size_t n, void *d_out) {
    BZK_ENTER(ctx);
    if (n && !d_out) return BZK_ERR_BAD_ARG;
    return random_g2(ctx, seed, n, (uint8_t *)d_out);
}
int32_t bzk_fr_random_dev(bzk_ctx *ctx, uint64_t seed, size_t n, void *d_out) {
    BZK_ENTER(ctx);
    if (n && !d_out) return BZK_ERR_BAD_ARG;
    return random_fr(ctx, seed, n, (Fr *)d_out);
}
int32_t bzk_fr_binop_dev(bzk_ctx *ctx, int32_t op, const void *d_a, const void *d_b, void *d_out, size_t n) {
    BZK_ENTER(ctx);
    if (op < 0 || op > 2 || (n && (!d_a || !d_b || !d_out))) return BZK_ERR_BAD_ARG;
    if (n == 0) return BZK_OK;
    k_fr_binop<<<div_up(n, 256), 256, 0, ctx->stream>>>(op, (const Fr *)d_a, (const Fr *)d_b, (Fr *)d_out, n);
    BZK_LAUNCHED(ctx);
    return BZK_OK;
}
int32_t bzk_fp_mul_dev(bzk_ctx *ctx, const void *d_a, const void *d_b, void *d_out, size_t n) {
    BZK_ENTER(ctx);
    if (n && (!d_a || !d_b || !d_out)) return BZK_ERR_BAD_ARG;
    if (n == 0) return BZK_OK;
    k_fp_mul<<<div_up(n, 256), 256, 0, ctx->stream>>>((const Fp *)d_a, (const Fp *)d_b, (Fp *)d_out, n);
    BZK_LAUNCHED(ctx);
    return BZK_OK;
}

}  // extern "C"
