// bazuka_b200 — Groth16 prover driver: R1CS evaluation, quotient polynomial, the five MSMs and the
// (r, s) blinding tail.
//
// GPU replacement for bellman 0.14.0 `groth16::prover::create_proof` (un-vendored crate; the
// reference reaches it from /root/reference/src/mpn/circuits/test.rs:135,175,215 and every gadget
// test; in production the call sits in the external prover that answers `MpnWork`,
// /root/reference/src/mpn/mod.rs:264-295).  Same dataflow as bellman:
//   a,b,c = <A_j,z>, <B_j,z>, <C_j,z> per constraint (+ the appended `Input(i) * 0 = 0` rows)
//   h     = first m-1 coefficients of icoset_fft((coset_fft(ifft a) * coset_fft(ifft b)
//           - coset_fft(ifft c)) / Z)
//   sums  : h*H, aux*L, [inputs ++ aux|A-density]*A, [inputs|B-density ++ aux|B-density]*B1, same*B2
//   A = alpha + r delta + a_sum ; B = beta + s delta + b2_sum ;
//   C = s a_sum + r b1_sum + r s delta + s alpha + r beta + h_sum + l_sum
// What is different: the constraint system is a device-resident CSR triple evaluated by an SpMV
// kernel instead of re-synthesising the circuit per proof; density trackers become index lists
// built once at upload; all vectors stay in HBM between stages.
#include "common.cuh"
#include "r1cs_blocked.cuh"
#include <algorithm>
#include <future>

namespace bzk {
int32_t precompute_g1(bzk_ctx *ctx, bzk_g1_bases *b, uint32_t max_levels);
int32_t precompute_g2(bzk_ctx *ctx, bzk_g2_bases *b, uint32_t max_levels);
int32_t groth16_h_launch(bzk_ctx *ctx, Fr *a, Fr *b, Fr *c, uint32_t log_n);
int32_t groth16_to_coset_launch(bzk_ctx *ctx, Fr *v, uint32_t log_n);
int32_t msm_g1_enqueue(bzk_ctx *ctx, cudaStream_t st, void **ws, size_t *ws_bytes, StreamPipe *pipe, const BasesRef<Fp> &d_bases, const Fr *d_scalars,
                       size_t n, void *h_win, MsmPlan *plan);
int32_t msm_g2_enqueue(bzk_ctx *ctx, cudaStream_t st, void **ws, size_t *ws_bytes, StreamPipe *pipe, const BasesRef<Fp2> &d_bases, const Fr *d_scalars,
                       size_t n, void *h_win, MsmPlan *plan);
void msm_g1_finish(const MsmPlan *plan, const void *h_win, bzk_g1_affine *out);
void msm_g2_finish(const MsmPlan *plan, const void *h_win, bzk_g2_affine *out);

struct DevCsr {
    uint64_t *rowptr = nullptr;
    uint32_t *col = nullptr;
    Fr *val = nullptr;
    uint64_t nnz = 0;
};
// a HostColList on the device
struct DevColList {
    uint64_t n = 0;
    uint32_t *col = nullptr, *row = nullptr;
    uint64_t *ptr = nullptr;
    Fr *val = nullptr;
};
// a HostBlockedT on the device: one side's transposed pieces, for bzk_r1cs_columns_dev
struct DevBlockedT {
    uint64_t span = 0;
    uint64_t *s_ptr = nullptr;
    uint32_t *s_row = nullptr;
    Fr *s_val = nullptr;
    DevColList shared, fixed;
};
}  // namespace bzk

// m[s] holds the stored rows: all ncons of them, or, for a blocked handle, head | template | tail (r1cs_blocked.cuh)
struct bzk_r1cs {
    uint64_t num_inputs = 0, num_aux = 0, ncons = 0;
    uint32_t log_m = 0;
    bzk::DevCsr m[3];
    uint32_t *d_a_idx = nullptr, *d_b_idx = nullptr;  // indices into z for the A / B sums
    uint64_t a_len = 0, b_len = 0;
    bool blocked = false;
    bzk::BlockedShape shape;
    bzk::DevBlockedT t[3];
    std::vector<void *> extra;  // the device arrays of t[]
};

namespace bzk {

// one thread per constraint row: out[row] = sum_k val[k] * z[col[k]]
__global__ void __launch_bounds__(256) k_csr_spmv(const uint64_t *__restrict__ rowptr, const uint32_t *__restrict__ col,
                                                  const Fr *__restrict__ val, uint64_t nrows, const Fr *__restrict__ z,
                                                  Fr *__restrict__ out) {
    const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= nrows) return;
    Fr acc = Fr::zero();
    const uint64_t k1 = rowptr[r + 1];
    for (uint64_t k = rowptr[r]; k < k1; k++) acc = acc + load_vec(val + k) * load_vec(z + col[k]);
    store_vec(out + r, acc);
}
__global__ void __launch_bounds__(256) k_gather_fr(const Fr *__restrict__ z, const uint32_t *__restrict__ idx, uint64_t n, Fr *__restrict__ out) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    store_vec(out + i, load_vec(z + idx[i]));
}
// count rows with a*b != c
__global__ void __launch_bounds__(256) k_check_sat(const Fr *__restrict__ a, const Fr *__restrict__ b, const Fr *__restrict__ c, uint64_t n, uint32_t *bad) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (load_vec(a + i) * load_vec(b + i) != load_vec(c + i)) atomicAdd(bad, 1u);
}
__global__ void __launch_bounds__(128) k_fixed_base_g1(G1Affine base, const Fr *__restrict__ k_mont, size_t n, uint8_t *__restrict__ out) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Fr k = load_vec(k_mont + i).from_mont();
    store_g1_image(out + i * 104, scalar_mul(base, k.l).to_affine());
}
__global__ void __launch_bounds__(64) k_fixed_base_g2(G2Affine base, const Fr *__restrict__ k_mont, size_t n, uint8_t *__restrict__ out) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Fr k = load_vec(k_mont + i).from_mont();
    store_g2_image(out + i * 200, scalar_mul(base, k.l).to_affine());
}

// one thread per logical row of a blocked R1CS; the template rows stay in L2 while the copies read them
__global__ void __launch_bounds__(256) k_blocked_spmv(BlockedShape b, const uint64_t *__restrict__ rowptr, const uint32_t *__restrict__ col,
                                                      const Fr *__restrict__ val, uint64_t nrows, const Fr *__restrict__ z, Fr *__restrict__ out) {
    const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= nrows) return;
    store_vec(out + r, blocked_row_dot(b, rowptr, col, val, r, z));
}
// the transposed product's passes (r1cs_blocked.cuh): every column's slot part (0 below var_lo), the per-row sums over the
// copies, then the shared and the head / tail lists added to the columns they name
__global__ void __launch_bounds__(256) k_blocked_slot_cols(BlockedShape b, uint64_t span, const uint64_t *__restrict__ s_ptr,
                                                           const uint32_t *__restrict__ s_row, const Fr *__restrict__ s_val,
                                                           const Fr *__restrict__ lag, uint64_t nv, Fr *__restrict__ out) {
    const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= nv) return;
    store_vec(out + j, blocked_slot_column(b, span, s_ptr, s_row, s_val, lag, j));
}
__global__ void __launch_bounds__(256) k_blocked_rowsum(BlockedShape b, const Fr *__restrict__ lag, Fr *__restrict__ sums) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= b.tmpl_rows) return;
    store_vec(sums + t, blocked_tmpl_rowsum(b, lag, t));
}
__global__ void __launch_bounds__(256) k_col_list_add(uint64_t n, const uint32_t *__restrict__ col, const uint64_t *__restrict__ ptr,
                                                      const uint32_t *__restrict__ row, const Fr *__restrict__ val, const Fr *__restrict__ w,
                                                      Fr *__restrict__ out) {
    const uint64_t u = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= n) return;
    Fr *o = out + col[u];
    store_vec(o, load_vec(o) + col_list_dot(ptr, row, val, w, u));
}
// k_fixed_base_g1 / _g2 with the packed point stored into a resident vector
__global__ void __launch_bounds__(128) k_fixed_base_packed_g1(G1Affine base, const Fr *__restrict__ k_mont, size_t n, G1Affine *__restrict__ out) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Fr k = load_vec(k_mont + i).from_mont();
    store_vec(out + i, scalar_mul(base, k.l).to_affine());
}
__global__ void __launch_bounds__(64) k_fixed_base_packed_g2(G2Affine base, const Fr *__restrict__ k_mont, size_t n, G2Affine *__restrict__ out) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Fr k = load_vec(k_mont + i).from_mont();
    store_vec(out + i, scalar_mul(base, k.l).to_affine());
}

static int32_t upload_csr(bzk_ctx *ctx, DevCsr &d, uint64_t nrows, const uint64_t *rp, const uint32_t *col, const bzk_fr *val) {
    d.nnz = rp[nrows];
    BZK_CUDA(ctx, cudaMalloc(&d.rowptr, (nrows + 1) * sizeof(uint64_t)));
    BZK_CUDA(ctx, cudaMalloc(&d.col, (d.nnz ? d.nnz : 1) * sizeof(uint32_t)));
    BZK_CUDA(ctx, cudaMalloc(&d.val, (d.nnz ? d.nnz : 1) * sizeof(Fr)));
    BZK_CUDA(ctx, cudaMemcpyAsync(d.rowptr, rp, (nrows + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, ctx->stream));
    BZK_CUDA(ctx, cudaMemcpyAsync(d.col, col, d.nnz * sizeof(uint32_t), cudaMemcpyHostToDevice, ctx->stream));
    BZK_CUDA(ctx, cudaMemcpyAsync(d.val, val, d.nnz * sizeof(Fr), cudaMemcpyHostToDevice, ctx->stream));
    return BZK_OK;
}
// a host vector copied into a new device array that the handle frees
template <class T>
static int32_t upload_extra(bzk_ctx *ctx, bzk_r1cs *r, const std::vector<T> &v, T **out) {
    BZK_CUDA(ctx, cudaMalloc(out, (v.size() ? v.size() : 1) * sizeof(T)));
    r->extra.push_back(*out);
    BZK_CUDA(ctx, cudaMemcpyAsync(*out, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice, ctx->stream));
    return BZK_OK;
}
static int32_t upload_col_list(bzk_ctx *ctx, bzk_r1cs *r, const HostColList &h, DevColList &d) {
    d.n = h.col.size();
    BZK_TRY(upload_extra(ctx, r, h.col, &d.col));
    BZK_TRY(upload_extra(ctx, r, h.ptr, &d.ptr));
    BZK_TRY(upload_extra(ctx, r, h.row, &d.row));
    return upload_extra(ctx, r, h.val, &d.val);
}
static int32_t upload_density(bzk_ctx *ctx, bzk_r1cs *r, const std::vector<uint32_t> &a_idx, const std::vector<uint32_t> &b_idx) {
    r->a_len = a_idx.size(); r->b_len = b_idx.size();
    BZK_CUDA(ctx, cudaMalloc(&r->d_a_idx, (a_idx.size() + 1) * 4));
    BZK_CUDA(ctx, cudaMalloc(&r->d_b_idx, (b_idx.size() + 1) * 4));
    BZK_CUDA(ctx, cudaMemcpyAsync(r->d_a_idx, a_idx.data(), a_idx.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
    BZK_CUDA(ctx, cudaMemcpyAsync(r->d_b_idx, b_idx.data(), b_idx.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
    return BZK_OK;
}
static void free_r1cs(bzk_r1cs *r) {
    for (auto &m : r->m) { if (m.rowptr) cudaFree(m.rowptr); if (m.col) cudaFree(m.col); if (m.val) cudaFree(m.val); }
    for (void *p : r->extra) cudaFree(p);
    if (r->d_a_idx) cudaFree(r->d_a_idx);
    if (r->d_b_idx) cudaFree(r->d_b_idx);
    delete r;
}

// ---- the prover's stages; the C entry points below are compositions of them -------------------------------------------

// the four sums a proof is assembled from (wire images)
struct Groth16Partials {
    bzk_g1_affine a, b1, hl;
    bzk_g2_affine b2;
};

// this handle's slice [lo, lo + n) of the terms of each sum: all of them when world == 1, else the shard's
struct Slices {
    uint64_t h_lo, h_n, l_lo, l_n, a_lo, a_n, b_lo, b_n;
};
static int32_t shard_slices(const bzk_groth16_params *pk, const bzk_r1cs *cs, Slices *s) {
    auto lo_of = [&](uint64_t len) { return len * pk->rank / pk->world; };
    auto cnt_of = [&](uint64_t len) { return len * (pk->rank + 1) / pk->world - lo_of(len); };
    const uint64_t h_len = ((uint64_t)1 << cs->log_m) - 1;
    *s = {lo_of(h_len), cnt_of(h_len), lo_of(cs->num_aux), cnt_of(cs->num_aux), lo_of(cs->a_len), cnt_of(cs->a_len), lo_of(cs->b_len), cnt_of(cs->b_len)};
    // a whole key's h may be longer than the domain needs; a shard's vectors are exactly its slices
    if ((pk->world == 1 ? pk->h->n < s->h_n : pk->h->n != s->h_n) || pk->l->n != s->l_n || pk->a->n != s->a_n || pk->b1->n != s->b_n ||
        pk->b2->n != s->b_n)
        return BZK_ERR_BAD_ARG;
    return BZK_OK;
}

// the staging arena: z | a, b, c evaluations (domain size) | the gathered A / B scalars | unsatisfied-row count
struct Stage {
    Fr *z, *ev[3], *gs_a, *gs_b;
    uint32_t *bad;
};
static int32_t stage_arena(bzk_ctx *ctx, const bzk_r1cs *cs, Stage *sg) {
    const uint64_t m = (uint64_t)1 << cs->log_m, gmax = std::max<uint64_t>(std::max(cs->a_len, cs->b_len), 1);
    auto carve = [&](void *base) {
        Carver cv(base);
        sg->z = cv.take<Fr>(cs->num_inputs + cs->num_aux);
        for (Fr *&e : sg->ev) e = cv.take<Fr>(m);
        sg->gs_a = cv.take<Fr>(gmax);
        sg->gs_b = cv.take<Fr>(gmax);
        sg->bad = cv.take<uint32_t>(4);
        return cv.used();
    };
    BZK_TRY(ensure_ws(ctx, &ctx->stage, &ctx->stage_bytes, carve(nullptr)));
    carve(ctx->stage);
    return BZK_OK;
}

// mark k of bzk_groth16_stage_ms, recorded on stream s when timing is on
static void g16_mark(bzk_ctx *ctx, int k, cudaStream_t s) {
    if (!ctx->timing) return;
    if (!ctx->g16_ev[k]) cudaEventCreate(&ctx->g16_ev[k]);
    cudaEventRecord(ctx->g16_ev[k], s);
}

// Starts a proof on the context (an open shard_begin is abandoned): z into the arena from `inputs` / `aux` (kind: host
// images or already on the device), then the SpMVs into the evaluation vectors ev[s] that are not null.  Rows >= ncons
// are the Input(i) * 0 = 0 rows appended to A, then zero padding.  With `check`, rows where a * b != c are refused.
static int32_t witness_side(bzk_ctx *ctx, const bzk_r1cs *cs, const Stage &sg, const bzk_fr *inputs, const bzk_fr *aux, cudaMemcpyKind kind,
                            Fr *const ev[3], bool check) {
    cudaStream_t st = ctx->stream;
    const uint64_t ni = cs->num_inputs, m = (uint64_t)1 << cs->log_m;
    ctx->split_open = false;
    ctx->g16_valid = false;
    g16_mark(ctx, 0, st);
    BZK_CUDA(ctx, cudaMemcpyAsync(sg.z, inputs, ni * sizeof(Fr), kind, st));
    if (cs->num_aux) BZK_CUDA(ctx, cudaMemcpyAsync(sg.z + ni, aux, cs->num_aux * sizeof(Fr), kind, st));
    for (int s = 0; s < 3; s++) {
        if (!ev[s]) continue;
        BZK_CUDA(ctx, cudaMemsetAsync(ev[s] + cs->ncons, 0, (m - cs->ncons) * sizeof(Fr), st));
        if (cs->ncons) {
            if (cs->blocked)
                k_blocked_spmv<<<div_up(cs->ncons, 256), 256, 0, st>>>(cs->shape, cs->m[s].rowptr, cs->m[s].col, cs->m[s].val, cs->ncons, sg.z, ev[s]);
            else
                k_csr_spmv<<<div_up(cs->ncons, 256), 256, 0, st>>>(cs->m[s].rowptr, cs->m[s].col, cs->m[s].val, cs->ncons, sg.z, ev[s]);
            BZK_LAUNCHED(ctx);
        }
    }
    if (ev[0]) BZK_CUDA(ctx, cudaMemcpyAsync(ev[0] + cs->ncons, sg.z, ni * sizeof(Fr), cudaMemcpyDeviceToDevice, st));
    if (!check || !cs->ncons) return BZK_OK;
    BZK_CUDA(ctx, cudaMemsetAsync(sg.bad, 0, 4, st));
    k_check_sat<<<div_up(cs->ncons, 256), 256, 0, st>>>(ev[0], ev[1], ev[2], cs->ncons, sg.bad);
    BZK_LAUNCHED(ctx);
    uint32_t bad = 0;
    BZK_CUDA(ctx, cudaMemcpyAsync(&bad, sg.bad, 4, cudaMemcpyDeviceToHost, st));
    BZK_CUDA(ctx, cudaStreamSynchronize(st));
    if (bad) {
        snprintf(ctx->err, sizeof ctx->err, "%u constraints unsatisfied by the witness", bad);
        return BZK_ERR_UNSAT;
    }
    return BZK_OK;
}

// one sum's window sums on the host (sized for G2); the pinned block holds five, in the order h, l, a, b_g1, b_g2
constexpr size_t kWinBytes = kMaxWinPoints * sizeof(G2Xyzz);

// The five sums are independent once z is on the device (h additionally needs the quotient): the gathers and the l, a,
// b_g1, b_g2 sums run on side streams with their own arenas, behind what the main stream has enqueued so far, while the
// main stream goes on to the quotient and the h sum.  So the latency-bound phases of one MSM (bucket reduction, side-list
// folding) overlap the throughput-bound phases of the others.  A sum over a host-resident vector streams it through its own
// pipe (ctx->pipe[k + 1]); its first chunks are copied at once, not behind aux_ev[0], since the bases do not depend on the
// witness.
static int32_t witness_sums(bzk_ctx *ctx, const bzk_groth16_params *pk, const bzk_r1cs *cs, const Stage &sg, const Slices &sl) {
    for (int k = 0; k < 4; k++)
        if (!ctx->aux_stream[k]) BZK_CUDA(ctx, cudaStreamCreateWithFlags(&ctx->aux_stream[k], cudaStreamNonBlocking));
    for (int k = 0; k < 3; k++)
        if (!ctx->aux_ev[k]) BZK_CUDA(ctx, cudaEventCreateWithFlags(&ctx->aux_ev[k], cudaEventDisableTiming));
    if (ctx->pinned_bytes < 5 * kWinBytes) {
        if (ctx->pinned) cudaFreeHost(ctx->pinned);
        ctx->pinned = nullptr;
        BZK_CUDA(ctx, cudaHostAlloc(&ctx->pinned, 5 * kWinBytes, cudaHostAllocDefault));
        ctx->pinned_bytes = 5 * kWinBytes;
    }
    char *hw = (char *)ctx->pinned;
    MsmPlan *plan = ctx->g16_plan;
    const uint64_t ni = cs->num_inputs;
    cudaStream_t st = ctx->stream, s_l = ctx->aux_stream[0], s_a = ctx->aux_stream[1], s_b1 = ctx->aux_stream[2], s_b2 = ctx->aux_stream[3];
    g16_mark(ctx, 1, st);
    BZK_CUDA(ctx, cudaEventRecord(ctx->aux_ev[0], st));  // z and the evaluations are enqueued behind this point
    BZK_CUDA(ctx, cudaStreamWaitEvent(s_l, ctx->aux_ev[0], 0));
    BZK_CUDA(ctx, cudaStreamWaitEvent(s_a, ctx->aux_ev[0], 0));
    BZK_CUDA(ctx, cudaStreamWaitEvent(s_b1, ctx->aux_ev[0], 0));
    BZK_TRY(msm_g1_enqueue(ctx, s_l, &ctx->aux_ws[0], &ctx->aux_ws_bytes[0], &ctx->pipe[1], bases_ref(pk->l), sg.z + ni + sl.l_lo, sl.l_n, hw + 1 * kWinBytes, &plan[1]));
    k_gather_fr<<<div_up(cs->a_len, 256), 256, 0, s_a>>>(sg.z, cs->d_a_idx, cs->a_len, sg.gs_a);
    BZK_LAUNCHED(ctx);
    BZK_TRY(msm_g1_enqueue(ctx, s_a, &ctx->aux_ws[1], &ctx->aux_ws_bytes[1], &ctx->pipe[2], bases_ref(pk->a), sg.gs_a + sl.a_lo, sl.a_n, hw + 2 * kWinBytes, &plan[2]));
    if (cs->b_len) {
        k_gather_fr<<<div_up(cs->b_len, 256), 256, 0, s_b1>>>(sg.z, cs->d_b_idx, cs->b_len, sg.gs_b);
        BZK_LAUNCHED(ctx);
    }
    BZK_CUDA(ctx, cudaEventRecord(ctx->aux_ev[1], s_b1));
    BZK_CUDA(ctx, cudaStreamWaitEvent(s_b2, ctx->aux_ev[1], 0));
    BZK_TRY(msm_g1_enqueue(ctx, s_b1, &ctx->aux_ws[2], &ctx->aux_ws_bytes[2], &ctx->pipe[3], bases_ref(pk->b1), sg.gs_b + sl.b_lo, sl.b_n, hw + 3 * kWinBytes, &plan[3]));
    BZK_TRY(msm_g2_enqueue(ctx, s_b2, &ctx->aux_ws[3], &ctx->aux_ws_bytes[3], &ctx->pipe[4], bases_ref(pk->b2), sg.gs_b + sl.b_lo, sl.b_n, hw + 4 * kWinBytes, &plan[4]));
    for (int k = 0; k < 4; k++) g16_mark(ctx, 4 + k, ctx->aux_stream[k]);
    return BZK_OK;
}

// the h sum over n quotient coefficients at src, on the main stream
static int32_t h_sum(bzk_ctx *ctx, const bzk_groth16_params *pk, const Fr *src, uint64_t n) {
    BZK_TRY(msm_g1_enqueue(ctx, ctx->stream, &ctx->ws, &ctx->ws_bytes, &ctx->pipe[0], bases_ref(pk->h), src, n, ctx->pinned, &ctx->g16_plan[0]));
    g16_mark(ctx, 3, ctx->stream);
    return BZK_OK;
}

// Waits for the main stream and the four side streams, then folds the five window sets into the four sums.  The folds
// are independent sub-millisecond jobs: they run on host threads instead of back to back.
static int32_t collect(bzk_ctx *ctx, bzk_g1_affine *a_sum, bzk_g1_affine *b1_sum, bzk_g2_affine *b2_sum, bzk_g1_affine *hl_sum) {
    BZK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    for (int k = 0; k < 4; k++) BZK_CUDA(ctx, cudaStreamSynchronize(ctx->aux_stream[k]));
    if (ctx->timing) {
        for (int k = 1; k < 8; k++) cudaEventElapsedTime(&ctx->g16_ms[k], ctx->g16_ev[0], ctx->g16_ev[k]);
        ctx->g16_ms[0] = 0;
        ctx->g16_valid = true;
    }
    const MsmPlan *plan = ctx->g16_plan;
    const char *hw = (const char *)ctx->pinned;
    bzk_g1_affine h, l;
    auto f_b2 = std::async(std::launch::async, [&] { msm_g2_finish(&plan[4], hw + 4 * kWinBytes, b2_sum); });
    auto f_a = std::async(std::launch::async, [&] { msm_g1_finish(&plan[2], hw + 2 * kWinBytes, a_sum); });
    auto f_b1 = std::async(std::launch::async, [&] { msm_g1_finish(&plan[3], hw + 3 * kWinBytes, b1_sum); });
    auto f_l = std::async(std::launch::async, [&] { msm_g1_finish(&plan[1], hw + 1 * kWinBytes, &l); });
    msm_g1_finish(&plan[0], hw, &h);
    f_l.get();
    G1Xyzz hl = G1Xyzz::from_affine(from_wire(&h));
    hl.madd(from_wire(&l));
    to_wire(hl_sum, hl.to_affine());
    f_b2.get(); f_a.get(); f_b1.get();
    return BZK_OK;
}

// everything a proof enqueues for one witness: z and the three evaluations (checked if asked), the four witness sums on
// the side streams, the quotient and the h sum on the main stream
static int32_t enqueue_proof(bzk_ctx *ctx, const bzk_groth16_params *pk, const bzk_r1cs *cs, const bzk_fr *inputs, const bzk_fr *aux,
                             cudaMemcpyKind kind, bool check) {
    Slices sl;
    Stage sg;
    BZK_TRY(shard_slices(pk, cs, &sl));
    BZK_TRY(stage_arena(ctx, cs, &sg));
    BZK_TRY(witness_side(ctx, cs, sg, inputs, aux, kind, sg.ev, check));
    BZK_TRY(witness_sums(ctx, pk, cs, sg, sl));
    BZK_TRY(groth16_h_launch(ctx, sg.ev[0], sg.ev[1], sg.ev[2], cs->log_m));  // a <- the quotient's coefficients
    g16_mark(ctx, 2, ctx->stream);
    return h_sum(ctx, pk, sg.ev[0] + sl.h_lo, sl.h_n);
}

// bellman `create_proof`'s last lines, from the key's points, (r, s) and the four sums:
//   A = r delta1 + alpha1 + a;  B = s delta2 + beta2 + b2;  C = rs delta1 + s alpha1 + r beta1 + s a + r b1 + (h + l)
// `sums` fills in the four sums (it may wait for the GPU, or fail); the terms without them are computed meanwhile.
template <class SumsFn>
static int32_t proof_tail(const G1Affine &alpha1, const G1Affine &beta1, const G2Affine &beta2, const G1Affine &delta1, const G2Affine &delta2,
                          const bzk_fr *r_mont, const bzk_fr *s_mont, SumsFn sums, bzk_g1_affine *proof_a, bzk_g2_affine *proof_b,
                          bzk_g1_affine *proof_c) {
    Fr r, s;
    memcpy(r.l, r_mont, 32);
    memcpy(s.l, s_mont, 32);
    const Fr rs = (r * s).from_mont(), rc = r.from_mont(), sc = s.from_mont();
    auto f_b = std::async(std::launch::async, [&] {
        G2Xyzz t = scalar_mul(delta2, sc.l);
        t.madd(beta2);
        return t;
    });
    auto f_c = std::async(std::launch::async, [&] {
        G1Xyzz t = scalar_mul(delta1, rs.l);
        t.add(scalar_mul(alpha1, sc.l));
        t.add(scalar_mul(beta1, rc.l));
        return t;
    });
    G1Xyzz ga = scalar_mul(delta1, rc.l);
    ga.madd(alpha1);
    Groth16Partials p;
    BZK_TRY(sums(&p));
    const G1Affine a = from_wire(&p.a);
    auto f_sa = std::async(std::launch::async, [&] { return scalar_mul(a, sc.l); });
    const G1Xyzz rb1 = scalar_mul(from_wire(&p.b1), rc.l);
    ga.madd(a);
    G1Xyzz gc = f_c.get();
    gc.add(f_sa.get());
    gc.add(rb1);
    gc.madd(from_wire(&p.hl));
    G2Xyzz gb = f_b.get();
    gb.madd(from_wire(&p.b2));
    to_wire(proof_a, ga.to_affine());
    to_wire(proof_b, gb.to_affine());
    to_wire(proof_c, gc.to_affine());
    return BZK_OK;
}

// a whole proof; kind: where `inputs` / `aux` live (host images, or already resident, e.g. written by bzk_witness_run_dev)
static int32_t whole_proof(bzk_ctx *ctx, const bzk_groth16_params *pk, const bzk_r1cs *cs, const bzk_fr *inputs, const bzk_fr *aux,
                           cudaMemcpyKind kind, const bzk_fr *r_mont, const bzk_fr *s_mont, int32_t check_satisfied, bzk_g1_affine *proof_a,
                           bzk_g2_affine *proof_b, bzk_g1_affine *proof_c) {
    if (!ctx || !pk || !cs || !inputs || (cs->num_aux && !aux) || !r_mont || !s_mont || !proof_a || !proof_b || !proof_c) return BZK_ERR_BAD_ARG;
    if (pk->world != 1) return BZK_ERR_BAD_ARG;  // a shard can only produce partial sums
    BZK_CUDA(ctx, cudaSetDevice(ctx->device));
    BZK_TRY(enqueue_proof(ctx, pk, cs, inputs, aux, kind, check_satisfied != 0));
    return proof_tail(pk->alpha_g1, pk->beta_g1, pk->beta_g2, pk->delta_g1, pk->delta_g2, r_mont, s_mont,
                      [&](Groth16Partials *p) { return collect(ctx, &p->a, &p->b1, &p->b2, &p->hl); }, proof_a, proof_b, proof_c);
}

}  // namespace bzk

using namespace bzk;

extern "C" {

int32_t bzk_r1cs_upload(bzk_ctx *ctx, uint64_t num_inputs, uint64_t num_aux, uint64_t ncons,
                        const uint64_t *a_rp, const uint32_t *a_col, const bzk_fr *a_val,
                        const uint64_t *b_rp, const uint32_t *b_col, const bzk_fr *b_val,
                        const uint64_t *c_rp, const uint32_t *c_col, const bzk_fr *c_val, bzk_r1cs **out) {
    if (!ctx || !out || !a_rp || !b_rp || !c_rp || num_inputs == 0) return BZK_ERR_BAD_ARG;
    BZK_CUDA(ctx, cudaSetDevice(ctx->device));
    *out = nullptr;
    const uint64_t nv = num_inputs + num_aux;
    if (nv >= (1ull << 32)) return BZK_ERR_BAD_ARG;
    const uint64_t *rp[3] = {a_rp, b_rp, c_rp};
    const uint32_t *cl[3] = {a_col, b_col, c_col};
    const bzk_fr *vl[3] = {a_val, b_val, c_val};
    uint32_t log_m = 0;
    while (log_m <= 28 && (1ull << log_m) < ncons + num_inputs) log_m++;
    if (log_m > 28) return BZK_ERR_BAD_ARG;
    // density (bellman `eval`: terms with a zero coefficient are skipped): A over aux only (all inputs are always
    // present), B over inputs and aux; found in the same pass over the terms that checks their columns and coefficients
    std::vector<uint8_t> a_d(nv, 0), b_d(nv, 0);
    uint8_t *pres[3] = {a_d.data(), b_d.data(), nullptr};
    for (int s = 0; s < 3; s++) {
        if (rp[s][0] != 0) return BZK_ERR_BAD_ARG;
        for (uint64_t j = 0; j < ncons; j++) if (rp[s][j + 1] < rp[s][j]) return BZK_ERR_BAD_ARG;
        if (rp[s][ncons] && (!cl[s] || !vl[s])) return BZK_ERR_BAD_ARG;
        for (uint64_t k = 0; k < rp[s][ncons]; k++) {
            const uint64_t *v = vl[s][k].l;
            if (cl[s][k] >= nv || !fr_image_canonical(v)) return BZK_ERR_BAD_ARG;
            if (pres[s] && (v[0] | v[1] | v[2] | v[3])) pres[s][cl[s][k]] = 1;
        }
    }
    bzk_r1cs *r = new (std::nothrow) bzk_r1cs();
    if (!r) return BZK_ERR_OOM;
    r->num_inputs = num_inputs; r->num_aux = num_aux; r->ncons = ncons; r->log_m = log_m;
    std::vector<uint32_t> a_idx, b_idx;
    density_lists(num_inputs, a_d, b_d, a_idx, b_idx);
    int32_t st = BZK_OK;
    for (int s = 0; s < 3 && st == BZK_OK; s++) st = upload_csr(ctx, r->m[s], ncons, rp[s], cl[s], vl[s]);
    if (st == BZK_OK) st = upload_density(ctx, r, a_idx, b_idx);
    if (st == BZK_OK) {
        cudaError_t e = cudaStreamSynchronize(ctx->stream);
        if (e != cudaSuccess) st = set_cuda_err(ctx, e, "r1cs upload", __FILE__, __LINE__);
    }
    if (st != BZK_OK) { free_r1cs(r); return st; }
    *out = r;
    return BZK_OK;
}

/* include/bzk.h: the stored rows head | template | tail per side; validated on the host before anything is allocated */
int32_t bzk_r1cs_upload_blocked(bzk_ctx *ctx, uint64_t num_inputs, uint64_t num_aux, uint64_t head_rows, uint64_t tmpl_rows, uint64_t reps,
                                uint64_t tail_rows, uint64_t var_lo, uint64_t var_stride, const uint64_t *const rowptr[3], const uint32_t *const col[3],
                                const bzk_fr *const val[3], bzk_r1cs **out) {
    if (!ctx || !out || !rowptr || !col || !val || num_inputs == 0) return BZK_ERR_BAD_ARG;
    *out = nullptr;
    const uint64_t nv = num_inputs + num_aux;
    if (nv < num_inputs || nv > (1ull << 32)) return BZK_ERR_BAD_ARG;
    BlockedShape b;
    b.head_rows = head_rows; b.tmpl_rows = tmpl_rows; b.reps = reps; b.tail_rows = tail_rows; b.var_lo = var_lo; b.var_stride = var_stride;
    // the logical row count must not wrap (and stays far below 2^32: the domain is at most 2^28)
    if (head_rows > (1ull << 32) || tmpl_rows > (1ull << 32) || tail_rows > (1ull << 32) || (tmpl_rows && reps > (1ull << 32) / tmpl_rows))
        return BZK_ERR_BAD_ARG;
    for (int s = 0; s < 3; s++)
        if (!blocked_valid(b, nv, rowptr[s], col[s], val[s])) return BZK_ERR_BAD_ARG;
    const uint64_t ncons = b.rows();
    uint32_t log_m = 0;
    while ((1ull << log_m) < ncons + num_inputs) log_m++;
    if (log_m > 28) return BZK_ERR_BAD_ARG;
    BZK_CUDA(ctx, cudaSetDevice(ctx->device));
    bzk_r1cs *r = new (std::nothrow) bzk_r1cs();
    if (!r) return BZK_ERR_OOM;
    r->num_inputs = num_inputs; r->num_aux = num_aux; r->ncons = ncons; r->log_m = log_m;
    r->blocked = true;
    r->shape = b;
    std::vector<uint8_t> a_d(nv, 0), b_d(nv, 0);
    blocked_presence(b, rowptr[0], col[0], (const Fr *)val[0], a_d);
    blocked_presence(b, rowptr[1], col[1], (const Fr *)val[1], b_d);
    std::vector<uint32_t> a_idx, b_idx;
    density_lists(num_inputs, a_d, b_d, a_idx, b_idx);
    auto upload = [&]() -> int32_t {
        for (int s = 0; s < 3; s++) {
            BZK_TRY(upload_csr(ctx, r->m[s], b.stored_rows(), rowptr[s], col[s], val[s]));
            const HostBlockedT h = blocked_transpose(b, rowptr[s], col[s], (const Fr *)val[s]);
            DevBlockedT &d = r->t[s];
            d.span = h.span;
            BZK_TRY(upload_extra(ctx, r, h.s_ptr, &d.s_ptr));
            BZK_TRY(upload_extra(ctx, r, h.s_row, &d.s_row));
            BZK_TRY(upload_extra(ctx, r, h.s_val, &d.s_val));
            BZK_TRY(upload_col_list(ctx, r, h.shared, d.shared));
            BZK_TRY(upload_col_list(ctx, r, h.fixed, d.fixed));
            BZK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // the host vectors go out of scope
        }
        BZK_TRY(upload_density(ctx, r, a_idx, b_idx));
        BZK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        return BZK_OK;
    };
    const int32_t st = upload();
    if (st != BZK_OK) { free_r1cs(r); return st; }
    *out = r;
    return BZK_OK;
}

/* d_out[j] = sum_row M_side[row][j] * d_lag[row] for every variable j, on the context's stream (blocked handles) */
int32_t bzk_r1cs_columns_dev(bzk_ctx *ctx, const bzk_r1cs *r, uint32_t side, const void *d_lag, void *d_out) {
    if (!ctx || !r || !r->blocked || side > 2 || !d_lag || !d_out) return BZK_ERR_BAD_ARG;
    BZK_CUDA(ctx, cudaSetDevice(ctx->device));
    const BlockedShape &b = r->shape;
    const DevBlockedT &t = r->t[side];
    const Fr *lag = (const Fr *)d_lag;
    Fr *o = (Fr *)d_out;
    const uint64_t nv = r->num_inputs + r->num_aux;
    cudaStream_t st = ctx->stream;
    k_blocked_slot_cols<<<div_up(nv, 256), 256, 0, st>>>(b, t.span, t.s_ptr, t.s_row, t.s_val, lag, nv, o);
    BZK_LAUNCHED(ctx);
    if (t.shared.n) {
        Fr *sums = nullptr;
        BZK_CUDA(ctx, cudaMalloc(&sums, b.tmpl_rows * sizeof(Fr)));
        k_blocked_rowsum<<<div_up(b.tmpl_rows, 256), 256, 0, st>>>(b, lag, sums);
        cudaError_t e = cudaGetLastError();
        if (e == cudaSuccess) {
            ctx->launches++;
            k_col_list_add<<<div_up(t.shared.n, 256), 256, 0, st>>>(t.shared.n, t.shared.col, t.shared.ptr, t.shared.row, t.shared.val, sums, o);
            e = cudaGetLastError();
            ctx->launches++;
        }
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        cudaFree(sums);
        if (e != cudaSuccess) return set_cuda_err(ctx, e, "r1cs columns", __FILE__, __LINE__);
    }
    if (t.fixed.n) {
        k_col_list_add<<<div_up(t.fixed.n, 256), 256, 0, st>>>(t.fixed.n, t.fixed.col, t.fixed.ptr, t.fixed.row, t.fixed.val, lag, o);
        BZK_LAUNCHED(ctx);
    }
    return BZK_OK;
}

int32_t bzk_r1cs_free(bzk_ctx *ctx, bzk_r1cs *r) {
    if (!ctx) return BZK_ERR_BAD_ARG;
    if (!r) return BZK_OK;
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    free_r1cs(r);
    return BZK_OK;
}

int32_t bzk_r1cs_shape(const bzk_r1cs *r, uint64_t out[5]) {
    if (!r || !out) return BZK_ERR_BAD_ARG;
    out[0] = r->log_m;
    out[1] = ((uint64_t)1 << r->log_m) - 1;  // |h|
    out[2] = r->num_aux;                      // |l|
    out[3] = r->a_len;                        // |a|
    out[4] = r->b_len;                        // |b_g1| = |b_g2|
    return BZK_OK;
}

int32_t bzk_csr_spmv_dev(bzk_ctx *ctx, const void *d_rowptr, const void *d_col, const void *d_val, uint64_t nrows, const void *d_vec, void *d_out) {
    if (!ctx || (nrows && (!d_rowptr || !d_vec || !d_out))) return BZK_ERR_BAD_ARG;
    BZK_CUDA(ctx, cudaSetDevice(ctx->device));
    if (nrows == 0) return BZK_OK;
    k_csr_spmv<<<div_up(nrows, 256), 256, 0, ctx->stream>>>((const uint64_t *)d_rowptr, (const uint32_t *)d_col, (const Fr *)d_val, nrows, (const Fr *)d_vec, (Fr *)d_out);
    BZK_LAUNCHED(ctx);
    return BZK_OK;
}

int32_t bzk_g1_fixed_base_mul_dev(bzk_ctx *ctx, const bzk_g1_affine *base, const void *d_scalars, size_t n, void *d_out) {
    if (!ctx || !base || (n && (!d_scalars || !d_out))) return BZK_ERR_BAD_ARG;
    BZK_CUDA(ctx, cudaSetDevice(ctx->device));
    if (n == 0) return BZK_OK;
    k_fixed_base_g1<<<div_up(n, 128), 128, 0, ctx->stream>>>(from_wire(base), (const Fr *)d_scalars, n, (uint8_t *)d_out);
    BZK_LAUNCHED(ctx);
    return BZK_OK;
}
int32_t bzk_g2_fixed_base_mul_dev(bzk_ctx *ctx, const bzk_g2_affine *base, const void *d_scalars, size_t n, void *d_out) {
    if (!ctx || !base || (n && (!d_scalars || !d_out))) return BZK_ERR_BAD_ARG;
    BZK_CUDA(ctx, cudaSetDevice(ctx->device));
    if (n == 0) return BZK_OK;
    k_fixed_base_g2<<<div_up(n, 64), 64, 0, ctx->stream>>>(from_wire(base), (const Fr *)d_scalars, n, (uint8_t *)d_out);
    BZK_LAUNCHED(ctx);
    return BZK_OK;
}

/* k_fixed_base_g1 / _g2 into a new resident vector: bases[i] = [k_i] base, never held as wire images */
int32_t bzk_g1_bases_fixed_base_mul(bzk_ctx *ctx, const bzk_g1_affine *base, const void *d_scalars, size_t n, bzk_g1_bases **out) {
    if (!ctx || !base || !out || (n && !d_scalars)) return BZK_ERR_BAD_ARG;
    *out = nullptr;
    BZK_CUDA(ctx, cudaSetDevice(ctx->device));
    bzk_g1_bases *b = new (std::nothrow) bzk_g1_bases();
    if (!b) return BZK_ERR_OOM;
    b->n = n;
    cudaError_t e = cudaMalloc(&b->d, (n ? n : 1) * sizeof(G1Affine));
    if (e == cudaSuccess && n) {
        k_fixed_base_packed_g1<<<div_up(n, 128), 128, 0, ctx->stream>>>(from_wire(base), (const Fr *)d_scalars, n, b->d);
        ctx->launches++;
        e = cudaGetLastError();
    }
    if (e != cudaSuccess) {
        if (b->d) cudaFree(b->d);
        delete b;
        return set_cuda_err(ctx, e, "g1 fixed-base bases", __FILE__, __LINE__);
    }
    *out = b;
    return BZK_OK;
}
int32_t bzk_g2_bases_fixed_base_mul(bzk_ctx *ctx, const bzk_g2_affine *base, const void *d_scalars, size_t n, bzk_g2_bases **out) {
    if (!ctx || !base || !out || (n && !d_scalars)) return BZK_ERR_BAD_ARG;
    *out = nullptr;
    BZK_CUDA(ctx, cudaSetDevice(ctx->device));
    bzk_g2_bases *b = new (std::nothrow) bzk_g2_bases();
    if (!b) return BZK_ERR_OOM;
    b->n = n;
    cudaError_t e = cudaMalloc(&b->d, (n ? n : 1) * sizeof(G2Affine));
    if (e == cudaSuccess && n) {
        k_fixed_base_packed_g2<<<div_up(n, 64), 64, 0, ctx->stream>>>(from_wire(base), (const Fr *)d_scalars, n, b->d);
        ctx->launches++;
        e = cudaGetLastError();
    }
    if (e != cudaSuccess) {
        if (b->d) cudaFree(b->d);
        delete b;
        return set_cuda_err(ctx, e, "g2 fixed-base bases", __FILE__, __LINE__);
    }
    *out = b;
    return BZK_OK;
}

int32_t bzk_groth16_params_create(bzk_ctx *ctx, const bzk_g1_affine *alpha_g1, const bzk_g1_affine *beta_g1, const bzk_g2_affine *beta_g2,
                                  const bzk_g1_affine *delta_g1, const bzk_g2_affine *delta_g2,
                                  bzk_g1_bases *h, bzk_g1_bases *l, bzk_g1_bases *a, bzk_g1_bases *b_g1, bzk_g2_bases *b_g2,
                                  bzk_groth16_params **out) {
    if (!ctx || !out || !alpha_g1 || !beta_g1 || !beta_g2 || !delta_g1 || !delta_g2 || !h || !l || !a || !b_g1 || !b_g2) return BZK_ERR_BAD_ARG;
    if (b_g1->n != b_g2->n) return BZK_ERR_BAD_ARG;
    bzk_groth16_params *p = new (std::nothrow) bzk_groth16_params();
    if (!p) return BZK_ERR_OOM;
    p->alpha_g1 = from_wire(alpha_g1); p->beta_g1 = from_wire(beta_g1); p->delta_g1 = from_wire(delta_g1);
    p->beta_g2 = from_wire(beta_g2); p->delta_g2 = from_wire(delta_g2);
    p->h = h; p->l = l; p->a = a; p->b1 = b_g1; p->b2 = b_g2;
    *out = p;
    return BZK_OK;
}
int32_t bzk_groth16_params_info(const bzk_groth16_params *p, uint64_t lens[5], bzk_g1_affine *alpha_g1, bzk_g1_affine *beta_g1,
                                bzk_g2_affine *beta_g2, bzk_g1_affine *delta_g1, bzk_g2_affine *delta_g2) {
    if (!p) return BZK_ERR_BAD_ARG;
    if (lens) { lens[0] = p->h->n; lens[1] = p->l->n; lens[2] = p->a->n; lens[3] = p->b1->n; lens[4] = p->b2->n; }
    if (alpha_g1) to_wire(alpha_g1, p->alpha_g1);
    if (beta_g1) to_wire(beta_g1, p->beta_g1);
    if (beta_g2) to_wire(beta_g2, p->beta_g2);
    if (delta_g1) to_wire(delta_g1, p->delta_g1);
    if (delta_g2) to_wire(delta_g2, p->delta_g2);
    return BZK_OK;
}
/* frees the handle and the five base vectors it adopted */
int32_t bzk_groth16_params_free(bzk_ctx *ctx, bzk_groth16_params *p) {
    if (!ctx) return BZK_ERR_BAD_ARG;
    if (!p) return BZK_OK;
    bzk_g1_bases_free(ctx, p->h); bzk_g1_bases_free(ctx, p->l); bzk_g1_bases_free(ctx, p->a); bzk_g1_bases_free(ctx, p->b1);
    bzk_g2_bases_free(ctx, p->b2);
    delete p;
    return BZK_OK;
}

int32_t bzk_groth16_prove(bzk_ctx *ctx, const bzk_groth16_params *pk, const bzk_r1cs *cs, const bzk_fr *inputs, const bzk_fr *aux,
                          const bzk_fr *r_mont, const bzk_fr *s_mont, int32_t check_satisfied,
                          bzk_g1_affine *proof_a, bzk_g2_affine *proof_b, bzk_g1_affine *proof_c) {
    return whole_proof(ctx, pk, cs, inputs, aux, cudaMemcpyHostToDevice, r_mont, s_mont, check_satisfied, proof_a, proof_b, proof_c);
}

int32_t bzk_groth16_prove_dev(bzk_ctx *ctx, const bzk_groth16_params *pk, const bzk_r1cs *cs, const void *d_inputs, const void *d_aux,
                              const bzk_fr *r_mont, const bzk_fr *s_mont, int32_t check_satisfied,
                              bzk_g1_affine *proof_a, bzk_g2_affine *proof_b, bzk_g1_affine *proof_c) {
    return whole_proof(ctx, pk, cs, (const bzk_fr *)d_inputs, (const bzk_fr *)d_aux, cudaMemcpyDeviceToDevice, r_mont, s_mont,
                       check_satisfied, proof_a, proof_b, proof_c);
}

/* milliseconds since the start of the last timed prove call (bzk_ctx_set_timing on) at which: [1] z upload + the three
 * SpMVs (+ satisfiability check) finished, [2] the quotient pipeline (7 NTTs) finished, [3] the h sum finished (main
 * stream), [4..7] the l / a / b_g1 / b_g2 sums finished (side streams, concurrent with the main one).  Returns 1 if valid. */
int32_t bzk_groth16_stage_ms(const bzk_ctx *ctx, float out[8]) {
    if (!ctx || !out) return BZK_ERR_BAD_ARG;
    for (int k = 0; k < 8; k++) out[k] = ctx->g16_ms[k];
    return ctx->g16_valid ? 1 : 0;
}

/* Fixed-base tables for the five base vectors of a key (they never change between proofs): up to `max_levels` levels
 * [2^(c*G*t)] P per base, so that the windows of a scalar share ceil(W/levels) bucket groups — fewer, larger windows and
 * one bucket reduction per group instead of per window.  max_levels = 0 picks the largest count (<= 16) whose tables fit
 * in `mem_fraction_percent` % of the currently free device memory.  Memory: levels x the device vectors' size.  Vectors in
 * host memory stay as they are: they have no tables. */
int32_t bzk_groth16_params_precompute(bzk_ctx *ctx, bzk_groth16_params *p, uint32_t max_levels, uint32_t mem_fraction_percent) {
    if (!ctx || !p) return BZK_ERR_BAD_ARG;
    BZK_CUDA(ctx, cudaSetDevice(ctx->device));
    if (max_levels == 0) {
        size_t free_b = 0, total_b = 0;
        BZK_CUDA(ctx, cudaMemGetInfo(&free_b, &total_b));
        auto dev_n = [](const auto *b) { return b->h ? 0.0 : (double)b->n; };
        const double key_bytes = (dev_n(p->h) + dev_n(p->l) + dev_n(p->a) + dev_n(p->b1)) * sizeof(G1Affine) + dev_n(p->b2) * sizeof(G2Affine);
        const double budget = (double)free_b * (mem_fraction_percent ? mem_fraction_percent : 50) / 100.0;
        uint32_t lv = key_bytes > 0 ? (uint32_t)(budget / key_bytes) + 1 : 16;  // level 0 is already resident
        max_levels = lv > 16 ? 16 : lv;
    }
    if (max_levels <= 1) return BZK_OK;
    for (bzk_g1_bases *b : {p->h, p->l, p->a, p->b1})
        if (!b->h) BZK_TRY(precompute_g1(ctx, b, max_levels));
    if (!p->b2->h) BZK_TRY(precompute_g2(ctx, p->b2, max_levels));
    return BZK_OK;
}

/* the key's five vectors to pinned host memory (bit v of host_mask, order h, l, a, b_g1, b_g2) or to the device (bit
 * clear); the moves to the host go first, so that device memory peaks no higher than before the call */
int32_t bzk_groth16_params_move(bzk_ctx *ctx, bzk_groth16_params *p, uint32_t host_mask) {
    if (!ctx || !p || host_mask > 31) return BZK_ERR_BAD_ARG;
    bzk_g1_bases *g1[4] = {p->h, p->l, p->a, p->b1};
    for (int to_host = 1; to_host >= 0; to_host--) {
        for (int v = 0; v < 4; v++)
            if ((int)((host_mask >> v) & 1) == to_host) BZK_TRY(bzk_g1_bases_move(ctx, g1[v], to_host));
        if ((int)((host_mask >> 4) & 1) == to_host) BZK_TRY(bzk_g2_bases_move(ctx, p->b2, to_host));
    }
    return BZK_OK;
}

int32_t bzk_groth16_params_set_shard(bzk_groth16_params *p, uint32_t rank, uint32_t world) {
    if (!p || world == 0 || rank >= world) return BZK_ERR_BAD_ARG;
    p->rank = rank;
    p->world = world;
    return BZK_OK;
}

int32_t bzk_groth16_prove_partial(bzk_ctx *ctx, const bzk_groth16_params *pk, const bzk_r1cs *cs, const void *inputs, const void *aux,
                                  int32_t witness_on_device, int32_t check_satisfied,
                                  bzk_g1_affine *a_sum, bzk_g1_affine *b1_sum, bzk_g2_affine *b2_sum, bzk_g1_affine *hl_sum) {
    if (!ctx || !pk || !cs || !inputs || (cs->num_aux && !aux) || !a_sum || !b1_sum || !b2_sum || !hl_sum) return BZK_ERR_BAD_ARG;
    BZK_CUDA(ctx, cudaSetDevice(ctx->device));
    BZK_TRY(enqueue_proof(ctx, pk, cs, (const bzk_fr *)inputs, (const bzk_fr *)aux, witness_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice,
                          check_satisfied != 0));
    return collect(ctx, a_sum, b1_sum, b2_sum, hl_sum);
}

/* The sharded schedule with the quotient pipeline split over the ranks (include/bzk.h).  begin: z, the evaluation vectors in
 * `poly_mask` (bit 0 = a, 1 = b, 2 = c) computed into the caller's buffers and taken to the coset, the l / a / b_g1 / b_g2
 * partial sums enqueued on their streams (they keep running while the caller moves vectors between GPUs).  finish: the h sum
 * over this rank's slice of the quotient coefficients, then the four partial sums as bzk_groth16_prove_partial returns them. */
int32_t bzk_groth16_shard_begin(bzk_ctx *ctx, const bzk_groth16_params *pk, const bzk_r1cs *cs, const void *inputs, const void *aux,
                                int32_t witness_on_device, uint32_t poly_mask, void *d_evals[3]) {
    if (!ctx || !pk || !cs || !inputs || (cs->num_aux && !aux) || !d_evals || poly_mask > 7) return BZK_ERR_BAD_ARG;
    Fr *ev[3];
    for (int s = 0; s < 3; s++) {
        const bool mine = (poly_mask >> s) & 1;
        if (mine && !d_evals[s]) return BZK_ERR_BAD_ARG;
        ev[s] = mine ? (Fr *)d_evals[s] : nullptr;
    }
    BZK_CUDA(ctx, cudaSetDevice(ctx->device));
    Slices sl;
    Stage sg;
    BZK_TRY(shard_slices(pk, cs, &sl));
    BZK_TRY(stage_arena(ctx, cs, &sg));
    BZK_TRY(witness_side(ctx, cs, sg, (const bzk_fr *)inputs, (const bzk_fr *)aux, witness_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice,
                         ev, false));
    BZK_TRY(witness_sums(ctx, pk, cs, sg, sl));
    // the pointwise step and the last transform happen on the rank that collects the three vectors (bzk_groth16_h_combine_dev)
    for (Fr *v : ev)
        if (v) BZK_TRY(groth16_to_coset_launch(ctx, v, cs->log_m));
    g16_mark(ctx, 2, ctx->stream);
    BZK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // the caller hands the vectors to its transport next
    ctx->split_open = true;
    return BZK_OK;
}
/* finish leaves the staging arena alone: the side-stream sums started by begin may still be reading z and the gathered
 * scalars from it */
int32_t bzk_groth16_shard_finish(bzk_ctx *ctx, const bzk_groth16_params *pk, const bzk_r1cs *cs, const void *d_h_shard,
                                 bzk_g1_affine *a_sum, bzk_g1_affine *b1_sum, bzk_g2_affine *b2_sum, bzk_g1_affine *hl_sum) {
    if (!ctx || !pk || !cs || !a_sum || !b1_sum || !b2_sum || !hl_sum) return BZK_ERR_BAD_ARG;
    if (!ctx->split_open || (!d_h_shard && pk->h->n)) return BZK_ERR_BAD_ARG;
    BZK_CUDA(ctx, cudaSetDevice(ctx->device));
    Slices sl;
    BZK_TRY(shard_slices(pk, cs, &sl));
    ctx->split_open = false;
    BZK_TRY(h_sum(ctx, pk, (const Fr *)d_h_shard, sl.h_n));
    return collect(ctx, a_sum, b1_sum, b2_sum, hl_sum);
}

/* the tail of bellman `create_proof` from the (summed) answers, on the host (proof_tail) */
int32_t bzk_groth16_finalize(const bzk_g1_affine *alpha_g1, const bzk_g1_affine *beta_g1, const bzk_g2_affine *beta_g2,
                             const bzk_g1_affine *delta_g1, const bzk_g2_affine *delta_g2,
                             const bzk_g1_affine *a_sum, const bzk_g1_affine *b1_sum, const bzk_g2_affine *b2_sum, const bzk_g1_affine *hl_sum,
                             const bzk_fr *r_mont, const bzk_fr *s_mont, bzk_g1_affine *proof_a, bzk_g2_affine *proof_b, bzk_g1_affine *proof_c) {
    if (!alpha_g1 || !beta_g1 || !beta_g2 || !delta_g1 || !delta_g2 || !a_sum || !b1_sum || !b2_sum || !hl_sum || !r_mont || !s_mont ||
        !proof_a || !proof_b || !proof_c)
        return BZK_ERR_BAD_ARG;
    auto sums = [&](Groth16Partials *p) {
        *p = Groth16Partials{*a_sum, *b1_sum, *hl_sum, *b2_sum};
        return (int32_t)BZK_OK;
    };
    return proof_tail(from_wire(alpha_g1), from_wire(beta_g1), from_wire(beta_g2), from_wire(delta_g1), from_wire(delta_g2), r_mont, s_mont, sums,
                      proof_a, proof_b, proof_c);
}

/* 387-byte bincode image of `Groth16Proof {a, b, c}` (/root/reference/src/zk/groth16/mod.rs:33-38) */
int32_t bzk_groth16_proof_bytes(const bzk_g1_affine *a, const bzk_g2_affine *b, const bzk_g1_affine *c, uint8_t out[387]) {
    if (!a || !b || !c || !out) return BZK_ERR_BAD_ARG;
    memcpy(out, a, 97);
    memcpy(out + 97, b, 193);
    memcpy(out + 290, c, 97);
    return BZK_OK;
}

}  // extern "C"
