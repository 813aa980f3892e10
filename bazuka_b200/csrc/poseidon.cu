// bazuka_b200 — batched Poseidon (x^5, t = 2..17) over BLS12-381 Fr.
//
// GPU replacement for `poseidon::poseidon` / `PoseidonState::hash`
// (/root/reference/src/zk/poseidon/mod.rs:24-84): state = [0] ++ inputs, R_F/2 full rounds,
// R_P partial rounds (S-box on lane 0), R_F/2 full rounds, each round = add t round constants
// (consumed sequentially), S-box, dense t x t MDS product; digest = lane 1.  The reference
// serialises all hashing behind a process-global Mutex<LruCache> (/root/reference/src/zk/mod.rs:491-511);
// here one thread owns one hash and a launch processes the whole batch.
//
// Layout: in[n][arity] / out[n] are Montgomery Fr images (32 B = one DRAM sector per element, so
// the strided per-thread reads are sector-exact).  The per-width constant table (round constants,
// then MDS rows) is staged into shared memory once per CTA and read as warp-uniform broadcasts.
// Bound: integer ALU (t=5: 1 888 Fr products per 160 B of traffic) — see DESIGN.md.
#include "common.cuh"
#include "hash_plan.cuh"

namespace bzk {

__device__ __forceinline__ Fr lds_fr(const Fr *s) {
    Fr r;
    const uint4 *p = (const uint4 *)s;
    uint4 a = p[0], b = p[1];
    r.l[0] = a.x; r.l[1] = a.y; r.l[2] = a.z; r.l[3] = a.w;
    r.l[4] = b.x; r.l[5] = b.y; r.l[6] = b.z; r.l[7] = b.w;
    return r;
}

__device__ __forceinline__ Fr pow5(const Fr &x) {
    Fr x2 = x.sqr();
    Fr x4 = x2.sqr();
    return x * x4;
}

// out = sum_k m[k] * s[k] with ONE Montgomery reduction: the 2N-limb products are accumulated
// unreduced (Fe::mul_wide / wide_accumulate) and reduced by N+1 limbs at the end (Fe::redc_wide), which is
// why the MDS rows read here are pre-multiplied by 2^32 at load time.  (64t + 72 limb products per row
// instead of 128t.)
template <int T>
__device__ __forceinline__ Fr mds_row_dot(const Fr *__restrict__ m_scaled, const Fr (&s)[T]) {
    uint32_t acc[17];
#pragma unroll
    for (int i = 0; i < 17; i++) acc[i] = 0;
#pragma unroll
    for (int k = 0; k < T; k++) {
        uint32_t w[16];
        Fr::mul_wide(w, lds_fr(m_scaled + k), s[k]);
        Fr::wide_accumulate(acc, w);
    }
    return Fr::redc_wide(acc);
}

// The constant table of width T (round constants, the MDS matrix, the MDS rows pre-scaled by 2^32) staged into shared
// memory by the whole CTA.
template <int T>
__device__ __forceinline__ void stage_consts(const Fr *__restrict__ consts, uint32_t rf, uint32_t rp, Fr *sc) {
    const uint32_t nconst = T * (rf + rp) + 2 * T * T;
    const uint4 *src = (const uint4 *)consts;
    uint4 *dst = (uint4 *)sc;
    for (uint32_t i = threadIdx.x; i < nconst * 2; i += blockDim.x) dst[i] = src[i];
    __syncthreads();
}

// The permutation on a register-resident state over the staged table: R_F/2 full rounds, R_P partial rounds, R_F/2 full
// rounds; the digest is s[1].
template <int T>
__device__ __forceinline__ void poseidon_rounds(Fr (&s)[T], const Fr *sc, uint32_t rf, uint32_t rp) {
    const Fr *mds = sc + T * (rf + rp) + T * T;  // rows pre-scaled by 2^32 for the lazy row product
    const uint32_t half = rf / 2;
    const Fr *rc = sc;
#pragma unroll 1
    for (uint32_t rnd = 0; rnd < rf + rp; rnd++) {
#pragma unroll
        for (int i = 0; i < T; i++) s[i] = s[i] + lds_fr(rc + i);
        rc += T;
        if (rnd < half || rnd >= half + rp) {
#pragma unroll
            for (int i = 0; i < T; i++) s[i] = pow5(s[i]);
        } else {
            s[0] = pow5(s[0]);
        }
        Fr o[T];
#pragma unroll
        for (int j = 0; j < T; j++) o[j] = mds_row_dot<T>(mds + j * T, s);
#pragma unroll
        for (int i = 0; i < T; i++) s[i] = o[i];
    }
}

// Register-resident state, fully unrolled lanes (T <= 9).
template <int T>
__global__ void __launch_bounds__(128) k_poseidon_reg(const Fr *__restrict__ consts, uint32_t rf, uint32_t rp,
                                                      const Fr *__restrict__ in, size_t n, Fr *__restrict__ out) {
    extern __shared__ uint4 smem_raw[];
    Fr *sc = (Fr *)smem_raw;
    stage_consts<T>(consts, rf, rp, sc);
    size_t h = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (h >= n) return;
    Fr s[T];
    s[0] = Fr::zero();
#pragma unroll
    for (int i = 1; i < T; i++) s[i] = load_vec(in + h * (T - 1) + (i - 1));
    poseidon_rounds<T>(s, sc, rf, rp);
    store_vec(out + h, s[1]);
}

// Generic width (T up to 17): state in shared memory, one thread per hash, rolled loops.
__global__ void __launch_bounds__(64) k_poseidon_gen(const Fr *__restrict__ consts, uint32_t T, uint32_t rf, uint32_t rp,
                                                     const Fr *__restrict__ in, size_t n, Fr *__restrict__ out) {
    extern __shared__ uint4 smem_raw[];
    Fr *sc = (Fr *)smem_raw;
    const uint32_t nconst = T * (rf + rp) + T * T;  // the unscaled MDS block only (rolled loops use plain products)
    {
        const uint4 *src = (const uint4 *)consts;
        uint4 *dst = (uint4 *)sc;
        for (uint32_t i = threadIdx.x; i < nconst * 2; i += blockDim.x) dst[i] = src[i];
    }
    // per-thread state and scratch rows, interleaved by thread to avoid bank conflicts on
    // 16-byte accesses: element i of thread x lives at st[(i * blockDim + x)]
    Fr *st = sc + nconst;
    Fr *tmp = st + (size_t)T * blockDim.x;
    __syncthreads();
    const Fr *mds = sc + T * (rf + rp);
    size_t h = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (h >= n) return;
    const uint32_t x = threadIdx.x, bd = blockDim.x;
    st[x] = Fr::zero();
    for (uint32_t i = 1; i < T; i++) st[i * bd + x] = load_vec(in + h * (T - 1) + (i - 1));
    const uint32_t half = rf / 2;
    const Fr *rc = sc;
    for (uint32_t rnd = 0; rnd < rf + rp; rnd++) {
        const bool full = (rnd < half || rnd >= half + rp);
        for (uint32_t i = 0; i < T; i++) {
            Fr v = lds_fr(&st[i * bd + x]) + lds_fr(rc + i);
            if (full || i == 0) v = pow5(v);
            st[i * bd + x] = v;
        }
        rc += T;
        for (uint32_t j = 0; j < T; j++) {
            Fr acc = lds_fr(mds + j * T) * lds_fr(&st[x]);
            for (uint32_t k = 1; k < T; k++) acc = acc + lds_fr(mds + j * T + k) * lds_fr(&st[k * bd + x]);
            tmp[j * bd + x] = acc;
        }
        for (uint32_t i = 0; i < T; i++) st[i * bd + x] = tmp[i * bd + x];
    }
    store_vec(out + h, lds_fr(&st[bd + x]));
}

template <int T>
static int32_t launch_reg(bzk_ctx *ctx, const PoseidonTable &pt, const Fr *d_in, size_t n, Fr *d_out) {
    const int threads = 128;
    size_t smem = (size_t)(pt.nrc + 2 * T * T) * sizeof(Fr);
    BZK_CUDA(ctx, cudaFuncSetAttribute(k_poseidon_reg<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_poseidon_reg<T><<<div_up(n, threads), threads, smem, ctx->stream>>>(pt.d_consts, pt.rf, pt.rp, d_in, n, d_out);
    BZK_LAUNCHED(ctx);
    return BZK_OK;
}

// ---------------------------------------------------------------------------------------------
// 4-ary Poseidon Merkle trees (dense): the hash structure of `KvStoreStateManager`
// (/root/reference/src/zk/state/mod.rs:218-264 prove, :310-420 set_data) and of the merkle gadget
// (/root/reference/src/zk/groth16/gadgets/merkle/mod.rs:21-65): node = Poseidon-4(children), proof =
// per level the 3 siblings in ascending child order with self skipped, leaf level first, child
// position = 2 index bits per level.
// Node buffer layout: level 0 (4^k leaves) | level 1 (4^(k-1)) | ... | root; (4^(k+1)-1)/3 elements.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_merkle4_prove(const Fr *__restrict__ nodes, uint32_t log4, const uint64_t *__restrict__ idx,
                                                       size_t m, Fr *__restrict__ proofs) {
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= m * log4) return;
    const size_t p = t / log4;
    const uint32_t lvl = (uint32_t)(t % log4);
    size_t off = 0;
    for (uint32_t l = 0; l < lvl; l++) off += (size_t)1 << (2 * (log4 - l));
    const uint64_t node = idx[p] >> (2 * lvl);
    const uint64_t base = node & ~(uint64_t)3;
    Fr *out = proofs + (p * log4 + lvl) * 3;
    int w = 0;
    for (int k = 0; k < 4; k++)
        if (base + k != node) store_vec(out + (w++), load_vec(nodes + off + base + k));
}

// one thread per path: recompute the root from (index, leaf, proof) — log4 sequential Poseidon-4
__global__ void __launch_bounds__(128) k_merkle4_root(const Fr *__restrict__ consts, uint32_t rf, uint32_t rp, uint32_t log4,
                                                      const uint64_t *__restrict__ idx, const Fr *__restrict__ leaves,
                                                      const Fr *__restrict__ proofs, size_t m, Fr *__restrict__ roots) {
    constexpr int T = 5;
    extern __shared__ uint4 smem_raw[];
    Fr *sc = (Fr *)smem_raw;
    stage_consts<T>(consts, rf, rp, sc);
    const size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= m) return;
    Fr cur = load_vec(leaves + p);
    uint64_t index = idx[p];
    for (uint32_t lvl = 0; lvl < log4; lvl++) {
        const uint32_t pos = (uint32_t)(index & 3);
        index >>= 2;
        Fr s[T];
        s[0] = Fr::zero();
        const Fr *sib = proofs + (p * log4 + lvl) * 3;
        int w = 0;
#pragma unroll
        for (int k = 0; k < 4; k++) {
            if ((uint32_t)k == pos) s[1 + k] = cur;
            else s[1 + k] = load_vec(sib + (w++));
        }
        poseidon_rounds<T>(s, sc, rf, rp);
        cur = s[1];
    }
    store_vec(roots + p, cur);
}

// ---------------------------------------------------------------------------------------------
// Versioned batch update of sparse 4-ary Poseidon trees (the transition builder's hot loop).
//
// The reference applies a batch of leaf writes ONE AT A TIME, re-hashing a root path per write and
// reading a Merkle proof between writes (`KvStoreStateManager::set_data` / `prove`,
// /root/reference/src/zk/state/mod.rs:218-264,310-420, driven by /root/reference/src/mpn/update.rs:40-258):
// n writes = n x depth strictly sequential hashes.  Here the whole batch is ONE pass per tree level: event
// e (write number e) owns a thread; at level l its node value is H(children), where the child on its own
// path is its value from level l-1 and each of the three siblings is the value of the LATEST EARLIER event
// whose path runs through that sibling (found by scanning the event list backwards), or — when no earlier
// event of the batch touched it — the sibling from the proof against the pre-batch tree that the host reads
// from its store (`init_proofs`, no hashing).  By induction over levels every event sees exactly the tree
// the sequential loop would have shown it, so
//     out_proofs[e]  = the Merkle proof of leaf idx[e] just before write e   (what `prove` returned)
//     vals[depth][e] = the root just after write e                            (what `set_data` produced)
// and depth launches replace n x depth dependent hashes.  `tree_id` lets one call update a forest (the
// per-account token trees).  The backward scan is O(n) per thread; batches are <= a few thousand writes.
__global__ void __launch_bounds__(128) k_tree4_versioned_level(const Fr *__restrict__ consts, uint32_t rf, uint32_t rp, uint32_t depth,
                                                               uint32_t lvl, const uint32_t *__restrict__ tree_id,
                                                               const uint64_t *__restrict__ idx, uint32_t n, Fr *vals,
                                                               const Fr *__restrict__ init_proofs, Fr *__restrict__ out_proofs) {
    constexpr int T = 5;
    extern __shared__ uint4 smem_raw[];
    Fr *sc = (Fr *)smem_raw;
    stage_consts<T>(consts, rf, rp, sc);
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n) return;
    const Fr *cur = vals + (size_t)lvl * n;
    const uint64_t me = idx[e];
    const uint32_t tid = tree_id[e], pos = (uint32_t)((me >> (2 * lvl)) & 3);
    const uint32_t up = 2 * lvl + 2;  // depth 32: the top level's shift is the full word
    const uint64_t prefix = up >= 64 ? 0 : me >> up;
    Fr s[T];
    s[0] = Fr::zero();
    {
        const Fr *sib = init_proofs + ((size_t)e * depth + lvl) * 3;
        int w = 0;
#pragma unroll
        for (int k = 0; k < 4; k++) {
            if ((uint32_t)k == pos) s[1 + k] = cur[e];
            else s[1 + k] = load_vec(sib + (w++));
        }
    }
    uint32_t found = 1u << pos;
    for (uint32_t b = e; b-- > 0 && found != 15u;) {
        const uint64_t other = idx[b];
        if (tree_id[b] != tid || (up >= 64 ? 0 : other >> up) != prefix) continue;
        const uint32_t k = (uint32_t)((other >> (2 * lvl)) & 3);
        if (found & (1u << k)) continue;
        found |= 1u << k;
        const Fr v = cur[b];
#pragma unroll
        for (int q = 0; q < 4; q++)
            if ((uint32_t)q == k) s[1 + q] = v;
    }
    {
        Fr *po = out_proofs + ((size_t)e * depth + lvl) * 3;
        int w = 0;
#pragma unroll
        for (int k = 0; k < 4; k++)
            if ((uint32_t)k != pos) store_vec(po + (w++), s[1 + k]);
    }
    poseidon_rounds<T>(s, sc, rf, rp);
    store_vec(vals + (size_t)(lvl + 1) * n + e, s[1]);
}

int32_t tree4_versioned_update(bzk_ctx *ctx, uint32_t depth, const uint32_t *d_tree_id, const uint64_t *d_idx, size_t n, Fr *d_vals,
                               const Fr *d_init_proofs, Fr *d_out_proofs) {
    if (!ctx->pos_loaded) return BZK_ERR_NO_PARAMS;
    if (depth == 0 || depth > 32 || n > (1u << 24) || (n && (!d_tree_id || !d_idx || !d_vals || !d_init_proofs || !d_out_proofs))) return BZK_ERR_BAD_ARG;
    if (n == 0) return BZK_OK;
    const PoseidonTable &pt = ctx->pos[5];
    const size_t smem = (size_t)(pt.nrc + 50) * sizeof(Fr);
    BZK_CUDA(ctx, cudaFuncSetAttribute(k_tree4_versioned_level, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    for (uint32_t lvl = 0; lvl < depth; lvl++) {
        k_tree4_versioned_level<<<div_up(n, 128), 128, smem, ctx->stream>>>(pt.d_consts, pt.rf, pt.rp, depth, lvl, d_tree_id, d_idx, (uint32_t)n, d_vals,
                                                                           d_init_proofs, d_out_proofs);
        BZK_LAUNCHED(ctx);
    }
    return BZK_OK;
}

int32_t poseidon_launch(bzk_ctx *ctx, uint32_t arity, const Fr *d_in, size_t n, Fr *d_out);

int32_t merkle4_build(bzk_ctx *ctx, Fr *d_nodes, uint32_t log4) {
    if (log4 > 15 || !d_nodes) return BZK_ERR_BAD_ARG;
    size_t off = 0;
    for (uint32_t lvl = 0; lvl < log4; lvl++) {
        const size_t n_lvl = (size_t)1 << (2 * (log4 - lvl));
        BZK_TRY(poseidon_launch(ctx, 4, d_nodes + off, n_lvl / 4, d_nodes + off + n_lvl));
        off += n_lvl;
    }
    return BZK_OK;
}
int32_t merkle4_prove(bzk_ctx *ctx, const Fr *d_nodes, uint32_t log4, const uint64_t *d_idx, size_t m, Fr *d_proofs) {
    // a one-leaf tree (log4 = 0) has empty proofs: like merkle4_root, no proof buffer is needed then
    if (log4 > 15 || (m && (!d_nodes || !d_idx || (log4 && !d_proofs)))) return BZK_ERR_BAD_ARG;
    if (m == 0 || log4 == 0) return BZK_OK;
    k_merkle4_prove<<<div_up(m * log4, 256), 256, 0, ctx->stream>>>(d_nodes, log4, d_idx, m, d_proofs);
    BZK_LAUNCHED(ctx);
    return BZK_OK;
}
int32_t merkle4_root(bzk_ctx *ctx, uint32_t log4, const uint64_t *d_idx, const Fr *d_leaves, const Fr *d_proofs, size_t m, Fr *d_roots) {
    if (!ctx->pos_loaded) return BZK_ERR_NO_PARAMS;
    if (log4 > 32 || (m && (!d_idx || !d_leaves || !d_roots || (log4 && !d_proofs)))) return BZK_ERR_BAD_ARG;
    if (m == 0) return BZK_OK;
    const PoseidonTable &pt = ctx->pos[5];
    const size_t smem = (size_t)(pt.nrc + 50) * sizeof(Fr);
    BZK_CUDA(ctx, cudaFuncSetAttribute(k_merkle4_root, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_merkle4_root<<<div_up(m, 128), 128, smem, ctx->stream>>>(pt.d_consts, pt.rf, pt.rp, log4, d_idx, d_leaves, d_proofs, m, d_roots);
    BZK_LAUNCHED(ctx);
    return BZK_OK;
}

int32_t poseidon_launch(bzk_ctx *ctx, uint32_t arity, const Fr *d_in, size_t n, Fr *d_out) {
    if (!ctx->pos_loaded) return BZK_ERR_NO_PARAMS;
    if (arity < 1 || arity > 16) return BZK_ERR_BAD_ARG;
    if (n == 0) return BZK_OK;
    const PoseidonTable &pt = ctx->pos[arity + 1];
    switch (arity + 1) {
        case 2: return launch_reg<2>(ctx, pt, d_in, n, d_out);
        case 3: return launch_reg<3>(ctx, pt, d_in, n, d_out);
        case 4: return launch_reg<4>(ctx, pt, d_in, n, d_out);
        case 5: return launch_reg<5>(ctx, pt, d_in, n, d_out);
        case 6: return launch_reg<6>(ctx, pt, d_in, n, d_out);
        case 7: return launch_reg<7>(ctx, pt, d_in, n, d_out);
        case 8: return launch_reg<8>(ctx, pt, d_in, n, d_out);
        default: break;
    }
    const uint32_t T = arity + 1;
    const int threads = 64;
    size_t smem = ((size_t)(pt.nrc + T * T) + (size_t)2 * T * threads) * sizeof(Fr);
    BZK_CUDA(ctx, cudaFuncSetAttribute(k_poseidon_gen, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_poseidon_gen<<<div_up(n, threads), threads, smem, ctx->stream>>>(pt.d_consts, T, pt.rf, pt.rp, d_in, n, d_out);
    BZK_LAUNCHED(ctx);
    return BZK_OK;
}

// ---------------------------------------------------------------------------------------------
// One step of a hash plan (hash_plan.cuh): one thread per output node; each operand comes from the previous step's outputs
// or from the plan's host-supplied values, as its tag says.  bzk_mpn_state_apply_delta runs a block's whole re-hash as a
// chain of these, one per tree level, with no host round trip in between.
// ---------------------------------------------------------------------------------------------
template <int T>
__global__ void __launch_bounds__(128) k_poseidon_plan_step(const Fr *__restrict__ consts, uint32_t rf, uint32_t rp, const uint32_t *__restrict__ ops,
                                                            size_t n, const Fr *__restrict__ prev, const Fr *__restrict__ host, Fr *__restrict__ out) {
    extern __shared__ uint4 smem_raw[];
    Fr *sc = (Fr *)smem_raw;
    stage_consts<T>(consts, rf, rp, sc);
    const size_t h = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (h >= n) return;
    Fr s[T];
    s[0] = Fr::zero();
#pragma unroll
    for (int i = 1; i < T; i++) s[i] = load_vec(plan_operand(ops[h * (T - 1) + (i - 1)], prev, host));
    poseidon_rounds<T>(s, sc, rf, rp);
    store_vec(out + h, s[1]);
}

template <int T>
static int32_t launch_plan_step(bzk_ctx *ctx, const uint32_t *d_ops, size_t n, const Fr *d_prev, const Fr *d_host, Fr *d_out) {
    const PoseidonTable &pt = ctx->pos[T];
    const size_t smem = (size_t)(pt.nrc + 2 * T * T) * sizeof(Fr);
    BZK_CUDA(ctx, cudaFuncSetAttribute(k_poseidon_plan_step<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_poseidon_plan_step<T><<<div_up(n, 128), 128, smem, ctx->stream>>>(pt.d_consts, pt.rf, pt.rp, d_ops, n, d_prev, d_host, d_out);
    BZK_LAUNCHED(ctx);
    return BZK_OK;
}

int32_t poseidon_plan_step(bzk_ctx *ctx, uint32_t arity, const uint32_t *d_ops, size_t n, const Fr *d_prev, const Fr *d_host, Fr *d_out) {
    if (!ctx->pos_loaded) return BZK_ERR_NO_PARAMS;
    if (n && (!d_ops || !d_host || !d_out)) return BZK_ERR_BAD_ARG;
    if (n == 0) return BZK_OK;
    switch (arity) {
        case 2: return launch_plan_step<3>(ctx, d_ops, n, d_prev, d_host, d_out);
        case 4: return launch_plan_step<5>(ctx, d_ops, n, d_prev, d_host, d_out);
        case 5: return launch_plan_step<6>(ctx, d_ops, n, d_prev, d_host, d_out);
        default: return BZK_ERR_BAD_ARG;
    }
}

}  // namespace bzk
