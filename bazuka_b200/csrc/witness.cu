// bazuka_b200 — witness generation for the MPN update circuit on the GPU.
//
// bellman's prover obtains the witness by running the circuit's `synthesize` with value closures
// (`ProvingAssignment`, driven from /root/reference/src/mpn/circuits/update_circuit.rs:49-494 and the gadgets
// under /root/reference/src/zk/groth16/gadgets/).  Every slot of the update batch executes the SAME sequence
// of allocations, so the host compiles that sequence once into a straight-line program
// (bazuka_b200/mpn/witness_program.py: RAW / MUL / BIT / ISZERO / INVZ / SELECT / JJ over pooled linear
// combinations) and this kernel interprets it with one thread per slot.
//
// Layout: V[slot][tx] (32 B per element, tx fastest) so that a warp's accesses to one variable are one
// contiguous 1 KB run; the program stream (ops, LC pool, coefficients) is read at warp-uniform addresses
// (broadcast).  The block's values are also written, slot-major -> tx-major, straight into the z vector the
// prover consumes (aux_out[tx * n_ops + j]), so the witness never visits the host.
//
// Round 2: ONE WARP PER SLOT, the program executed level by level.  At upload the host orders the ops by their depth in the
// data-flow graph (level = 1 + the deepest operand); the ops of one level are independent, the lanes of the slot's warp take
// them 32 at a time and a __syncwarp() separates levels.  A slot's critical path — the Merkle paths' Poseidon rounds, the two
// 255-step EdDSA ladders — is ~5x shorter than its op count (a Poseidon state is t lanes wide, the ladders run side by side,
// bit decompositions are flat), and the slot's variables are read straight out of its z segment (slot-major: no transposed
// V array, no second store).  The one-thread-per-slot kernel stays for A/B runs (BZK_WITNESS_SERIAL=1).
#include <algorithm>
#include <vector>

#include "common.cuh"
#include "witness_core.cuh"

namespace bzk {

// V[variable][slot] in global memory, tx fastest; block values also go slot-major into z
struct WitMemDev {
    Fr *V, *aux_out;
    uint32_t ntx, tx, n_ops;
    __device__ __forceinline__ Fr load(int32_t slot) const {
        Fr r;
        const uint4 *s = (const uint4 *)(V + (size_t)slot * ntx + tx);
        uint4 a = s[0], b = s[1];
        r.l[0] = a.x; r.l[1] = a.y; r.l[2] = a.z; r.l[3] = a.w;
        r.l[4] = b.x; r.l[5] = b.y; r.l[6] = b.z; r.l[7] = b.w;
        return r;
    }
    __device__ __forceinline__ void store(uint32_t slot, const Fr &v) const { store_vec(V + (size_t)slot * ntx + tx, v); }
    __device__ __forceinline__ void out(uint32_t j, const Fr &v) const { store_vec(aux_out + (size_t)tx * n_ops + j, v); }
    // the interpreter's loads are otherwise serialised behind one another (V of a 256-slot batch is ~460 MB, so
    // they are DRAM latencies); addresses are warp-uniform in the slot and consecutive in tx
    __device__ __forceinline__ void prefetch(int32_t slot) const {
        asm volatile("prefetch.global.L1 [%0];" ::"l"(__cvta_generic_to_global(V + (size_t)slot * ntx + tx)));
    }
};

__global__ void __launch_bounds__(32) k_witness_run(WitProgDev P, Fr jj_d, const Fr *__restrict__ raws, const Fr *__restrict__ ext,
                                                    uint32_t ntx, Fr *V, Fr *__restrict__ aux_out) {
    const uint32_t tx = blockIdx.x * blockDim.x + threadIdx.x;
    if (tx >= ntx) return;
    WitMemDev mem{V, aux_out, ntx, tx, P.n_ops};
    wit_run_slot(P, jj_d, raws + (size_t)tx * P.n_raw, ext + (size_t)tx * P.n_ext, mem);
}

// ---- level-parallel execution: a warp per slot -------------------------------------------------------------------
struct WitSched {
    const int32_t *sops;       // [n_exec][8]: code, lc0..lc3, imm, op index, unused — in (level, opcode) order, NOPs dropped
    const int32_t *level_ptr;  // [n_levels + 1] into sops
    uint32_t n_levels;
};

// the slot's variables live in its z segment; slots below block0 (ONE, externals) in a small side array
struct WitMemSeg {
    const Fr *pre;
    Fr *z;
    uint32_t block0;
    __device__ __forceinline__ Fr load(int32_t slot) const {
        const Fr *p = (uint32_t)slot < block0 ? pre + slot : z + ((uint32_t)slot - block0);
        Fr r;
        const uint4 *s = (const uint4 *)p;
        uint4 a = s[0], b = s[1];
        r.l[0] = a.x; r.l[1] = a.y; r.l[2] = a.z; r.l[3] = a.w;
        r.l[4] = b.x; r.l[5] = b.y; r.l[6] = b.z; r.l[7] = b.w;
        return r;
    }
    __device__ __forceinline__ void store(uint32_t slot, const Fr &v) const { store_vec(z + (slot - block0), v); }
    __device__ __forceinline__ void out(uint32_t, const Fr &) const {}
    __device__ __forceinline__ void prefetch(int32_t) const {}
};

__global__ void __launch_bounds__(32) k_witness_levels(WitProgDev P, WitSched S, Fr jj_d, const Fr *__restrict__ raws, const Fr *__restrict__ ext,
                                                       uint32_t ntx, Fr *pre, Fr *aux_out) {
    const uint32_t tx = blockIdx.x, lane = threadIdx.x, block0 = 1 + P.n_ext;
    if (tx >= ntx) return;
    Fr *mine = pre + (size_t)tx * block0;
    if (lane == 0) store_vec(mine, Fr::one());
    for (uint32_t k = lane; k < P.n_ext; k += 32) store_vec(mine + 1 + k, ext[(size_t)tx * P.n_ext + k].to_mont());
    __syncwarp();
    WitMemSeg mem{mine, aux_out + (size_t)tx * P.n_ops, block0};
    const Fr *row = raws + (size_t)tx * P.n_raw;
    int32_t lo = S.level_ptr[0];
    for (uint32_t L = 0; L < S.n_levels; L++) {
        const int32_t hi = S.level_ptr[L + 1];
        for (int32_t i = lo + (int32_t)lane; i < hi; i += 32) {
            const int4 *q = (const int4 *)(S.sops + (size_t)i * 8);
            const int4 u = q[0], v = q[1];
            wit_exec_op(P, jj_d, row, (uint32_t)v.z, u.x, u.y, u.z, u.w, v.x, v.y, mem);
        }
        lo = hi;
        __syncwarp();  // orders this level's stores before the next level's loads (same warp, same SM)
    }
}

}  // namespace bzk

using namespace bzk;

struct bzk_witness_program {
    WitProgDev d{};
    WitSched sched{};
    Fr jj_d;
    void *blob = nullptr;
    uint64_t n_lc = 0, n_terms = 0, n_coefs = 0;
};

namespace bzk {
// a field image is usable as it stands only below r: the device arithmetic assumes reduced operands
static bool fr_image_below_r(const bzk_fr *v) {
    Fr a;
    memcpy(&a, v, sizeof(Fr));
    return Fr::reduce_once(a) == a;
}

// the shape a driver must match before it hands rows to the interpreter (csrc/mpn_host.cu)
void witness_program_shape(const bzk_witness_program *p, uint64_t *n_ops, uint32_t *n_raw, uint32_t *n_ext) {
    *n_ops = p->d.n_ops; *n_raw = p->d.n_raw; *n_ext = p->d.n_ext;
}
}  // namespace bzk

extern "C" {

int32_t bzk_witness_program_upload(bzk_ctx *ctx, const int32_t *ops, uint64_t n_ops, const int32_t *lc_ptr, uint64_t n_lc,
                                   const int32_t *lc_slot, const int32_t *lc_coef, uint64_t n_terms, const bzk_fr *coefs,
                                   uint64_t n_coefs, uint32_t n_raw, uint32_t n_ext, const bzk_fr *jj_d, bzk_witness_program **out) {
    if (!ctx || !ops || !lc_ptr || !coefs || !jj_d || !out || !n_ops || !n_coefs || (n_terms && (!lc_slot || !lc_coef))) return BZK_ERR_BAD_ARG;
    // validate on the host: the device interpreter trusts the program.  It takes coefficient index 0 as one without
    // reading coefs[0], so any other value there would make the device and the program's own meaning disagree.
    Fr c0;
    memcpy(&c0, coefs, sizeof(Fr));
    if (c0 != Fr::one() || !fr_image_below_r(jj_d)) return BZK_ERR_BAD_ARG;
    for (uint64_t k = 1; k < n_coefs; k++)
        if (!fr_image_below_r(coefs + k)) return BZK_ERR_BAD_ARG;
    const uint64_t kSlotBlock0 = 1 + (uint64_t)n_ext;
    for (uint64_t j = 0; j < n_ops; j++) {
        const int32_t *op = ops + j * 6;
        if (op[0] < W_RAW || op[0] > W_NOP) return BZK_ERR_BAD_ARG;
        if (op[0] == W_RAW && (op[5] < 0 || (uint32_t)op[5] >= n_raw)) return BZK_ERR_BAD_ARG;
        if (op[0] == W_BIT && (op[5] < 0 || op[5] > 255)) return BZK_ERR_BAD_ARG;
        if (op[0] == W_JJ && (j + 1 >= n_ops || ops[(j + 1) * 6] != W_NOP)) return BZK_ERR_BAD_ARG;
        // a NOP is only the second half of a JJ (which writes both variables); alone it would leave its variable unwritten
        if (op[0] == W_NOP && (j == 0 || ops[(j - 1) * 6] != W_JJ)) return BZK_ERR_BAD_ARG;
        const int nlc = op[0] == W_JJ ? 4 : op[0] == W_SELECT ? 3 : op[0] == W_MUL ? 2 : (op[0] == W_RAW || op[0] == W_NOP) ? 0 : 1;
        for (int a = 0; a < nlc; a++) {
            const int32_t l = op[1 + a];
            if (l < 0 || (uint64_t)l >= n_lc) return BZK_ERR_BAD_ARG;
            for (int32_t k = lc_ptr[l]; k < lc_ptr[l + 1]; k++) {
                if (k < 0 || (uint64_t)k >= n_terms) return BZK_ERR_BAD_ARG;
                if (lc_slot[k] < 0 || (uint64_t)lc_slot[k] >= kSlotBlock0 + j) return BZK_ERR_BAD_ARG;  // reads only earlier variables
                if (lc_coef[k] < 0 || (uint64_t)lc_coef[k] >= n_coefs) return BZK_ERR_BAD_ARG;
            }
        }
    }
    // schedule: depth of every variable in the data-flow graph, ops ordered by (depth, opcode)
    std::vector<int32_t> level_ptr, sops;
    const uint32_t n_levels = wit_build_schedule(ops, n_ops, lc_ptr, lc_slot, n_ext, sops, level_ptr);
    BZK_CUDA(ctx, cudaSetDevice(ctx->device));
    auto *p = new (std::nothrow) bzk_witness_program;
    if (!p) return BZK_ERR_OOM;
    size_t need;
    {
        Carver cv(nullptr);
        cv.take<int32_t>(n_ops * 6); cv.take<int32_t>(n_lc + 1); cv.take<int32_t>(n_terms + 1); cv.take<int32_t>(n_terms + 1); cv.take<Fr>(n_coefs);
        cv.take<int32_t>(sops.size()); cv.take<int32_t>(level_ptr.size());
        need = cv.used();
    }
    if (cudaMalloc(&p->blob, need) != cudaSuccess) { delete p; cudaGetLastError(); return BZK_ERR_OOM; }
    Carver cv(p->blob);
    int32_t *d_ops = cv.take<int32_t>(n_ops * 6), *d_ptr = cv.take<int32_t>(n_lc + 1), *d_slot = cv.take<int32_t>(n_terms + 1),
            *d_coef = cv.take<int32_t>(n_terms + 1);
    Fr *d_coefs = cv.take<Fr>(n_coefs);
    int32_t *d_sops = cv.take<int32_t>(sops.size()), *d_level_ptr = cv.take<int32_t>(level_ptr.size());
    cudaError_t e = cudaMemcpyAsync(d_ops, ops, n_ops * 6 * 4, cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_sops, sops.data(), sops.size() * 4, cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_level_ptr, level_ptr.data(), level_ptr.size() * 4, cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_ptr, lc_ptr, (n_lc + 1) * 4, cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess && n_terms) e = cudaMemcpyAsync(d_slot, lc_slot, n_terms * 4, cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess && n_terms) e = cudaMemcpyAsync(d_coef, lc_coef, n_terms * 4, cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_coefs, coefs, n_coefs * sizeof(Fr), cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess) { cudaFree(p->blob); delete p; BZK_CUDA(ctx, e); }
    p->d = WitProgDev{d_ops, d_ptr, d_slot, d_coef, d_coefs, (uint32_t)n_ops, n_raw, n_ext};
    p->sched = WitSched{d_sops, d_level_ptr, n_levels};
    memcpy(&p->jj_d, jj_d, sizeof(Fr));
    p->n_lc = n_lc; p->n_terms = n_terms; p->n_coefs = n_coefs;
    *out = p;
    return BZK_OK;
}

int32_t bzk_witness_program_free(bzk_ctx *ctx, bzk_witness_program *p) {
    if (!p) return BZK_OK;
    if (ctx) cudaSetDevice(ctx->device);
    if (p->blob) cudaFree(p->blob);
    delete p;
    return BZK_OK;
}

int32_t bzk_witness_run_dev(bzk_ctx *ctx, const bzk_witness_program *p, const bzk_fr *raws, const bzk_fr *ext, uint64_t ntx, void *d_aux_out) {
    if (!ctx || !p || (p->d.n_raw && !raws) || (p->d.n_ext && !ext) || !d_aux_out || !ntx || ntx > (1u << 24)) return BZK_ERR_BAD_ARG;
    BZK_CUDA(ctx, cudaSetDevice(ctx->device));
    static const bool serial = getenv("BZK_WITNESS_SERIAL") && atoi(getenv("BZK_WITNESS_SERIAL")) != 0;
    // scratch: the serial kernel's transposed variable array, or the level kernel's {ONE, externals} rows
    const size_t n_scratch = serial ? ((size_t)1 + p->d.n_ext + p->d.n_ops) * ntx : ((size_t)1 + p->d.n_ext) * ntx;
    size_t need;
    {
        Carver cv(nullptr);
        cv.take<Fr>(n_scratch); cv.take<Fr>((size_t)p->d.n_raw * ntx + 1); cv.take<Fr>((size_t)p->d.n_ext * ntx + 1);
        need = cv.used();
    }
    BZK_TRY(ensure_ws(ctx, &ctx->ws, &ctx->ws_bytes, need));
    Carver cv(ctx->ws);
    Fr *V = cv.take<Fr>(n_scratch), *d_raws = cv.take<Fr>((size_t)p->d.n_raw * ntx + 1), *d_ext = cv.take<Fr>((size_t)p->d.n_ext * ntx + 1);
    if (p->d.n_raw) BZK_CUDA(ctx, cudaMemcpyAsync(d_raws, raws, (size_t)p->d.n_raw * ntx * sizeof(Fr), cudaMemcpyHostToDevice, ctx->stream));
    if (p->d.n_ext) BZK_CUDA(ctx, cudaMemcpyAsync(d_ext, ext, (size_t)p->d.n_ext * ntx * sizeof(Fr), cudaMemcpyHostToDevice, ctx->stream));
    if (serial)
        k_witness_run<<<(unsigned)div_up(ntx, 32), 32, 0, ctx->stream>>>(p->d, p->jj_d, d_raws, d_ext, (uint32_t)ntx, V, (Fr *)d_aux_out);
    else
        k_witness_levels<<<(unsigned)ntx, 32, 0, ctx->stream>>>(p->d, p->sched, p->jj_d, d_raws, d_ext, (uint32_t)ntx, V, (Fr *)d_aux_out);
    BZK_LAUNCHED(ctx);
    BZK_CUDA(ctx, cudaGetLastError());
    // the host buffers may be pageable: the copies above are complete for the caller only after this
    BZK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return BZK_OK;
}

}  // extern "C"
