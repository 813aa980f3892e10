// bazuka_b200 — context, error plumbing and device workspace shared by all kernels' host stubs.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <new>
#include <vector>
#include "../../include/bzk.h"
#include "ec.cuh"

namespace bzk {

constexpr int kNumSMs = 132;  // H100 SXM; bzk_ctx_create replaces it with the device's count

struct PoseidonTable {
    uint32_t t = 0, rf = 0, rp = 0, nrc = 0;
    Fr *d_consts = nullptr;  // device: nrc round constants then t*t MDS entries, Montgomery
};

// MSM window plan (shared by the MSM translation units and the Groth16 driver)
struct MsmPlan {
    uint32_t c = 0;   // window bits
    uint32_t W = 0;   // windows (0: empty sum)
    uint32_t NB = 0;  // buckets per bucket group = 2^(c-1)
    uint32_t TB = 0;  // total buckets = G * NB
    uint32_t T = 1;   // table levels in use: level t holds [2^(c*G*t)] P (1 = plain bases)
    uint32_t G = 0;   // bucket groups = ceil(W / T): window j = t*G + g feeds group g from level t
    uint32_t slice = 0, nbits = 0;  // bucket reduction: buckets per slice, bits of the slice index (host fold)
};
constexpr uint32_t kMaxWinPoints = 320;  // >= G * (1 + nbits) for every plan make_plan can produce

// What one sum needs to stream a host-resident base vector (msm_impl.cuh): a copy stream and two device chunk buffers,
// grown only.  ready[b]: the copy into buffer b is done; freed[b]: the last kernel that read buffer b is done.
struct StreamPipe {
    cudaStream_t copy = nullptr;
    void *buf = nullptr;
    size_t bytes = 0;
    cudaEvent_t ready[2] = {nullptr, nullptr}, freed[2] = {nullptr, nullptr};
};

struct NttTables {
    Fr *d_fwd = nullptr;  // omega^j, j < n/2
    Fr *d_inv = nullptr;  // omega^-j
    uint32_t log_n = 0;
};

}  // namespace bzk

struct bzk_ctx {
    int device = 0;
    cudaStream_t own_stream = nullptr;
    cudaStream_t stream = nullptr;
    char err[512] = {0};
    uint64_t launches = 0;
    // grow-only scratch arenas (one for MSM, one for staging host<->device copies)
    void *ws = nullptr;
    size_t ws_bytes = 0;
    void *stage = nullptr;
    size_t stage_bytes = 0;
    void *pinned = nullptr;
    size_t pinned_bytes = 0;
    bzk::PoseidonTable pos[18];
    bool pos_loaded = false;
    bzk::NttTables ntt[29];
    bzk::Fr *d_gpow = nullptr;  // coset generator power tables, see ntt.cu
    int sm_count = bzk::kNumSMs;
    int affine_rounds[2] = {-1, -1};  // batched-affine rounds for G1 / G2 sums (-1: BZK_AFFINE_ROUNDS[_G2] or the default 0)
    uint32_t table_c = 0;             // window of the fixed-base tables built from now on (0: BZK_TABLE_C or the cost model)
    // plan of the last single MSM (msm_run): c, W, T, G, NB, slice, nbits, long-run queue length (timing on, else 0)
    uint32_t last_plan[8] = {0};
    // side streams + arenas so that independent MSMs of one proof run concurrently (groth16.cu)
    cudaStream_t aux_stream[4] = {nullptr, nullptr, nullptr, nullptr};
    void *aux_ws[4] = {nullptr, nullptr, nullptr, nullptr};
    size_t aux_ws_bytes[4] = {0, 0, 0, 0};
    cudaEvent_t aux_ev[3] = {nullptr, nullptr, nullptr};
    // streamed sums over host vectors: pipe 0 serves the context's stream (single MSMs, the h sum), 1..4 the side streams
    bzk::StreamPipe pipe[5];
    uint64_t stream_chunk = 0;     // points per chunk buffer (0: the default of msm_impl.cuh), bzk_ctx_set_msm_stream_chunk
    uint64_t last_stream[4] = {0};  // of the last single MSM: chunks, chunk points, bytes copied host->device, 1 if streamed
    // optional per-stage device timing (CUDA events on the launching stream), see bzk_ctx_set_timing
    bool timing = false;
    static constexpr int kMaxStages = 16;
    cudaEvent_t ev[kMaxStages + 1] = {nullptr};
    int n_marks = 0;
    float stage_ms[kMaxStages] = {0};
    double stage_ms_sum[kMaxStages] = {0};
    uint64_t stage_runs = 0;
    // Groth16 driver marks (timing on): 0 start, 1 z+evaluations done, 2 quotient (7 NTTs) done, 3 h sum done
    // (all on the main stream); 4..7 = end of the l / a / b_g1 / b_g2 side streams
    cudaEvent_t g16_ev[8] = {nullptr};
    float g16_ms[8] = {0};
    bool g16_valid = false;
    bzk::MsmPlan g16_plan[5];            // plans of the five sums of the proof in flight (kept across bzk_groth16_shard_begin / _finish)
    bool split_open = false;        // a shard_begin is waiting for its shard_finish
    // JubJub fixed-base table of BASE (jubjub.cuh, kJJFixedEntries JJNiels) for the curve d it was built with, made by the first
    // batch signature check (jubjub.cu)
    void *d_jj_table = nullptr;
    bzk::Fr jj_table_d{};
    // Ed25519 fixed-base table of B (ed25519.cuh, kJJFixedEntries EdNiels25519), made by the first batch Ed25519 check (ed25519.cu)
    void *d_ed_table = nullptr;
};

// A base vector, in one of two places.  On the device, `d` holds it; after bzk_g*_bases_precompute `d` holds tab_T levels
// of n points each: level t = [2^(tab_c * tab_G * t)] P_i (level 0 = the bases), so that the windows t*G+g of every scalar
// share bucket group g.  In host memory (bzk_g*_bases_move), `h` holds level 0 in pinned memory, `d` is null and there is
// no table; its MSMs stream the points to the device.
struct bzk_g1_bases {
    bzk::G1Affine *d = nullptr;
    bzk::G1Affine *h = nullptr;
    size_t n = 0;
    uint32_t tab_c = 0, tab_T = 1, tab_G = 0;
};
struct bzk_g2_bases {
    bzk::G2Affine *d = nullptr;
    bzk::G2Affine *h = nullptr;
    size_t n = 0;
    uint32_t tab_c = 0, tab_T = 1, tab_G = 0;
};

// A proving key (groth16.cu; read from / written to bellman's file format by params_io.cu).
struct bzk_groth16_params {
    bzk::G1Affine alpha_g1, beta_g1, delta_g1;
    bzk::G2Affine beta_g2, delta_g2;
    bzk_g1_bases *h = nullptr, *l = nullptr, *a = nullptr, *b1 = nullptr;
    bzk_g2_bases *b2 = nullptr;
    // base sharding (SURVEY.md §8e): this handle holds the contiguous range
    // [len*rank/world, len*(rank+1)/world) of each of the five base vectors
    uint32_t rank = 0, world = 1;
};

namespace bzk {
// what one MSM call sees of a base vector: the sub-range [off, off + n) of a (possibly multi-level) table
template <class F>
struct BasesRef {
    const Affine<F> *tab = nullptr;
    size_t n_tab = 0, off = 0;
    uint32_t c = 0, T = 1, G = 0;  // c == 0: no table, the plan is free to choose its window
    bool host = false;             // tab is pinned host memory: the sum streams it (msm_impl.cuh)
};
template <class B>
inline auto bases_ref(const B *b, size_t off = 0) {
    BasesRef<decltype(b->d->x)> r;
    r.tab = b->h ? b->h : b->d; r.n_tab = b->n; r.off = off; r.c = b->tab_c; r.T = b->tab_T; r.G = b->tab_G;
    r.host = b->h != nullptr;
    return r;
}
// storage for a new n-point vector, in pinned host memory or on the device; BZK_ERR_OOM (size in the context's error)
// when it cannot be had — a host vector never falls back to pageable memory
template <class B>
inline int32_t bases_alloc(bzk_ctx *ctx, B *b, bool on_host) {
    const size_t bytes = (b->n ? b->n : 1) * sizeof(*b->d);
    const cudaError_t e = on_host ? cudaHostAlloc((void **)&b->h, bytes, cudaHostAllocDefault) : cudaMalloc((void **)&b->d, bytes);
    if (e == cudaSuccess) return BZK_OK;
    cudaGetLastError();
    if (on_host) b->h = nullptr; else b->d = nullptr;
    snprintf(ctx->err, sizeof ctx->err, "%s(%zu bytes) for a base vector: %s", on_host ? "cudaHostAlloc" : "cudaMalloc", bytes, cudaGetErrorString(e));
    return e == cudaErrorMemoryAllocation ? BZK_ERR_OOM : BZK_ERR_CUDA;
}
// frees the vector's storage and the handle
template <class B>
inline void bases_release(B *b) {
    if (b->d) cudaFree(b->d);
    if (b->h) cudaFreeHost(b->h);
    delete b;
}
}  // namespace bzk

namespace bzk {

inline int32_t set_cuda_err(bzk_ctx *ctx, cudaError_t e, const char *what, const char *file, int line) {
    if (ctx) snprintf(ctx->err, sizeof ctx->err, "%s: %s (%s:%d)", what, cudaGetErrorString(e), file, line);
    return (e == cudaErrorMemoryAllocation) ? BZK_ERR_OOM : BZK_ERR_CUDA;
}

#define BZK_CUDA(ctx, call)                                                              \
    do {                                                                                 \
        cudaError_t e_ = (call);                                                         \
        if (e_ != cudaSuccess) return bzk::set_cuda_err((ctx), e_, #call, __FILE__, __LINE__); \
    } while (0)

#define BZK_TRY(call)               \
    do {                            \
        int32_t s_ = (call);        \
        if (s_ != BZK_OK) return s_; \
    } while (0)

// check the launch itself (configuration errors); execution errors surface at the next sync
#define BZK_LAUNCHED(ctx)                                                                         \
    do {                                                                                          \
        (ctx)->launches++;                                                                        \
        cudaError_t e_ = cudaGetLastError();                                                      \
        if (e_ != cudaSuccess) return bzk::set_cuda_err((ctx), e_, "kernel launch", __FILE__, __LINE__); \
    } while (0)

inline int32_t ensure_ws(bzk_ctx *ctx, void **p, size_t *have, size_t need) {
    if (*have >= need) return BZK_OK;
    if (*p) {
        BZK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        BZK_CUDA(ctx, cudaFree(*p));
        *p = nullptr;
        *have = 0;
    }
    size_t want = need + need / 8;
    cudaError_t e = cudaMalloc(p, want);
    if (e != cudaSuccess) {
        want = need;
        e = cudaMalloc(p, want);
    }
    if (e != cudaSuccess) return set_cuda_err(ctx, e, "cudaMalloc(workspace)", __FILE__, __LINE__);
    *have = want;
    return BZK_OK;
}

// carve aligned sub-buffers out of one arena
struct Carver {
    char *base;
    size_t off = 0;
    explicit Carver(void *b) : base((char *)b) {}
    template <class T>
    T *take(size_t count) {
        off = (off + 255) & ~(size_t)255;
        T *p = (T *)(base + off);
        off += count * sizeof(T);
        return p;
    }
    size_t used() const { return (off + 255) & ~(size_t)255; }
};

// stage marks: mark(ctx) records an event between kernels when timing is on; collect() after the
// stream was synchronised turns consecutive marks into per-stage milliseconds.
inline void timing_begin(bzk_ctx *ctx) {
    ctx->n_marks = 0;
    if (!ctx->timing) return;
    for (int i = 0; i <= bzk_ctx::kMaxStages; i++)
        if (!ctx->ev[i]) cudaEventCreate(&ctx->ev[i]);
    cudaEventRecord(ctx->ev[0], ctx->stream);
    ctx->n_marks = 1;
}
inline void timing_mark(bzk_ctx *ctx) {
    if (!ctx->timing || ctx->n_marks == 0 || ctx->n_marks > bzk_ctx::kMaxStages) return;
    cudaEventRecord(ctx->ev[ctx->n_marks++], ctx->stream);
}
inline void timing_collect(bzk_ctx *ctx) {
    if (!ctx->timing || ctx->n_marks < 2) return;
    for (int i = 0; i + 1 < ctx->n_marks; i++) {
        float ms = 0;
        cudaEventElapsedTime(&ms, ctx->ev[i], ctx->ev[i + 1]);
        ctx->stage_ms[i] = ms;
        ctx->stage_ms_sum[i] += ms;
    }
    for (int i = ctx->n_marks - 1; i < bzk_ctx::kMaxStages; i++) ctx->stage_ms[i] = 0;
    ctx->stage_runs++;
}

inline uint32_t div_up(size_t a, size_t b) { return (uint32_t)((a + b - 1) / b); }

// ---- wire <-> packed conversions (device) -------------------------------------------------
// 104-byte G1 / 200-byte G2 images are only 8-byte aligned per element: read as u64.
__device__ __forceinline__ G1Affine load_g1_image(const uint8_t *img) {
    const uint64_t *w = (const uint64_t *)img;
    G1Affine p;
    if (img[96]) return G1Affine::inf();
#pragma unroll
    for (int i = 0; i < 6; i++) {
        uint64_t vx = w[i], vy = w[6 + i];
        p.x.l[2 * i] = (uint32_t)vx; p.x.l[2 * i + 1] = (uint32_t)(vx >> 32);
        p.y.l[2 * i] = (uint32_t)vy; p.y.l[2 * i + 1] = (uint32_t)(vy >> 32);
    }
    return p;
}
__device__ __forceinline__ void store_g1_image(uint8_t *img, const G1Affine &p) {
    uint64_t *w = (uint64_t *)img;
    if (p.is_inf()) {
        Fp one = Fp::one();
#pragma unroll
        for (int i = 0; i < 6; i++) { w[i] = 0; w[6 + i] = (uint64_t)one.l[2 * i] | ((uint64_t)one.l[2 * i + 1] << 32); }
        w[12] = 1;
        return;
    }
#pragma unroll
    for (int i = 0; i < 6; i++) {
        w[i] = (uint64_t)p.x.l[2 * i] | ((uint64_t)p.x.l[2 * i + 1] << 32);
        w[6 + i] = (uint64_t)p.y.l[2 * i] | ((uint64_t)p.y.l[2 * i + 1] << 32);
    }
    w[12] = 0;
}
__device__ __forceinline__ G2Affine load_g2_image(const uint8_t *img) {
    const uint64_t *w = (const uint64_t *)img;
    G2Affine p;
    if (img[192]) return G2Affine::inf();
    Fp *f[4] = {&p.x.c0, &p.x.c1, &p.y.c0, &p.y.c1};
#pragma unroll
    for (int k = 0; k < 4; k++)
#pragma unroll
        for (int i = 0; i < 6; i++) {
            uint64_t v = w[6 * k + i];
            f[k]->l[2 * i] = (uint32_t)v; f[k]->l[2 * i + 1] = (uint32_t)(v >> 32);
        }
    return p;
}
__device__ __forceinline__ void store_g2_image(uint8_t *img, const G2Affine &p) {
    uint64_t *w = (uint64_t *)img;
    if (p.is_inf()) {
        Fp one = Fp::one();
#pragma unroll
        for (int i = 0; i < 24; i++) w[i] = 0;
#pragma unroll
        for (int i = 0; i < 6; i++) w[12 + i] = (uint64_t)one.l[2 * i] | ((uint64_t)one.l[2 * i + 1] << 32);
        w[24] = 1;
        return;
    }
    const Fp *f[4] = {&p.x.c0, &p.x.c1, &p.y.c0, &p.y.c1};
#pragma unroll
    for (int k = 0; k < 4; k++)
#pragma unroll
        for (int i = 0; i < 6; i++) w[6 * k + i] = (uint64_t)f[k]->l[2 * i] | ((uint64_t)f[k]->l[2 * i + 1] << 32);
    w[24] = 0;
}

// ---- wire <-> packed conversions (host): bzk_g1_affine / bzk_g2_affine <-> G1Affine / G2Affine --------------------------
// The same images as above; the identity is written with y = Montgomery one and the flag set.
inline G1Affine from_wire(const bzk_g1_affine *img) {
    if (img->infinity) return G1Affine::inf();
    G1Affine p;
    memcpy(p.x.l, img->x, 48);
    memcpy(p.y.l, img->y, 48);
    return p;
}
inline G2Affine from_wire(const bzk_g2_affine *img) {
    if (img->infinity) return G2Affine::inf();
    G2Affine p;
    memcpy(p.x.c0.l, img->x, 48); memcpy(p.x.c1.l, img->x + 6, 48);
    memcpy(p.y.c0.l, img->y, 48); memcpy(p.y.c1.l, img->y + 6, 48);
    return p;
}
inline void to_wire(bzk_g1_affine *img, const G1Affine &p) {
    memset(img, 0, sizeof *img);
    if (p.is_inf()) { const Fp one = Fp::one(); memcpy(img->y, one.l, 48); img->infinity = 1; return; }
    memcpy(img->x, p.x.l, 48);
    memcpy(img->y, p.y.l, 48);
}
inline void to_wire(bzk_g2_affine *img, const G2Affine &p) {
    memset(img, 0, sizeof *img);
    if (p.is_inf()) { const Fp one = Fp::one(); memcpy(img->y, one.l, 48); img->infinity = 1; return; }
    memcpy(img->x, p.x.c0.l, 48); memcpy(img->x + 6, p.x.c1.l, 48);
    memcpy(img->y, p.y.c0.l, 48); memcpy(img->y + 6, p.y.c1.l, 48);
}

// 128-bit vector load/store of a field element / packed point from 16-byte aligned memory
template <class T>
__device__ __forceinline__ T load_vec(const T *p) {
    static_assert(sizeof(T) % 16 == 0, "16-byte multiple");
    T r;
    const uint4 *s = (const uint4 *)p;
    uint4 *d = (uint4 *)&r;
#pragma unroll
    for (int i = 0; i < (int)(sizeof(T) / 16); i++) d[i] = __ldg(s + i);
    return r;
}
template <class T>
__device__ __forceinline__ void store_vec(T *p, const T &v) {
    static_assert(sizeof(T) % 16 == 0, "16-byte multiple");
    uint4 *d = (uint4 *)p;
    const uint4 *s = (const uint4 *)&v;
#pragma unroll
    for (int i = 0; i < (int)(sizeof(T) / 16); i++) d[i] = s[i];
}

// SplitMix64 draw #idx of stream `seed` without iterating (state after k steps = seed + k*gamma)
__host__ __device__ __forceinline__ uint64_t splitmix_at(uint64_t seed, uint64_t k) {
    uint64_t z = seed + (k + 1) * 0x9E3779B97F4A7C15ULL;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
    return z ^ (z >> 31);
}
// i-th Fr of the stream: 4 draws -> 256-bit LE integer mod r (canonical, not Montgomery)
__host__ __device__ __forceinline__ Fr splitmix_fr_canonical(uint64_t seed, uint64_t i) {
    Fr v;
#pragma unroll
    for (int k = 0; k < 4; k++) {
        uint64_t d = splitmix_at(seed, 4 * i + k);
        v.l[2 * k] = (uint32_t)d;
        v.l[2 * k + 1] = (uint32_t)(d >> 32);
    }
    // v < 2^256 < 5r: at most 4 conditional subtractions (v < 2r is required by reduce_once only
    // for its "no carry" argument on addition, not here: it is a plain compare-and-subtract)
    for (int k = 0; k < 4; k++) v = Fr::reduce_once(v);
    return v;
}

}  // namespace bzk

// kernels' host entry points implemented across the .cu files
namespace bzk {
int32_t poseidon_launch(bzk_ctx *ctx, uint32_t arity, const Fr *d_in, size_t n, Fr *d_out);
int32_t ntt_launch(bzk_ctx *ctx, Fr *d, uint32_t log_n, int32_t op);
}  // namespace bzk
