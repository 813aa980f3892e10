// bazuka_b200 — proving keys in bellman 0.14's `Parameters` file format (`Parameters::write` / `Parameters::read`).
//
// Layout (bellman 0.14 / bls12_381 0.8, restated in oracle/py/bellman_params.py, which the tests hold this file to):
//   VerifyingKey::write   alpha_g1, beta_g1, beta_g2, gamma_g2, delta_g1, delta_g2 uncompressed,
//                         u32 big-endian |ic|, the ic points
//   then for each of h, l, a, b_g1, b_g2: u32 big-endian length, that many uncompressed points.
// Point encodings and the per-point checks: params_io.cuh.  `Parameters::read(checked)` reads the verifying key checked
// (curve + subgroup) whatever `checked` says, the five vectors checked or not, and refuses the identity anywhere in ic
// and the five vectors; nothing after b_g2 is read.  libbzk's key also needs |b_g1| == |b_g2| (bellman's generator
// always makes them so).  An unchecked read keeps an encoded (0, 0) as the identity: such a point is off the curve and
// no key bellman writes holds one.
//
// Pipeline.  Points stream through two pinned host buffers and two device buffers of kChunk = 2^16 points (12.6 MB for
// G2) each, never the whole file: the host copies chunk k+1 into one pinned buffer and a copy stream moves it to the
// device while the decode kernel of chunk k runs on the context's stream; events order the reuse of each buffer.  The
// decode kernels write the packed Montgomery points straight into the key's resident base vectors, so device memory
// beyond the key is the two chunks.  A refused point is reported through one atomicMin over (vector, index, reason): the
// first bad point in file order wins.  The writer runs the same pipeline backwards (encode kernel, D2H, host copy).
// A vector placed in host memory (bzk_groth16_params_read_placed) is decoded into a device landing chunk that is then
// copied, on the same stream, into the vector's pinned allocation; the writer copies such a vector's chunks to the device
// before it encodes them.  Device memory is then the pipe's buffers, the landing chunk and the device-placed vectors.
#include "common.cuh"
#include "params_io.cuh"
#include <algorithm>

namespace bzk {

constexpr uint32_t kChunk = 1u << 16;                 // points per staged chunk
constexpr size_t kChunkBytes = (size_t)kChunk * 192;  // a chunk of G2 images
constexpr uint64_t kNoFault = ~0ull;

// the file's point sequences in order: the verifying key's six points, ic, then the five vectors
enum { kAlphaG1, kBetaG1, kBetaG2, kGammaG2, kDeltaG1, kDeltaG2, kIc, kH, kL, kA, kBG1, kBG2, kSegs };
static const char *const kSegName[kSegs] = {"alpha_g1", "beta_g1", "beta_g2", "gamma_g2", "delta_g1", "delta_g2", "ic", "h", "l", "a", "b_g1", "b_g2"};
static bool seg_is_g2(int s) { return s == kBetaG2 || s == kGammaG2 || s == kDeltaG2 || s == kBG2; }
static size_t seg_point_bytes(int s) { return seg_is_g2(s) ? 192 : 96; }

struct Seg {
    uint64_t off = 0;  // byte offset of the first point in the file
    uint64_t n = 0;
};

static uint32_t be32(const uint8_t *p) { return ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3]; }
static void put_be32(uint8_t *p, uint32_t v) { p[0] = (uint8_t)(v >> 24); p[1] = (uint8_t)(v >> 16); p[2] = (uint8_t)(v >> 8); p[3] = (uint8_t)v; }

// Walk the lengths; BZK_ERR_BAD_ENCODING when the image ends before what it states.  *total = bytes the lengths imply.
static int32_t parse_layout(const uint8_t *b, size_t len, Seg seg[kSegs], uint64_t *total, char *why, size_t why_cap) {
    uint64_t off = 0;
    for (int s = 0; s < kSegs; s++) {
        if (s >= kIc) {
            if (off + 4 > len) {
                snprintf(why, why_cap, "truncated: the image ends (%zu bytes) before the length of %s", len, kSegName[s]);
                return BZK_ERR_BAD_ENCODING;
            }
            seg[s].n = be32(b + off);
            off += 4;
        } else {
            seg[s].n = 1;
        }
        seg[s].off = off;
        off += seg[s].n * seg_point_bytes(s);
    }
    *total = off;
    if (off > len) {
        snprintf(why, why_cap, "truncated: the lengths state %llu bytes, the image has %zu", (unsigned long long)off, len);
        return BZK_ERR_BAD_ENCODING;
    }
    return BZK_OK;
}

// subgroup-test constants, derived once (params_io.cuh)
static const EndoConsts *endo_consts() {
    static EndoConsts c;
    static const bool ok = derive_endo_consts(&c);
    return ok ? &c : nullptr;
}

// ---- kernels ---------------------------------------------------------------------------------------------------------
template <class A, int W>  // W: 32-bit words per image (24 G1, 48 G2)
__global__ void __launch_bounds__(128) k_decode(const uint8_t *__restrict__ src, uint32_t n, uint64_t first, uint64_t seg, uint32_t checked,
                                                uint32_t allow_inf, EndoConsts k, A *__restrict__ dst, unsigned long long *fault) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t w[W];
    const uint4 *s = (const uint4 *)(src + (size_t)i * (W * 4));
#pragma unroll
    for (int j = 0; j < W / 4; j++) {
        const uint4 v = s[j];
        w[4 * j] = v.x; w[4 * j + 1] = v.y; w[4 * j + 2] = v.z; w[4 * j + 3] = v.w;
    }
    A p;
    const uint32_t f = decode_point(w, checked != 0, allow_inf != 0, k, p);
    if (f != kPointOk) {
        atomicMin(fault, (unsigned long long)((seg << 40) | ((first + i) << 8) | f));
        return;
    }
    store_vec(dst + i, p);
}

template <class A, int W>
__global__ void __launch_bounds__(128) k_encode(const A *__restrict__ src, uint32_t n, uint8_t *__restrict__ dst) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t w[W];
    encode_point(load_vec(src + i), w);
    uint4 *d = (uint4 *)(dst + (size_t)i * (W * 4));
#pragma unroll
    for (int j = 0; j < W / 4; j++) d[j] = make_uint4(w[4 * j], w[4 * j + 1], w[4 * j + 2], w[4 * j + 3]);
}

// ---- the double-buffered staging pipeline ----------------------------------------------------------------------------
struct Pipe {
    bzk_ctx *ctx;
    cudaStream_t copy = nullptr;
    uint8_t *pin[2] = {nullptr, nullptr}, *dev[2] = {nullptr, nullptr};
    cudaEvent_t done[2] = {nullptr, nullptr}, copied[2] = {nullptr, nullptr};  // kernel / copy that last used buffer b
    int next = 0;

    explicit Pipe(bzk_ctx *c) : ctx(c) {}
    int32_t open() {
        BZK_CUDA(ctx, cudaStreamCreateWithFlags(&copy, cudaStreamNonBlocking));
        for (int b = 0; b < 2; b++) {
            BZK_CUDA(ctx, cudaHostAlloc(&pin[b], kChunkBytes, cudaHostAllocDefault));
            BZK_CUDA(ctx, cudaMalloc(&dev[b], kChunkBytes));
            BZK_CUDA(ctx, cudaEventCreateWithFlags(&done[b], cudaEventDisableTiming));
            BZK_CUDA(ctx, cudaEventCreateWithFlags(&copied[b], cudaEventDisableTiming));
        }
        return BZK_OK;
    }
    ~Pipe() {
        if (copy) cudaStreamSynchronize(copy);
        cudaStreamSynchronize(ctx->stream);
        for (int b = 0; b < 2; b++) {
            if (pin[b]) cudaFreeHost(pin[b]);
            if (dev[b]) cudaFree(dev[b]);
            if (done[b]) cudaEventDestroy(done[b]);
            if (copied[b]) cudaEventDestroy(copied[b]);
        }
        if (copy) cudaStreamDestroy(copy);
    }

    // host bytes -> device chunk -> decode kernel
    int32_t decode(const uint8_t *src, int seg, uint64_t first, uint32_t n, bool checked, const EndoConsts &k, void *dst, unsigned long long *fault) {
        const int b = next;
        next ^= 1;
        const size_t bytes = (size_t)n * seg_point_bytes(seg);
        BZK_CUDA(ctx, cudaEventSynchronize(done[b]));  // the kernel that last read dev[b] (so also the copy from pin[b]) is done
        memcpy(pin[b], src, bytes);
        BZK_CUDA(ctx, cudaMemcpyAsync(dev[b], pin[b], bytes, cudaMemcpyHostToDevice, copy));
        BZK_CUDA(ctx, cudaEventRecord(copied[b], copy));
        BZK_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, copied[b], 0));
        const bool chk = checked || seg <= kIc;  // the verifying key (ic included) is always read checked
        const uint32_t allow_inf = seg < kIc;    // the identity is refused in ic and the five vectors
        if (seg_is_g2(seg))
            k_decode<G2Affine, 48><<<div_up(n, 128), 128, 0, ctx->stream>>>(dev[b], n, first, (uint64_t)seg, chk, allow_inf, k, (G2Affine *)dst, fault);
        else
            k_decode<G1Affine, 24><<<div_up(n, 128), 128, 0, ctx->stream>>>(dev[b], n, first, (uint64_t)seg, chk, allow_inf, k, (G1Affine *)dst, fault);
        BZK_LAUNCHED(ctx);
        BZK_CUDA(ctx, cudaEventRecord(done[b], ctx->stream));
        return BZK_OK;
    }

    // encode kernel -> device chunk -> pinned buffer; the host copy out happens one chunk later (drain)
    struct Pending {
        int b = -1;
        uint8_t *out = nullptr;
        size_t bytes = 0;
    } pending;
    int32_t drain() {
        if (pending.b < 0) return BZK_OK;
        BZK_CUDA(ctx, cudaEventSynchronize(copied[pending.b]));
        memcpy(pending.out, pin[pending.b], pending.bytes);
        pending.b = -1;
        return BZK_OK;
    }
    int32_t encode(const void *src, int seg, uint32_t n, uint8_t *out) {
        const int b = next;
        next ^= 1;
        const size_t bytes = (size_t)n * seg_point_bytes(seg);
        // dev[b] / pin[b] were last used two chunks ago and drained one chunk ago
        if (seg_is_g2(seg))
            k_encode<G2Affine, 48><<<div_up(n, 128), 128, 0, ctx->stream>>>((const G2Affine *)src, n, dev[b]);
        else
            k_encode<G1Affine, 24><<<div_up(n, 128), 128, 0, ctx->stream>>>((const G1Affine *)src, n, dev[b]);
        BZK_LAUNCHED(ctx);
        BZK_CUDA(ctx, cudaEventRecord(done[b], ctx->stream));
        BZK_CUDA(ctx, cudaStreamWaitEvent(copy, done[b], 0));
        BZK_CUDA(ctx, cudaMemcpyAsync(pin[b], dev[b], bytes, cudaMemcpyDeviceToHost, copy));
        BZK_CUDA(ctx, cudaEventRecord(copied[b], copy));
        BZK_TRY(drain());
        pending.b = b;
        pending.out = out;
        pending.bytes = bytes;
        return BZK_OK;
    }
};

static const char *fault_text(uint32_t f) {
    switch (f) {
        case kCompressionFlag: return "compression flag set";
        case kSortFlag: return "sort flag set";
        case kXNotCanonical: return "x coordinate not below p";
        case kYNotCanonical: return "y coordinate not below p";
        case kInfinityWithBits: return "infinity flag with coordinate bits set";
        case kPointAtInfinity: return "point at infinity";
        case kNotOnCurve: return "not on the curve";
        case kNotInSubgroup: return "not in the prime-order subgroup";
        default: return "bad point";
    }
}
static int32_t fault_status(uint32_t f) {
    return f == kNotOnCurve ? BZK_ERR_NOT_ON_CURVE : f == kNotInSubgroup ? BZK_ERR_NOT_IN_SUBGROUP : BZK_ERR_BAD_ENCODING;
}

}  // namespace bzk

using namespace bzk;

extern "C" {

int32_t bzk_groth16_params_file_info(const uint8_t *bytes, size_t len, bzk_params_file_info *out) {
    if (!out || (len && !bytes)) return BZK_ERR_BAD_ARG;
    Seg seg[kSegs];
    uint64_t total = 0;
    char why[160];
    BZK_TRY(parse_layout(bytes, len, seg, &total, why, sizeof why));
    out->n_ic = seg[kIc].n; out->n_h = seg[kH].n; out->n_l = seg[kL].n; out->n_a = seg[kA].n;
    out->n_b_g1 = seg[kBG1].n; out->n_b_g2 = seg[kBG2].n; out->bytes = total;
    return BZK_OK;
}

int32_t bzk_groth16_params_read_placed(bzk_ctx *ctx, const uint8_t *bytes, size_t len, int32_t checked, bzk_g1_affine *alpha_g1,
                                       bzk_g1_affine *beta_g1, bzk_g2_affine *beta_g2, bzk_g2_affine *gamma_g2, bzk_g1_affine *delta_g1,
                                       bzk_g2_affine *delta_g2, bzk_g1_affine *ic, size_t ic_cap, uint32_t host_mask, bzk_groth16_params **out) {
    if (!ctx || !out || (len && !bytes) || !alpha_g1 || !beta_g1 || !beta_g2 || !gamma_g2 || !delta_g1 || !delta_g2 || host_mask > 31)
        return BZK_ERR_BAD_ARG;
    *out = nullptr;
    BZK_CUDA(ctx, cudaSetDevice(ctx->device));
    Seg seg[kSegs];
    uint64_t total = 0;
    BZK_TRY(parse_layout(bytes, len, seg, &total, ctx->err, sizeof ctx->err));
    if (seg[kBG1].n != seg[kBG2].n) {
        snprintf(ctx->err, sizeof ctx->err, "b_g1 has %llu points and b_g2 %llu: the key needs them equal", (unsigned long long)seg[kBG1].n,
                 (unsigned long long)seg[kBG2].n);
        return BZK_ERR_BAD_ENCODING;
    }
    if (ic_cap < seg[kIc].n || (seg[kIc].n && !ic)) return BZK_ERR_BAD_ARG;
    const EndoConsts *k = endo_consts();
    if (!k) {
        snprintf(ctx->err, sizeof ctx->err, "subgroup-test constants failed their self-check");
        return BZK_ERR_CUDA;
    }

    // destinations: the five vectors (device or pinned host memory, as host_mask says), and a scratch block for the
    // verifying key's points and the landing chunk of the host-placed vectors
    bzk_g1_bases *g1v[4] = {nullptr, nullptr, nullptr, nullptr};
    bzk_g2_bases *b2 = nullptr;
    void *scratch = nullptr;
    auto release = [&]() {
        cudaStreamSynchronize(ctx->stream);
        for (auto *b : g1v) if (b) bases_release(b);
        if (b2) bases_release(b2);
        if (scratch) cudaFree(scratch);
    };
    int32_t st = BZK_OK;
    const uint64_t n_ic = seg[kIc].n;
    const size_t landing_bytes = host_mask ? (size_t)kChunk * sizeof(G2Affine) : 0;
    const size_t scratch_bytes = 256 + 3 * sizeof(G1Affine) + 3 * sizeof(G2Affine) + (n_ic ? n_ic : 1) * sizeof(G1Affine) + landing_bytes + 4 * 256;
    cudaError_t e = cudaMalloc(&scratch, scratch_bytes);
    if (e != cudaSuccess) {
        st = set_cuda_err(ctx, e, "cudaMalloc(proving key)", __FILE__, __LINE__);
        release();
        return st;
    }
    for (int v = 0; v < 4 && st == BZK_OK; v++) {
        g1v[v] = new (std::nothrow) bzk_g1_bases();
        if (!g1v[v]) { release(); return BZK_ERR_OOM; }
        g1v[v]->n = seg[kH + v].n;
        st = bases_alloc(ctx, g1v[v], (host_mask >> v) & 1);
    }
    if (st == BZK_OK) {
        b2 = new (std::nothrow) bzk_g2_bases();
        if (!b2) { release(); return BZK_ERR_OOM; }
        b2->n = seg[kBG2].n;
        st = bases_alloc(ctx, b2, (host_mask >> 4) & 1);
    }
    if (st != BZK_OK) {
        release();
        return st;
    }
    Carver cv(scratch);
    unsigned long long *d_fault = cv.take<unsigned long long>(1);
    G1Affine *d_vk1 = cv.take<G1Affine>(3);  // alpha, beta, delta
    G2Affine *d_vk2 = cv.take<G2Affine>(3);  // beta, gamma, delta
    G1Affine *d_ic = cv.take<G1Affine>(n_ic ? n_ic : 1);
    char *landing = cv.take<char>(landing_bytes);
    auto place = [](auto *b) { return b->h ? (void *)b->h : (void *)b->d; };
    void *dst[kSegs] = {d_vk1, d_vk1 + 1, d_vk2, d_vk2 + 1, d_vk1 + 2, d_vk2 + 2, d_ic, place(g1v[0]), place(g1v[1]), place(g1v[2]), place(g1v[3]), place(b2)};

    {
        Pipe pipe(ctx);
        st = pipe.open();
        if (st == BZK_OK) {
            e = cudaMemsetAsync(d_fault, 0xff, sizeof *d_fault, ctx->stream);
            if (e != cudaSuccess) st = set_cuda_err(ctx, e, "cudaMemsetAsync", __FILE__, __LINE__);
        }
        for (int s = 0; s < kSegs && st == BZK_OK; s++) {
            const size_t pb = seg_point_bytes(s), packed = seg_is_g2(s) ? sizeof(G2Affine) : sizeof(G1Affine);
            const bool on_host = s >= kH && ((host_mask >> (s - kH)) & 1);
            for (uint64_t i = 0; i < seg[s].n && st == BZK_OK; i += kChunk) {
                const uint32_t n = (uint32_t)std::min<uint64_t>(kChunk, seg[s].n - i);
                char *d = (char *)dst[s] + i * packed;
                st = pipe.decode(bytes + seg[s].off + i * pb, s, i, n, checked != 0, *k, on_host ? landing : d, d_fault);
                // the landing chunk's next decode is behind this copy on the same stream
                if (st == BZK_OK && on_host) {
                    e = cudaMemcpyAsync(d, landing, n * packed, cudaMemcpyDeviceToHost, ctx->stream);
                    if (e != cudaSuccess) st = set_cuda_err(ctx, e, "cudaMemcpyAsync(host vector)", __FILE__, __LINE__);
                }
            }
        }
    }  // the pipe synchronises both streams and releases its buffers
    unsigned long long fault = kNoFault;
    if (st == BZK_OK) {
        e = cudaMemcpy(&fault, d_fault, sizeof fault, cudaMemcpyDeviceToHost);
        if (e != cudaSuccess) st = set_cuda_err(ctx, e, "cudaMemcpy(fault)", __FILE__, __LINE__);
    }
    if (st == BZK_OK && fault != kNoFault) {
        const uint32_t s = (uint32_t)(fault >> 40), f = (uint32_t)(fault & 0xff);
        const unsigned long long idx = (fault >> 8) & 0xffffffffull;
        snprintf(ctx->err, sizeof ctx->err, "%s[%llu]: %s", s < kSegs ? kSegName[s] : "?", idx, fault_text(f));
        st = fault_status(f);
    }
    G1Affine vk1[3];
    G2Affine vk2[3];
    std::vector<G1Affine> ic_pts(n_ic);
    if (st == BZK_OK) {
        e = cudaMemcpy(vk1, d_vk1, sizeof vk1, cudaMemcpyDeviceToHost);
        if (e == cudaSuccess) e = cudaMemcpy(vk2, d_vk2, sizeof vk2, cudaMemcpyDeviceToHost);
        if (e == cudaSuccess && n_ic) e = cudaMemcpy(ic_pts.data(), d_ic, n_ic * sizeof(G1Affine), cudaMemcpyDeviceToHost);
        if (e != cudaSuccess) st = set_cuda_err(ctx, e, "cudaMemcpy(verifying key)", __FILE__, __LINE__);
    }
    if (st != BZK_OK) {
        release();
        return st;
    }
    cudaFree(scratch);
    scratch = nullptr;
    to_wire(alpha_g1, vk1[0]); to_wire(beta_g1, vk1[1]); to_wire(delta_g1, vk1[2]);
    to_wire(beta_g2, vk2[0]); to_wire(gamma_g2, vk2[1]); to_wire(delta_g2, vk2[2]);
    for (uint64_t i = 0; i < n_ic; i++) to_wire(ic + i, ic_pts[i]);
    st = bzk_groth16_params_create(ctx, alpha_g1, beta_g1, beta_g2, delta_g1, delta_g2, g1v[0], g1v[1], g1v[2], g1v[3], b2, out);
    if (st != BZK_OK) release();
    return st;
}

int32_t bzk_groth16_params_read(bzk_ctx *ctx, const uint8_t *bytes, size_t len, int32_t checked, bzk_g1_affine *alpha_g1, bzk_g1_affine *beta_g1,
                                bzk_g2_affine *beta_g2, bzk_g2_affine *gamma_g2, bzk_g1_affine *delta_g1, bzk_g2_affine *delta_g2, bzk_g1_affine *ic,
                                size_t ic_cap, bzk_groth16_params **out) {
    return bzk_groth16_params_read_placed(ctx, bytes, len, checked, alpha_g1, beta_g1, beta_g2, gamma_g2, delta_g1, delta_g2, ic, ic_cap, 0, out);
}

int32_t bzk_groth16_params_write(bzk_ctx *ctx, const bzk_groth16_params *params, const bzk_g2_affine *gamma_g2, const bzk_g1_affine *ic, size_t n_ic,
                                 uint8_t *out, size_t cap, size_t *len) {
    if (!ctx || !params || !gamma_g2 || (n_ic && !ic) || !len) return BZK_ERR_BAD_ARG;
    if (params->world != 1) {
        snprintf(ctx->err, sizeof ctx->err, "a shard (rank %u of %u) holds part of each vector: it has no file image", params->rank, params->world);
        return BZK_ERR_BAD_ARG;
    }
    Seg seg[kSegs];
    const uint64_t lens[kSegs] = {1, 1, 1, 1, 1, 1, n_ic, params->h->n, params->l->n, params->a->n, params->b1->n, params->b2->n};
    uint64_t off = 0;
    for (int s = 0; s < kSegs; s++) {
        if (lens[s] > 0xffffffffull) return BZK_ERR_BAD_ARG;  // lengths are u32 on file
        if (s >= kIc) off += 4;
        seg[s].off = off;
        seg[s].n = lens[s];
        off += lens[s] * seg_point_bytes(s);
    }
    *len = off;
    if (!out) return BZK_OK;
    if (cap < off) return BZK_ERR_BAD_ARG;
    BZK_CUDA(ctx, cudaSetDevice(ctx->device));
    for (int s = kIc; s < kSegs; s++) put_be32(out + seg[s].off - 4, (uint32_t)seg[s].n);

    // the verifying key's points go through the same kernels from a scratch block
    std::vector<G1Affine> vk1(3 + n_ic);
    G2Affine vk2[3] = {params->beta_g2, from_wire(gamma_g2), params->delta_g2};
    vk1[0] = params->alpha_g1; vk1[1] = params->beta_g1; vk1[2] = params->delta_g1;
    for (size_t i = 0; i < n_ic; i++) vk1[3 + i] = from_wire(ic + i);
    // ... and a host-resident vector's chunks through a landing chunk on the device
    const bool any_host = params->h->h || params->l->h || params->a->h || params->b1->h || params->b2->h;
    const size_t landing_bytes = any_host ? (size_t)kChunk * sizeof(G2Affine) : 0;
    void *scratch = nullptr;
    Carver sizer(nullptr);
    sizer.take<G1Affine>(vk1.size()); sizer.take<G2Affine>(3); sizer.take<char>(landing_bytes);
    BZK_CUDA(ctx, cudaMalloc(&scratch, sizer.used()));
    Carver cv(scratch);
    G1Affine *d_vk1 = cv.take<G1Affine>(vk1.size());
    G2Affine *d_vk2 = cv.take<G2Affine>(3);
    char *landing = cv.take<char>(landing_bytes);
    auto place = [](const auto *b) { return b->h ? (const void *)b->h : (const void *)b->d; };
    const void *src[kSegs] = {d_vk1, d_vk1 + 1, d_vk2, d_vk2 + 1, d_vk1 + 2, d_vk2 + 2, d_vk1 + 3,
                              place(params->h), place(params->l), place(params->a), place(params->b1), place(params->b2)};
    const bool seg_host[kSegs] = {false, false, false, false, false, false, false,
                                  params->h->h != nullptr, params->l->h != nullptr, params->a->h != nullptr, params->b1->h != nullptr, params->b2->h != nullptr};
    int32_t st = BZK_OK;
    cudaError_t e = cudaMemcpyAsync(d_vk1, vk1.data(), vk1.size() * sizeof(G1Affine), cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_vk2, vk2, sizeof vk2, cudaMemcpyHostToDevice, ctx->stream);
    if (e != cudaSuccess) st = set_cuda_err(ctx, e, "cudaMemcpyAsync(verifying key)", __FILE__, __LINE__);
    {
        Pipe pipe(ctx);
        if (st == BZK_OK) st = pipe.open();
        for (int s = 0; s < kSegs && st == BZK_OK; s++) {
            const size_t pb = seg_point_bytes(s), packed = seg_is_g2(s) ? sizeof(G2Affine) : sizeof(G1Affine);
            for (uint64_t i = 0; i < seg[s].n && st == BZK_OK; i += kChunk) {
                const uint32_t n = (uint32_t)std::min<uint64_t>(kChunk, seg[s].n - i);
                const char *from = (const char *)src[s] + i * packed;
                if (seg_host[s]) {
                    // the previous chunk's encode kernel read the landing chunk earlier on the same stream
                    e = cudaMemcpyAsync(landing, from, n * packed, cudaMemcpyHostToDevice, ctx->stream);
                    if (e != cudaSuccess) { st = set_cuda_err(ctx, e, "cudaMemcpyAsync(host vector)", __FILE__, __LINE__); break; }
                    from = landing;
                }
                st = pipe.encode(from, s, n, out + seg[s].off + i * pb);
            }
        }
        if (st == BZK_OK) st = pipe.drain();
    }
    cudaFree(scratch);
    return st;
}

}  // extern "C"
