// bazuka_b200 — Ed25519 signature checks (ed25519-dalek 1.x `PublicKey::verify`, the reference's `Ed25519::verify`) in batches
// on the GPU: what a node runs on the L1 signature of every MPN deposit (`ContractDeposit::verify_signature`,
// src/core/transaction.rs:192-201) and of every `TransactionAndDelta` (src/core/transaction.rs:386-397), for a whole batch at
// once instead of one signature per host call.
//
// One thread per signature, two kernels per chunk of items:
//   prepare  s < l, A decompressed (sqrt_ratio_i by the (p-5)/8 power), k = SHA-512(R || pk || M) mod l;
//   verify   [k](-A) by a 4-bit window, [s]B from the context's fixed-base table of B, compress the sum (one inversion) and
//            compare it with the signature's R bytes.
// Messages have any length: they travel as one byte buffer and n + 1 offsets.  The arithmetic and the predicate are
// ed25519.cuh's, the text the host call bzk_ed25519_verify runs too.
#include <algorithm>

#include "common.cuh"
#include "ed25519.cuh"
#include "mpn_wire.cuh"

namespace bzk {
namespace {

// a chunk holds at most this many items and, unless one message alone is longer, this many message bytes: about 180 MB of
// device memory at most
constexpr size_t kEdChunk = size_t(1) << 18;
constexpr uint64_t kEdChunkBytes = uint64_t(1) << 26;

// a[i] = (A.x, A.y) Montgomery, k[i] = SHA-512(R || pk || M) mod l (plain), flag[i] = s < l and A decompresses.  Message i is
// msgs[offs[i] - base .. offs[i + 1] - base).
__global__ void __launch_bounds__(128) k_ed25519_prepare(const uint8_t *__restrict__ pks, const uint8_t *__restrict__ sigs, const uint8_t *__restrict__ msgs,
                                                         const uint64_t *__restrict__ offs, uint64_t base, size_t n, Fe25519 *__restrict__ a,
                                                         Sc25519 *__restrict__ k, uint8_t *__restrict__ flag) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t lo = offs[i], hi = offs[i + 1];
    Fe25519 ax = Fe25519::zero(), ay = Fe25519::zero();
    Sc25519 kk = Sc25519::zero();
    const bool ok = ed25519_prepare(pks + 32 * i, sigs + 64 * i, msgs + (lo - base), hi - lo, &ax, &ay, &kk);
    store_vec(a + 2 * i, ax);
    store_vec(a + 2 * i + 1, ay);
    store_vec(k + i, kk);
    flag[i] = ok;
}

__global__ void __launch_bounds__(128) k_ed25519_verify(const Fe25519 *__restrict__ a, const Sc25519 *__restrict__ k, const uint8_t *__restrict__ sigs,
                                                        const uint8_t *__restrict__ flag, const EdNiels25519 *__restrict__ tab, size_t n,
                                                        uint8_t *__restrict__ ok) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (!flag[i]) { ok[i] = 0; return; }
    ok[i] = ed25519_finish(load_vec(a + 2 * i), load_vec(a + 2 * i + 1), load_vec(k + i), sigs + 64 * i, tab);
}

int32_t ensure_table(bzk_ctx *ctx) {
    if (ctx->d_ed_table) return BZK_OK;
    const std::vector<EdNiels25519> tab = ed_base_table();
    const size_t bytes = tab.size() * sizeof(EdNiels25519);
    void *d = nullptr;
    BZK_CUDA(ctx, cudaMalloc(&d, bytes));
    const cudaError_t e = cudaMemcpyAsync(d, tab.data(), bytes, cudaMemcpyHostToDevice, ctx->stream);
    const cudaError_t s = e == cudaSuccess ? cudaStreamSynchronize(ctx->stream) : e;
    if (s != cudaSuccess) {
        cudaFree(d);
        return set_cuda_err(ctx, s, "ed25519 table upload", __FILE__, __LINE__);
    }
    ctx->d_ed_table = d;
    return BZK_OK;
}

bool offsets_ok(const uint64_t *offs, size_t n) {
    if (offs[0] != 0) return false;
    for (size_t i = 0; i < n; i++)
        if (offs[i + 1] < offs[i]) return false;
    return true;
}

// The arguments are checked; n > 0.
int32_t verify_batch(bzk_ctx *ctx, const uint8_t *pks, const uint8_t *sigs, const uint8_t *msgs, const uint64_t *offs, size_t n, uint8_t *ok,
                     uint64_t *n_ok) {
    BZK_CUDA(ctx, cudaSetDevice(ctx->device));
    BZK_TRY(ensure_table(ctx));
    cudaStream_t st = ctx->stream;
    uint64_t accepted = 0;
    for (size_t off = 0; off < n;) {
        // as many items as fit both bounds, at least one
        const size_t cap = std::min(n - off, kEdChunk);
        const uint64_t base = offs[off];
        size_t m = (size_t)(std::upper_bound(offs + off + 1, offs + off + cap + 1, base + kEdChunkBytes) - (offs + off + 1));
        if (m == 0) m = 1;
        const uint64_t bytes = offs[off + m] - base;
        auto carve = [&](Carver &c, uint8_t **d_pks, uint8_t **d_sigs, uint8_t **d_msgs, uint64_t **d_offs, Fe25519 **d_a, Sc25519 **d_k, uint8_t **d_flag,
                         uint8_t **d_ok) {
            *d_pks = c.take<uint8_t>(32 * m);
            *d_sigs = c.take<uint8_t>(64 * m);
            *d_msgs = c.take<uint8_t>(bytes);
            *d_offs = c.take<uint64_t>(m + 1);
            *d_a = c.take<Fe25519>(2 * m);
            *d_k = c.take<Sc25519>(m);
            *d_flag = c.take<uint8_t>(m);
            *d_ok = c.take<uint8_t>(m);
        };
        uint8_t *d_pks, *d_sigs, *d_msgs, *d_flag, *d_ok;
        uint64_t *d_offs;
        Fe25519 *d_a;
        Sc25519 *d_k;
        Carver size(nullptr);
        carve(size, &d_pks, &d_sigs, &d_msgs, &d_offs, &d_a, &d_k, &d_flag, &d_ok);
        BZK_TRY(ensure_ws(ctx, &ctx->ws, &ctx->ws_bytes, size.used()));
        Carver c(ctx->ws);
        carve(c, &d_pks, &d_sigs, &d_msgs, &d_offs, &d_a, &d_k, &d_flag, &d_ok);
        BZK_CUDA(ctx, cudaMemcpyAsync(d_pks, pks + 32 * off, 32 * m, cudaMemcpyHostToDevice, st));
        BZK_CUDA(ctx, cudaMemcpyAsync(d_sigs, sigs + 64 * off, 64 * m, cudaMemcpyHostToDevice, st));
        if (bytes) BZK_CUDA(ctx, cudaMemcpyAsync(d_msgs, msgs + base, bytes, cudaMemcpyHostToDevice, st));
        BZK_CUDA(ctx, cudaMemcpyAsync(d_offs, offs + off, (m + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, st));
        const unsigned blocks = div_up(m, 128);
        k_ed25519_prepare<<<blocks, 128, 0, st>>>(d_pks, d_sigs, d_msgs, d_offs, base, m, d_a, d_k, d_flag);
        BZK_LAUNCHED(ctx);
        k_ed25519_verify<<<blocks, 128, 0, st>>>(d_a, d_k, d_sigs, d_flag, (const EdNiels25519 *)ctx->d_ed_table, m, d_ok);
        BZK_LAUNCHED(ctx);
        BZK_CUDA(ctx, cudaMemcpyAsync(ok + off, d_ok, m, cudaMemcpyDeviceToHost, st));
        BZK_CUDA(ctx, cudaStreamSynchronize(st));
        for (size_t j = 0; j < m; j++) accepted += ok[off + j];
        off += m;
    }
    if (n_ok) *n_ok = accepted;
    return BZK_OK;
}

}  // namespace
}  // namespace bzk

using namespace bzk;

extern "C" {

int32_t bzk_ed25519_verify(const uint8_t pk[32], const uint8_t *msg, size_t len, const uint8_t sig[64]) {
    if (!pk || !sig || (len && !msg)) return BZK_ERR_BAD_ARG;
    static const std::vector<EdNiels25519> tab = ed_base_table();
    Fe25519 ax, ay;
    Sc25519 k;
    if (!ed25519_prepare(pk, sig, msg, len, &ax, &ay, &k)) return 0;
    return ed25519_finish(ax, ay, k, sig, tab.data()) ? 1 : 0;
}

int32_t bzk_ed25519_verify_batch(bzk_ctx *ctx, const uint8_t *pks, const uint8_t *sigs, const uint8_t *msgs, const uint64_t *offsets, size_t n,
                                 uint8_t *ok, uint64_t *n_ok) {
    if (!ctx || (n && (!pks || !sigs || !offsets || !ok))) return BZK_ERR_BAD_ARG;
    if (n && (!offsets_ok(offsets, n) || (offsets[n] && !msgs))) return BZK_ERR_BAD_ARG;
    if (n_ok) *n_ok = 0;
    if (n == 0) return BZK_OK;
    return verify_batch(ctx, pks, sigs, msgs, offsets, n, ok, n_ok);
}

int32_t bzk_mpn_deposits_verify_bytes(bzk_ctx *ctx, const uint8_t *bytes, size_t len, uint8_t *ok, size_t cap, uint64_t *n, uint64_t *n_ok) {
    if (!ctx || !n || (len && !bytes)) return BZK_ERR_BAD_ARG;
    std::vector<wire::MpnDeposit> deps;
    if (!wire::dec_deposits(bytes, len, deps)) return BZK_ERR_BAD_ARG;
    const size_t count = deps.size();
    *n = count;
    if (!ok) return BZK_OK;
    if (cap < count) return BZK_ERR_BAD_ARG;
    if (n_ok) *n_ok = 0;
    // sig None or not 64 bytes: 0 without a check (in the reference such a deposit has no signature, or does not deserialize)
    std::vector<size_t> idx;
    std::vector<uint8_t> pks, sigs;
    std::vector<uint64_t> offs(1, 0);
    wire::Writer msgs;
    for (size_t i = 0; i < count; i++) {
        const wire::ContractDeposit &p = deps[i].payment;
        if (!p.has_sig || p.sig.size() != 64) continue;
        idx.push_back(i);
        pks.insert(pks.end(), p.src, p.src + 32);
        sigs.insert(sigs.end(), p.sig.begin(), p.sig.end());
        wire::enc_contract_deposit_unsigned(msgs, p);
        offs.push_back(msgs.b.size());
    }
    std::vector<uint8_t> got(idx.size());
    if (!idx.empty()) BZK_TRY(verify_batch(ctx, pks.data(), sigs.data(), msgs.b.data(), offs.data(), idx.size(), got.data(), nullptr));
    memset(ok, 0, count);
    uint64_t accepted = 0;
    for (size_t j = 0; j < idx.size(); j++) {
        ok[idx[j]] = got[j];
        accepted += got[j];
    }
    if (n_ok) *n_ok = accepted;
    return BZK_OK;
}

}  // extern "C"
