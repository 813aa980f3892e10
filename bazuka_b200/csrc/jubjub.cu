// bazuka_b200 — EdDSA-Poseidon signature checks of JubJub in batches on the GPU: what a node runs on every MPN transaction and
// withdrawal entering its mempool (`MpnTransaction::verify_signature`, src/zk/mod.rs:609-627; `MpnWithdraw::verify_signature`,
// src/core/transaction.rs:183-189), for a whole peer response at once instead of one signature per host call.
//
// One thread per signature, in three steps per chunk of items:
//   prepare  canonical checks, key decompression (Tonelli-Shanks on the device), the rows of the hashes;
//   hashes   the transaction message (Poseidon-7) or the withdrawal message (Poseidon-2), then h = Poseidon-5(R, A, msg), as
//            batched launches of poseidon.cu's kernels;
//   verify   A and R on the curve, [h] A + R == [s] BASE: a 4-bit window for [h] A, the context's fixed-base table for [s] BASE.
// The group law, the square root and the predicate are jubjub.cuh's, the text the host calls run too.
#include "common.cuh"
#include "jubjub.cuh"
#include "mpn_wire.cuh"

namespace bzk {
namespace {

// items per pass through the context's arena (about 190 MB of device memory for transactions)
constexpr size_t kEddsaChunk = size_t(1) << 18;

BZK_HD bool is_canonical(const Fr &v) { return Fr::reduce_once(v) == v; }

// a canonical scalar of an ABI struct (8-byte aligned), as plain limbs
__device__ __forceinline__ Fr ld_scalar(const bzk_fr *p) {
    Fr v;
#pragma unroll
    for (int k = 0; k < 4; k++) {
        const uint64_t w = p->l[k];
        v.l[2 * k] = (uint32_t)w;
        v.l[2 * k + 1] = (uint32_t)(w >> 32);
    }
    return v;
}
__device__ __forceinline__ Fr fr_u64(uint64_t v) {
    Fr a = Fr::zero();
    a.l[0] = (uint32_t)v;
    a.l[1] = (uint32_t)(v >> 32);
    return a.to_mont();
}
__device__ __forceinline__ bool decompress(const Fr &x, bool odd, const Fr &d, Fr *y) {
    Fr root;
    if (!jj_decompress_root(x, d, &root)) return false;
    *y = jj_with_parity(root, odd);
    return true;
}

// rows[i] = {R.x, R.y, A.x, A.y, msg} (Montgomery; msg from `msg` when given, else the item's), s[i] = s, flag[i] = the checks
// that precede the hash
__global__ void __launch_bounds__(128) k_eddsa_prepare_items(const bzk_eddsa_item *__restrict__ items, size_t n, const Fr *__restrict__ msg, Fr d,
                                                             Fr *__restrict__ rows, Fr *__restrict__ s_out, uint8_t *__restrict__ flag) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const bzk_eddsa_item &it = items[i];
    const Fr px = ld_scalar(&it.pk_x), m = ld_scalar(&it.message), rx = ld_scalar(&it.sig_rx), ry = ld_scalar(&it.sig_ry), s = ld_scalar(&it.sig_s);
    bool ok = is_canonical(px) && is_canonical(rx) && is_canonical(ry) && is_canonical(s) && (msg || is_canonical(m));
    const Fr ax = px.to_mont();
    Fr ay = Fr::zero();
    ok = ok && decompress(ax, it.pk_odd != 0, d, &ay);
    Fr *row = rows + i * 5;
    store_vec(row + 0, rx.to_mont());
    store_vec(row + 1, ry.to_mont());
    store_vec(row + 2, ax);
    store_vec(row + 3, ay);
    store_vec(row + 4, msg ? load_vec(msg + i) : m.to_mont());
    store_vec(s_out + i, s);
    flag[i] = ok;
}

// as above for transactions: the source key is A; tx_rows[i] = the inputs of the message hash (slot 4 of rows is filled from
// its digests)
__global__ void __launch_bounds__(128) k_eddsa_prepare_txs(const bzk_mpn_tx *__restrict__ txs, size_t n, Fr d, Fr *__restrict__ rows,
                                                           Fr *__restrict__ tx_rows, Fr *__restrict__ s_out, uint8_t *__restrict__ flag) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const bzk_mpn_tx &t = txs[i];
    const Fr src = ld_scalar(&t.src_pk_x), dst = ld_scalar(&t.dst_pk_x), at = ld_scalar(&t.amount_token_id), ft = ld_scalar(&t.fee_token_id),
             rx = ld_scalar(&t.sig_rx), ry = ld_scalar(&t.sig_ry), s = ld_scalar(&t.sig_s);
    bool ok = is_canonical(src) && is_canonical(dst) && is_canonical(at) && is_canonical(ft) && is_canonical(rx) && is_canonical(ry) && is_canonical(s);
    const Fr ax = src.to_mont(), dx = dst.to_mont();
    Fr ay = Fr::zero(), dy = Fr::zero();
    ok = ok && decompress(ax, t.src_pk_odd != 0, d, &ay) && decompress(dx, t.dst_pk_odd != 0, d, &dy);
    Fr *m = tx_rows + i * 7;
    store_vec(m + 0, fr_u64(t.nonce));
    store_vec(m + 1, dx);
    store_vec(m + 2, dy);
    store_vec(m + 3, at.to_mont());
    store_vec(m + 4, fr_u64(t.amount));
    store_vec(m + 5, ft.to_mont());
    store_vec(m + 6, fr_u64(t.fee));
    Fr *row = rows + i * 5;
    store_vec(row + 0, rx.to_mont());
    store_vec(row + 1, ry.to_mont());
    store_vec(row + 2, ax);
    store_vec(row + 3, ay);
    store_vec(s_out + i, s);
    flag[i] = ok;
}

__global__ void __launch_bounds__(128) k_eddsa_verify(const Fr *__restrict__ rows, const Fr *__restrict__ h, const Fr *__restrict__ s,
                                                      const uint8_t *__restrict__ flag, Fr d, const JJNiels *__restrict__ tab, size_t n,
                                                      uint8_t *__restrict__ ok) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (!flag[i]) { ok[i] = 0; return; }
    const Fr *row = rows + i * 5;
    const JJ sB = jj_mul_fixed(tab, load_vec(s + i));
    ok[i] = jj_eddsa_check(d, load_vec(row + 2), load_vec(row + 3), load_vec(row + 0), load_vec(row + 1), load_vec(h + i).from_mont(), sB);
}

int32_t ensure_table(bzk_ctx *ctx, const Fr &d) {
    if (ctx->d_jj_table && ctx->jj_table_d == d) return BZK_OK;
    const std::vector<JJNiels> tab = jj_fixed_base_table(d);
    const size_t bytes = tab.size() * sizeof(JJNiels);
    if (!ctx->d_jj_table) BZK_CUDA(ctx, cudaMalloc(&ctx->d_jj_table, bytes));
    BZK_CUDA(ctx, cudaMemcpyAsync(ctx->d_jj_table, tab.data(), bytes, cudaMemcpyHostToDevice, ctx->stream));
    BZK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    ctx->jj_table_d = d;
    return BZK_OK;
}

enum class Items { kEddsa, kTx };

// The arguments are checked; n > 0.  msg2 (withdrawals, kEddsa only): [n][2] Montgomery inputs of the message hashes.
int32_t verify_batch(bzk_ctx *ctx, const Fr &d, Items kind, const void *in, size_t n, const Fr *msg2, uint8_t *ok, uint64_t *n_ok) {
    BZK_CUDA(ctx, cudaSetDevice(ctx->device));
    BZK_TRY(ensure_table(ctx, d));
    const size_t item_bytes = kind == Items::kTx ? sizeof(bzk_mpn_tx) : sizeof(bzk_eddsa_item);
    cudaStream_t st = ctx->stream;
    uint64_t accepted = 0;
    for (size_t off = 0; off < n; off += kEddsaChunk) {
        const size_t m = n - off < kEddsaChunk ? n - off : kEddsaChunk;
        const bool tx = kind == Items::kTx;
        auto carve = [&](Carver &c, uint8_t **d_in, Fr **d_msg2, Fr **d_msg, Fr **d_rows, Fr **d_tx_rows, Fr **d_h, Fr **d_s, uint8_t **d_flag,
                         uint8_t **d_ok) {
            *d_in = c.take<uint8_t>(m * item_bytes);
            *d_msg2 = c.take<Fr>(msg2 ? 2 * m : 0);
            *d_msg = c.take<Fr>(m);
            *d_rows = c.take<Fr>(5 * m);
            *d_tx_rows = c.take<Fr>(tx ? 7 * m : 0);
            *d_h = c.take<Fr>(m);
            *d_s = c.take<Fr>(m);
            *d_flag = c.take<uint8_t>(m);
            *d_ok = c.take<uint8_t>(m);
        };
        uint8_t *d_in, *d_flag, *d_ok;
        Fr *d_msg2, *d_msg, *d_rows, *d_tx_rows, *d_h, *d_s;
        Carver size(nullptr);
        carve(size, &d_in, &d_msg2, &d_msg, &d_rows, &d_tx_rows, &d_h, &d_s, &d_flag, &d_ok);
        BZK_TRY(ensure_ws(ctx, &ctx->ws, &ctx->ws_bytes, size.used()));
        Carver c(ctx->ws);
        carve(c, &d_in, &d_msg2, &d_msg, &d_rows, &d_tx_rows, &d_h, &d_s, &d_flag, &d_ok);
        BZK_CUDA(ctx, cudaMemcpyAsync(d_in, (const uint8_t *)in + off * item_bytes, m * item_bytes, cudaMemcpyHostToDevice, st));
        const unsigned blocks = div_up(m, 128);
        if (tx) {
            k_eddsa_prepare_txs<<<blocks, 128, 0, st>>>((const bzk_mpn_tx *)d_in, m, d, d_rows, d_tx_rows, d_s, d_flag);
            BZK_LAUNCHED(ctx);
            BZK_TRY(poseidon_launch(ctx, 7, d_tx_rows, m, d_msg));
            BZK_CUDA(ctx, cudaMemcpy2DAsync(d_rows + 4, 5 * sizeof(Fr), d_msg, sizeof(Fr), sizeof(Fr), m, cudaMemcpyDeviceToDevice, st));
        } else {
            if (msg2) {
                BZK_CUDA(ctx, cudaMemcpyAsync(d_msg2, msg2 + 2 * off, 2 * m * sizeof(Fr), cudaMemcpyHostToDevice, st));
                BZK_TRY(poseidon_launch(ctx, 2, d_msg2, m, d_msg));
            }
            k_eddsa_prepare_items<<<blocks, 128, 0, st>>>((const bzk_eddsa_item *)d_in, m, msg2 ? d_msg : nullptr, d, d_rows, d_s, d_flag);
            BZK_LAUNCHED(ctx);
        }
        BZK_TRY(poseidon_launch(ctx, 5, d_rows, m, d_h));
        k_eddsa_verify<<<blocks, 128, 0, st>>>(d_rows, d_h, d_s, d_flag, d, (const JJNiels *)ctx->d_jj_table, m, d_ok);
        BZK_LAUNCHED(ctx);
        BZK_CUDA(ctx, cudaMemcpyAsync(ok + off, d_ok, m, cudaMemcpyDeviceToHost, st));
        BZK_CUDA(ctx, cudaStreamSynchronize(st));
        for (size_t k = 0; k < m; k++) accepted += ok[off + k];
    }
    if (n_ok) *n_ok = accepted;
    return BZK_OK;
}

// jubjub_d canonical -> Montgomery; false if it is not canonical
bool curve_d(const bzk_fr *jubjub_d, Fr *d) {
    memcpy(d->l, jubjub_d, 32);
    if (!is_canonical(*d)) return false;
    *d = d->to_mont();
    return true;
}
void canon_of(bzk_fr *out, const Fr &mont) {
    const Fr c = mont.from_mont();
    memcpy(out, c.l, 32);
}

}  // namespace
}  // namespace bzk

using namespace bzk;

extern "C" {

int32_t bzk_jubjub_eddsa_verify_batch(bzk_ctx *ctx, const bzk_fr *jubjub_d, const bzk_eddsa_item *items, size_t n, uint8_t *ok, uint64_t *n_ok) {
    Fr d;
    if (!ctx || !jubjub_d || (n && (!items || !ok)) || !curve_d(jubjub_d, &d)) return BZK_ERR_BAD_ARG;
    if (n_ok) *n_ok = 0;
    if (n == 0) return BZK_OK;
    if (!ctx->pos_loaded) return BZK_ERR_NO_PARAMS;
    return verify_batch(ctx, d, Items::kEddsa, items, n, nullptr, ok, n_ok);
}

int32_t bzk_mpn_tx_verify_batch(bzk_ctx *ctx, const bzk_fr *jubjub_d, const bzk_mpn_tx *txs, size_t n, uint8_t *ok, uint64_t *n_ok) {
    Fr d;
    if (!ctx || !jubjub_d || (n && (!txs || !ok)) || !curve_d(jubjub_d, &d)) return BZK_ERR_BAD_ARG;
    if (n_ok) *n_ok = 0;
    if (n == 0) return BZK_OK;
    if (!ctx->pos_loaded) return BZK_ERR_NO_PARAMS;
    return verify_batch(ctx, d, Items::kTx, txs, n, nullptr, ok, n_ok);
}

int32_t bzk_mpn_signatures_verify_bytes(bzk_ctx *ctx, const bzk_fr *jubjub_d, uint32_t kind, const uint8_t *bytes, size_t len, uint8_t *ok,
                                        size_t cap, uint64_t *n, uint64_t *n_ok) {
    Fr d;
    if (!ctx || !jubjub_d || !n || (len && !bytes) || !curve_d(jubjub_d, &d)) return BZK_ERR_BAD_ARG;
    std::vector<wire::MpnWithdraw> wds;
    std::vector<wire::MpnTx> txs;
    if (kind == wire::KIND_WITHDRAW) {
        if (!wire::dec_withdraws(bytes, len, wds)) return BZK_ERR_BAD_ARG;
    } else if (kind == wire::KIND_UPDATE) {
        if (!wire::dec_txs(bytes, len, txs)) return BZK_ERR_BAD_ARG;
    } else {
        return BZK_ERR_BAD_ARG;   // deposits carry ed25519 signatures of the L1 payment
    }
    const size_t count = kind == wire::KIND_WITHDRAW ? wds.size() : txs.size();
    *n = count;
    if (!ok) return BZK_OK;
    if (cap < count) return BZK_ERR_BAD_ARG;
    if (n_ok) *n_ok = 0;
    if (count == 0) return BZK_OK;
    if (!ctx->pos_loaded) return BZK_ERR_NO_PARAMS;
    if (kind == wire::KIND_UPDATE) {
        std::vector<bzk_mpn_tx> in(count);
        for (size_t k = 0; k < count; k++) {
            const wire::MpnTx &t = txs[k];
            bzk_mpn_tx &o = in[k];
            memset(&o, 0, sizeof o);
            o.nonce = t.nonce; o.amount = t.amount.amount; o.fee = t.fee.amount;
            o.src_pk_odd = t.src.odd ? 1 : 0; o.dst_pk_odd = t.dst.odd ? 1 : 0;
            canon_of(&o.src_pk_x, t.src.x); canon_of(&o.dst_pk_x, t.dst.x);
            canon_of(&o.amount_token_id, t.amount.token.scalar()); canon_of(&o.fee_token_id, t.fee.token.scalar());
            canon_of(&o.sig_rx, t.sig.r.x); canon_of(&o.sig_ry, t.sig.r.y); canon_of(&o.sig_s, t.sig.s);
        }
        return verify_batch(ctx, d, Items::kTx, in.data(), count, nullptr, ok, n_ok);
    }
    std::vector<bzk_eddsa_item> in(count);
    std::vector<Fr> msg2(2 * count);
    for (size_t k = 0; k < count; k++) {
        const wire::MpnWithdraw &w = wds[k];
        bzk_eddsa_item &o = in[k];
        memset(&o, 0, sizeof o);
        canon_of(&o.pk_x, w.mpn_address.x); o.pk_odd = w.mpn_address.odd ? 1 : 0;
        canon_of(&o.sig_rx, w.sig.r.x); canon_of(&o.sig_ry, w.sig.r.y); canon_of(&o.sig_s, w.sig.s);
        msg2[2 * k] = wire::withdraw_fingerprint(w.payment);
        msg2[2 * k + 1] = fr_from_u64(w.nonce);
    }
    return verify_batch(ctx, d, Items::kEddsa, in.data(), count, msg2.data(), ok, n_ok);
}

}  // extern "C"
