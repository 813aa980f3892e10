// bazuka_b200 — the MPN ledger and the transition builders as native host code over the GPU primitives.
//
// Mirrors `mpn::{update,deposit,withdraw}` (/root/reference/src/mpn/update.rs:8-299, deposit.rs, withdraw.rs) on the state model of
// /root/reference/src/mpn/mod.rs:219-240 and /root/reference/src/zk/state/mod.rs:93-208 (account leaf =
// Poseidon-5(tx_nonce, withdraw_nonce, pk.x, pk.y, tokens_root); token leaf = Poseidon-2(token_id, amount);
// 4-ary sparse trees with `compress_default` defaults), but in the two-phase shape of DESIGN.md §3.7:
//   1. ledger decisions, sequential, no hashing (acceptance rules, balances, slot choice);
//   2. all hashing in batches on the GPU: bzk_poseidon_hash for the leaves, the versioned level-synchronous
//      tree update (poseidon.cu) for the token forest and the state tree.
// Output = the reference's transition structs, what a circuit row needs besides them, and the three state-dependent
// public inputs; the C ABI writes the rows through the circuits' writers (mpn_wire.cu).  Scalars cross the ABI as
// canonical 32-byte little-endian integers.
#include "common.cuh"
#include "hash_plan.cuh"
#include "jubjub.cuh"
#include "mpn_wire.cuh"
#include <algorithm>
#include <cstdarg>
#include <functional>
#include <map>
#include <set>
#include <string>
#include <unordered_map>
#include <vector>

#if !defined(__CUDACC__)
// A host compile of this file (the CPU test tier builds the ledger's host code with g++ over a host stand-in of the batched
// Poseidon launch, bzk_poseidon_hash) has no kernels: there a plan step gathers its rows by hash_plan.cuh's per-node rule and
// hashes them in one bzk_poseidon_hash call.  libbzk is compiled by nvcc and runs k_poseidon_plan_step (poseidon.cu) instead.
namespace bzk {
int32_t poseidon_plan_step(bzk_ctx *ctx, uint32_t arity, const uint32_t *ops, size_t n, const Fr *prev, const Fr *host, Fr *out) {
    if (arity != 2 && arity != 4 && arity != 5) return BZK_ERR_BAD_ARG;
    std::vector<Fr> rows(n * arity);
    for (size_t k = 0; k < n * arity; k++) rows[k] = *plan_operand(ops[k], prev, host);
    return n ? bzk_poseidon_hash(ctx, arity, (const bzk_fr *)rows.data(), n, (bzk_fr *)out) : BZK_OK;
}
}  // namespace bzk
#endif

namespace bzk {
int32_t tree4_versioned_update(bzk_ctx *ctx, uint32_t depth, const uint32_t *d_tree_id, const uint64_t *d_idx, size_t n, Fr *d_vals,
                               const Fr *d_init_proofs, Fr *d_out_proofs);
void witness_program_shape(const bzk_witness_program *p, uint64_t *n_ops, uint32_t *n_raw, uint32_t *n_ext);
}
using namespace bzk;

namespace {

struct FrKey {  // Montgomery limbs as a map key
    uint32_t l[8];
    bool operator<(const FrKey &o) const { return std::lexicographical_compare(l, l + 8, o.l, o.l + 8); }
};
inline FrKey key_of(const Fr &a) { FrKey k; memcpy(k.l, a.l, 32); return k; }
inline Fr fr_from_canon(const bzk_fr *c) { Fr a; memcpy(a.l, c, 32); return a.to_mont(); }

struct Money { Fr token_id; uint64_t amount; };  // token_id in Montgomery form
struct Account {
    uint64_t tx_nonce = 0, withdraw_nonce = 0;
    Fr ax = Fr::zero(), ay = Fr::zero();
    std::map<uint32_t, Money> tokens;  // ordered: `find_token_index` scans slots in ascending order
};

struct Point { Fr x, y; };
constexpr size_t kDecompressCacheCap = 1u << 16;  // decompressed keys kept per ledger (cleared when full)

}  // namespace

struct bzk_mpn_state {
    uint32_t A = 0, T = 0;
    Fr jj_d;
    std::vector<Fr> defaults, tdefaults;                     // per level: state tree / token tree
    std::vector<std::unordered_map<uint64_t, Fr>> levels;    // sparse state tree, level 0 = leaves; defaults are not stored
    std::map<uint64_t, Account> accounts;
    // The chain's own tables, which the builders only READ (`get_mpn_account_indices`, `get_mpn_account_count`,
    // /root/reference/src/mpn/update.rs:29,47-70): they change when a block is applied, not when a batch is built.
    std::map<std::pair<FrKey, FrKey>, uint64_t> by_addr;      // address -> index of the first account holding it
    uint64_t account_count = 0;
    // `new_account_indices`: accounts created by the batches built so far on this fork (threaded through deposit ->
    // withdraw -> update by `prepare_works`, /root/reference/src/mpn/mod.rs:330,353-414); bzk_mpn_state_commit_accounts
    // moves them into the chain tables
    std::map<std::pair<FrKey, FrKey>, uint64_t> pending;
    uint64_t state_size = 0;  // ZkCompressedState::state_size = number of non-zero scalar leaves
    std::map<FrKey, Point> decompress_cache;

    Fr node(uint32_t lvl, uint64_t idx) const {
        auto it = levels[lvl].find(idx);
        return it == levels[lvl].end() ? defaults[lvl] : it->second;
    }
    void put(uint32_t lvl, uint64_t idx, const Fr &v) {
        if (v == defaults[lvl]) levels[lvl].erase(idx);
        else levels[lvl][idx] = v;
    }
    void prove(uint64_t idx, Fr *out /*[A][3]*/) const {
        for (uint32_t l = 0; l < A; l++) {
            const uint64_t base = (idx >> 2) << 2;
            int w = 0;
            for (uint64_t k = 0; k < 4; k++)
                if (base + k != idx) out[l * 3 + (w++)] = node(l, base + k);
            idx >>= 2;
        }
    }
};

namespace {

// PointCompressed::decompress (/root/reference/src/crypto/jubjub/curve.rs:78-88); x canonical in, Montgomery out
bool jj_decompress(bzk_mpn_state *s, const bzk_fr *x_canon, bool odd, Point *out) {
    Fr x = fr_from_canon(x_canon);
    auto it = s->decompress_cache.find(key_of(x));
    Point p;
    if (it != s->decompress_cache.end()) p = it->second;
    else {
        Fr y;
        if (!jj_decompress_root(x, s->jj_d, &y)) return false;
        p = Point{x, y};
        if (s->decompress_cache.size() >= kDecompressCacheCap) s->decompress_cache.clear();
        s->decompress_cache[key_of(x)] = p;
    }
    out->x = p.x;
    out->y = jj_with_parity(p.y, odd);
    return true;
}

// non-zero scalar leaves of one account (`set_data` counts a leaf when it becomes non-zero,
// /root/reference/src/zk/state/mod.rs:327-341)
uint64_t leaf_count(const Account &a) {
    uint64_t n = (a.tx_nonce != 0) + (a.withdraw_nonce != 0) + !a.ax.is_zero() + !a.ay.is_zero();
    for (auto &kv : a.tokens) n += !kv.second.token_id.is_zero() + (kv.second.amount != 0);
    return n;
}
bool canonical(const bzk_fr &v) {
    Fr a;
    memcpy(a.l, &v, 32);
    for (int i = 7; i >= 0; i--) {
        if (a.l[i] < FrParams::p(i)) return true;
        if (a.l[i] > FrParams::p(i)) return false;
    }
    return false;  // == r
}

int find_token_index(const Account &a, uint32_t T, const Fr &token_id, bool empty_allowed) {
    for (auto &kv : a.tokens)
        if (kv.second.token_id == token_id) return (int)kv.first;
    if (empty_allowed)
        for (uint32_t i = 0; i < (1u << (2 * T)); i++)
            if (!a.tokens.count(i)) return (int)i;
    return -1;
}

// host front-end of the versioned tree update: vals[(depth+1)*n] (vals[0..n) in), proofs [n][depth][3]
int32_t tree_update_host(bzk_ctx *ctx, uint32_t depth, const std::vector<uint32_t> &tid, const std::vector<uint64_t> &idx,
                         std::vector<Fr> &vals, const std::vector<Fr> &init, std::vector<Fr> &proofs) {
    const size_t n = idx.size();
    proofs.assign(n * depth * 3, Fr::zero());
    if (n == 0) return BZK_OK;
    size_t o_tid = 0, o_idx = (n * 4 + 255) & ~(size_t)255, o_vals = o_idx + ((n * 8 + 255) & ~(size_t)255),
           o_init = o_vals + (depth + 1) * n * sizeof(Fr), o_pr = o_init + n * depth * 3 * sizeof(Fr), total = o_pr + n * depth * 3 * sizeof(Fr);
    // the context's grow-only arena: no cudaMalloc / cudaFree (device-wide synchronisations) per batch
    BZK_TRY(ensure_ws(ctx, &ctx->ws, &ctx->ws_bytes, total));
    char *b = (char *)ctx->ws;
    cudaStream_t st = ctx->stream;
    BZK_CUDA(ctx, cudaMemcpyAsync(b + o_tid, tid.data(), n * 4, cudaMemcpyHostToDevice, st));
    BZK_CUDA(ctx, cudaMemcpyAsync(b + o_idx, idx.data(), n * 8, cudaMemcpyHostToDevice, st));
    BZK_CUDA(ctx, cudaMemcpyAsync(b + o_vals, vals.data(), n * sizeof(Fr), cudaMemcpyHostToDevice, st));
    BZK_CUDA(ctx, cudaMemcpyAsync(b + o_init, init.data(), n * depth * 3 * sizeof(Fr), cudaMemcpyHostToDevice, st));
    BZK_TRY(tree4_versioned_update(ctx, depth, (const uint32_t *)(b + o_tid), (const uint64_t *)(b + o_idx), n, (Fr *)(b + o_vals),
                                   (const Fr *)(b + o_init), (Fr *)(b + o_pr)));
    vals.resize((size_t)(depth + 1) * n);
    BZK_CUDA(ctx, cudaMemcpyAsync(vals.data(), b + o_vals, (depth + 1) * n * sizeof(Fr), cudaMemcpyDeviceToHost, st));
    BZK_CUDA(ctx, cudaMemcpyAsync(proofs.data(), b + o_pr, n * depth * 3 * sizeof(Fr), cudaMemcpyDeviceToHost, st));
    BZK_CUDA(ctx, cudaStreamSynchronize(st));
    return BZK_OK;
}

int32_t hash_rows(bzk_ctx *ctx, uint32_t arity, const std::vector<Fr> &rows, std::vector<Fr> &out) {
    const size_t n = rows.size() / arity;
    out.assign(n, Fr::zero());
    if (n == 0) return BZK_OK;
    return bzk_poseidon_hash(ctx, arity, (const bzk_fr *)rows.data(), n, (bzk_fr *)out.data());
}

// the token forest of a batch: pre-batch tokens of the touched accounts enter as writes into empty trees
struct Forest {
    uint32_t T;
    std::map<uint64_t, uint32_t> tree_of;
    std::vector<Fr> rows;  // [n][2]
    std::vector<uint32_t> tid;
    std::vector<uint64_t> idx;
    std::vector<Fr> vals, proofs;
    std::vector<Fr> cur;  // current root per tree while replaying
    size_t n_init = 0;
    size_t write(uint64_t acc, uint32_t index, const Money &m) {
        rows.push_back(m.token_id);
        rows.push_back(fr_from_u64(m.amount));
        tid.push_back(tree_of.at(acc));
        idx.push_back(index);
        return idx.size() - 1;
    }
    int32_t run(bzk_ctx *ctx, const std::vector<Fr> &tdef) {
        std::vector<Fr> leaves;
        BZK_TRY(hash_rows(ctx, 2, rows, leaves));
        const size_t n = idx.size();
        std::vector<Fr> init(n * T * 3);
        for (size_t e = 0; e < n; e++)
            for (uint32_t l = 0; l < T; l++)
                for (int k = 0; k < 3; k++) init[(e * T + l) * 3 + k] = tdef[l];
        vals = leaves;
        BZK_TRY(tree_update_host(ctx, T, tid, idx, vals, init, proofs));
        cur.assign(tree_of.size(), tdef[T]);
        for (size_t e = 0; e < n_init; e++) cur[tid[e]] = vals[(size_t)T * n + e];
        return BZK_OK;
    }
    Fr root(uint64_t acc) const { return cur[tree_of.at(acc)]; }
    Fr applied(uint64_t acc, size_t e) {
        const Fr r = vals[(size_t)T * idx.size() + e];
        cur[tree_of.at(acc)] = r;
        return r;
    }
};


// `JubJub::verify` (/root/reference/src/crypto/jubjub/mod.rs:151-167) given h = Poseidon(R.x, R.y, A.x, A.y, msg) (Montgomery)
inline bool eddsa_verify_with_h(const bzk_mpn_state *s, const Point &pk, const Point &sig_r, const Fr &sig_s_canon, const Fr &h_mont) {
    Fr bx, by;
    jj_base(&bx, &by);
    const JJ sB = jj_mul(jj_from_affine(bx, by), sig_s_canon, s->jj_d.dbl());
    return jj_eddsa_check(s->jj_d, pk.x, pk.y, sig_r.x, sig_r.y, h_mont.from_mont(), sB);
}

}  // namespace

// `JubJub::verify` (/root/reference/src/crypto/jubjub/mod.rs:151-167) as a stand-alone host call: the signature check the
// withdraw builder applies (and a bank node applies to every MPN transaction before it enters the pool), on libbzk's host
// field arithmetic and the host Poseidon.  All scalars canonical.  Returns 1 (valid), 0 (invalid) or a negative status.
extern "C" int32_t bzk_jubjub_eddsa_verify(const bzk_poseidon_host *hasher, const bzk_fr *jubjub_d, const bzk_fr pk_xy[2], const bzk_fr *message,
                                           const bzk_fr sig_r_xy[2], const bzk_fr *sig_s) {
    if (!hasher || !jubjub_d || !pk_xy || !message || !sig_r_xy || !sig_s) return BZK_ERR_BAD_ARG;
    if (!canonical(pk_xy[0]) || !canonical(pk_xy[1]) || !canonical(sig_r_xy[0]) || !canonical(sig_r_xy[1]) || !canonical(*sig_s) || !canonical(*message))
        return 0;
    bzk_mpn_state tmp;
    tmp.jj_d = fr_from_canon(jubjub_d);
    const Point pk{fr_from_canon(pk_xy + 0), fr_from_canon(pk_xy + 1)}, r{fr_from_canon(sig_r_xy + 0), fr_from_canon(sig_r_xy + 1)};
    const Fr in[5] = {r.x, r.y, pk.x, pk.y, fr_from_canon(message)};
    Fr h;
    BZK_TRY(bzk_poseidon_host_hash(hasher, 5, (const bzk_fr *)in, 1, (bzk_fr *)&h));
    Fr s_canon;
    memcpy(s_canon.l, sig_s, 32);
    return eddsa_verify_with_h(&tmp, pk, r, s_canon, h) ? 1 : 0;
}

namespace {

// root of `List<log4 B>(Struct[...])` over the batch's rows (deposit.rs:178-218, withdraw.rs:190-245): one hash per row,
// then the 4-ary tree — every level one batched launch
int32_t list_root(bzk_ctx *ctx, uint32_t arity, const std::vector<Fr> &rows, Fr *out) {
    std::vector<Fr> cur;
    BZK_TRY(hash_rows(ctx, arity, rows, cur));
    while (cur.size() > 1) {
        std::vector<Fr> nxt;
        BZK_TRY(hash_rows(ctx, 4, cur, nxt));
        cur.swap(nxt);
    }
    *out = cur[0];
    return BZK_OK;
}

// ---- the builders' values as the reference's transition structs
wire::Money wire_money(const Money &m) {
    wire::Money w;
    w.token = wire::ContractId::of_scalar(m.token_id);
    w.amount = m.amount;
    return w;
}
wire::Account wire_account(const Account &a) {
    wire::Account w;
    w.tx_nonce = a.tx_nonce; w.withdraw_nonce = a.withdraw_nonce;
    w.address.x = a.ax; w.address.y = a.ay;
    for (auto &kv : a.tokens) w.tokens.emplace_back((uint64_t)kv.first, wire_money(kv.second));   // ascending slot order
    return w;
}
}  // namespace

extern "C" {

int32_t bzk_mpn_update_raw_width(uint32_t A, uint32_t T, uint32_t *n_raw) {
    if (!n_raw || A == 0 || A > 31 || T == 0 || T > 8) return BZK_ERR_BAD_ARG;
    *n_raw = update_raw_width(A, T);
    return BZK_OK;
}

int32_t bzk_mpn_state_create(bzk_ctx *ctx, uint32_t log4_tree, uint32_t log4_token, const bzk_fr *jj_d_canon, bzk_mpn_state **out) {
    if (!ctx || !out || !jj_d_canon || log4_tree == 0 || log4_tree > 31 || log4_token == 0 || log4_token > 8) return BZK_ERR_BAD_ARG;
    auto *s = new (std::nothrow) bzk_mpn_state;
    if (!s) return BZK_ERR_OOM;
    s->A = log4_tree; s->T = log4_token;
    s->jj_d = fr_from_canon(jj_d_canon);
    // compress_default (/root/reference/src/zk/mod.rs:401-423): token leaf H(0,0), lists H([d;4]) per level,
    // account struct H(0,0,0,0,token-list default)
    std::vector<Fr> in, h;
    in.assign(2, Fr::zero());
    int32_t st = hash_rows(ctx, 2, in, h);
    s->tdefaults.push_back(st == BZK_OK ? h[0] : Fr::zero());
    for (uint32_t l = 0; st == BZK_OK && l < log4_token; l++) {
        in.assign(4, s->tdefaults.back());
        st = hash_rows(ctx, 4, in, h);
        if (st == BZK_OK) s->tdefaults.push_back(h[0]);
    }
    if (st == BZK_OK) {
        in.assign(5, Fr::zero());
        in[4] = s->tdefaults.back();
        st = hash_rows(ctx, 5, in, h);
        if (st == BZK_OK) s->defaults.push_back(h[0]);
    }
    for (uint32_t l = 0; st == BZK_OK && l < log4_tree; l++) {
        in.assign(4, s->defaults.back());
        st = hash_rows(ctx, 4, in, h);
        if (st == BZK_OK) s->defaults.push_back(h[0]);
    }
    if (st != BZK_OK) { delete s; return st; }
    s->levels.resize(log4_tree + 1);
    *out = s;
    return BZK_OK;
}

int32_t bzk_mpn_state_free(bzk_mpn_state *s) {
    delete s;
    return BZK_OK;
}

int32_t bzk_mpn_state_root(const bzk_mpn_state *s, bzk_fr *root) {
    if (!s || !root) return BZK_ERR_BAD_ARG;
    fr_to_canon(root, s->node(s->A, 0));
    return BZK_OK;
}

// `set_mpn_account` (/root/reference/src/zk/state/mod.rs:140-208): one account, sequential path re-hash (used to load
// a ledger; batches go through bzk_mpn_update_build)
int32_t bzk_mpn_state_set_account(bzk_ctx *ctx, bzk_mpn_state *s, uint64_t index, uint64_t tx_nonce, uint64_t withdraw_nonce,
                                  const bzk_fr *addr_x, const bzk_fr *addr_y, const uint32_t *token_index, const bzk_fr *token_id,
                                  const uint64_t *token_amount, uint32_t n_tokens) {
    if (!ctx || !s || !addr_x || !addr_y || (n_tokens && (!token_index || !token_id || !token_amount))) return BZK_ERR_BAD_ARG;
    if (index >> (2 * s->A)) return BZK_ERR_BAD_ARG;
    Account a;
    a.tx_nonce = tx_nonce; a.withdraw_nonce = withdraw_nonce;
    a.ax = fr_from_canon(addr_x); a.ay = fr_from_canon(addr_y);
    if (!canonical(*addr_x) || !canonical(*addr_y)) return BZK_ERR_BAD_ARG;
    for (uint32_t k = 0; k < n_tokens; k++) {
        if (token_index[k] >> (2 * s->T) || !canonical(token_id[k])) return BZK_ERR_BAD_ARG;
        const Fr id = fr_from_canon(token_id + k);
        if (id.is_zero()) continue;  // `get_mpn_account` drops slots whose token id is zero (state/mod.rs:127-130)
        a.tokens[token_index[k]] = Money{id, token_amount[k]};
    }
    Forest f;
    f.T = s->T;
    f.tree_of[index] = 0;
    for (auto &kv : a.tokens) f.write(index, kv.first, kv.second);
    f.n_init = f.idx.size();
    BZK_TRY(f.run(ctx, s->tdefaults));
    std::vector<Fr> row = {fr_from_u64(a.tx_nonce), fr_from_u64(a.withdraw_nonce), a.ax, a.ay, f.root(index)}, leaf;
    BZK_TRY(hash_rows(ctx, 5, row, leaf));
    std::vector<Fr> vals = {leaf[0]}, init(s->A * 3), proofs;
    s->prove(index, init.data());
    BZK_TRY(tree_update_host(ctx, s->A, {0u}, {index}, vals, init, proofs));
    uint64_t node = index;
    for (uint32_t l = 0; l <= s->A; l++) { s->put(l, node, vals[l]); node >>= 2; }
    auto old = s->accounts.find(index);
    if (old != s->accounts.end()) {
        s->state_size -= leaf_count(old->second);
        // an overwritten account gives its address back if the table pointed at this slot
        auto oit = s->by_addr.find(std::make_pair(key_of(old->second.ax), key_of(old->second.ay)));
        if (oit != s->by_addr.end() && oit->second == index && !(old->second.ax == a.ax && old->second.ay == a.ay)) s->by_addr.erase(oit);
    }
    s->state_size += leaf_count(a);
    s->accounts[index] = a;
    if (!(a.ax.is_zero() && a.ay.is_zero())) s->by_addr.emplace(std::make_pair(key_of(a.ax), key_of(a.ay)), index);
    s->account_count = std::max(s->account_count, index + 1);
    return BZK_OK;
}

/* An independent copy of the ledger (`db.fork_on_ram()`, /root/reference/src/mpn/mod.rs:313): build the batches of a
 * block on the copy and keep it only if the block is accepted — bzk_mpn_update_build writes the ledger it is given. */
int32_t bzk_mpn_state_clone(const bzk_mpn_state *s, bzk_mpn_state **out) {
    if (!s || !out) return BZK_ERR_BAD_ARG;
    auto *c = new (std::nothrow) bzk_mpn_state(*s);
    if (!c) return BZK_ERR_OOM;
    c->decompress_cache.clear();
    *out = c;
    return BZK_OK;
}
/* `ZkCompressedState { state_hash, state_size }` of the ledger (/root/reference/src/zk/mod.rs: state_size = non-zero scalar
 * leaves) and the chain-side account count */
int32_t bzk_mpn_state_info(const bzk_mpn_state *s, bzk_fr *state_hash, uint64_t *state_size, uint64_t *account_count, uint64_t *pending_accounts) {
    if (!s) return BZK_ERR_BAD_ARG;
    if (state_hash) fr_to_canon(state_hash, s->node(s->A, 0));
    if (state_size) *state_size = s->state_size;
    if (account_count) *account_count = s->account_count;
    if (pending_accounts) *pending_accounts = s->pending.size();
    return BZK_OK;
}
/* out[2] = {log4_tree, log4_token} the ledger was created with */
int32_t bzk_mpn_state_shape(const bzk_mpn_state *s, uint32_t out[2]) {
    if (!s || !out) return BZK_ERR_BAD_ARG;
    out[0] = s->A; out[1] = s->T;
    return BZK_OK;
}
/* `MpnWorkPool.final_delta` (/root/reference/src/mpn/mod.rs:17-45,416-417): every scalar leaf in which `after` (the fork
 * prepare_works returned) differs from `before`, as the bincode of `ZkDeltaPairs(HashMap<ZkDataLocator(Vec<u64>), Option<ZkScalar>>)`:
 * locator [account, field] for the four account scalars, [account, 4, token slot, 0 | 1] for a token's id / balance
 * (`set_mpn_account`, /root/reference/src/zk/state/mod.rs:140-208); a leaf that became zero is a `Remove` (None).  Entries in
 * ascending locator order.  Release the buffer with bzk_buffer_free. */
int32_t bzk_mpn_state_delta(const bzk_mpn_state *before, const bzk_mpn_state *after, uint8_t **bytes, size_t *len, uint64_t *n_entries) {
    if (!before || !after || !bytes || !len) return BZK_ERR_BAD_ARG;
    using Loc = std::vector<uint64_t>;
    auto leaves = [](const bzk_mpn_state *s, uint64_t idx, std::map<Loc, Fr> &out) {
        auto it = s->accounts.find(idx);
        if (it == s->accounts.end()) return;
        const Account &a = it->second;
        const Fr f[4] = {fr_from_u64(a.tx_nonce), fr_from_u64(a.withdraw_nonce), a.ax, a.ay};
        for (uint64_t k = 0; k < 4; k++) out[Loc{idx, k}] = f[k];
        for (auto &kv : a.tokens) {
            out[Loc{idx, 4, kv.first, 0}] = kv.second.token_id;
            out[Loc{idx, 4, kv.first, 1}] = fr_from_u64(kv.second.amount);
        }
    };
    std::set<uint64_t> touched;
    for (auto &kv : before->accounts) touched.insert(kv.first);
    for (auto &kv : after->accounts) touched.insert(kv.first);
    wire::Writer w;
    uint64_t n = 0;
    w.u64(0);
    for (uint64_t idx : touched) {
        std::map<Loc, Fr> o, a;
        leaves(before, idx, o);
        leaves(after, idx, a);
        std::set<Loc> locs;
        for (auto &kv : o) locs.insert(kv.first);
        for (auto &kv : a) locs.insert(kv.first);
        for (const Loc &l : locs) {
            const Fr ov = o.count(l) ? o[l] : Fr::zero(), nv = a.count(l) ? a[l] : Fr::zero();
            if (ov == nv) continue;
            w.u64(l.size());
            for (uint64_t x : l) w.u64(x);
            if (nv.is_zero()) w.u8(0);
            else { w.u8(1); w.fr(nv); }
            n++;
        }
    }
    memcpy(w.b.data(), &n, 8);
    uint8_t *buf = (uint8_t *)malloc(w.b.size());
    if (!buf) return BZK_ERR_OOM;
    memcpy(buf, w.b.data(), w.b.size());
    *bytes = buf; *len = w.b.size();
    if (n_entries) *n_entries = n;
    return BZK_OK;
}
/* The block built on this fork was applied: its new accounts enter the chain's index table. */
int32_t bzk_mpn_state_commit_accounts(bzk_mpn_state *s) {
    if (!s) return BZK_ERR_BAD_ARG;
    for (auto &kv : s->pending) {
        s->by_addr.emplace(kv.first, kv.second);
        s->account_count = std::max(s->account_count, kv.second + 1);
    }
    s->pending.clear();
    return BZK_OK;
}
}  // extern "C"

// ---------------------------------------------------------------------------------------------
// A block's `ZkDeltaPairs` applied to the ledger (DESIGN.md §3.12): decode and validate every entry, fold the entries into
// the final accounts, plan the re-hash of every touched token tree, account leaf and state-tree node (which nodes are dirty
// does not depend on any hash), run the plan as one launch per level, check the result, and only then write the ledger.
// ---------------------------------------------------------------------------------------------
namespace {

struct DeltaLeaf {
    uint64_t acc;
    uint32_t sub;    // 0..3: account scalar; 4 + 2 * slot + k: the token slot's id (k = 0) or balance (k = 1)
    uint64_t entry;  // position in the image
    Fr v;            // Montgomery
};

int32_t refuse(bzk_ctx *ctx, const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(ctx->err, sizeof ctx->err, fmt, ap);
    va_end(ap);
    return BZK_ERR_BAD_ARG;
}
std::string loc_str(const uint64_t *loc, uint64_t n) {
    std::string o = "[";
    for (uint64_t k = 0; k < n; k++) o += (k ? ", " : "") + std::to_string(loc[k]);
    return o + "]";
}
std::string loc_str(uint64_t acc, uint32_t sub) {
    const uint64_t loc[4] = {acc, sub < 4 ? sub : 4, (sub - 4) >> 1, (sub - 4) & 1};
    return loc_str(loc, sub < 4 ? 2 : 4);
}
std::string fr_hex(const Fr &a) {
    const Fr c = a.from_mont();
    char b[68] = "0x";
    for (int i = 7; i >= 0; i--) snprintf(b + 2 + 8 * (7 - i), 9, "%08x", c.l[i]);
    return b;
}
bool fits_u64(const Fr &a, uint64_t *out) {
    const Fr c = a.from_mont();
    for (int i = 2; i < 8; i++)
        if (c.l[i]) return false;
    *out = (uint64_t)c.l[0] | ((uint64_t)c.l[1] << 32);
    return true;
}
bool is_empty(const Account &a) { return !a.tx_nonce && !a.withdraw_nonce && a.ax.is_zero() && a.ay.is_zero() && a.tokens.empty(); }

// bincode of ZkDeltaPairs -> leaves sorted by (account, leaf); refuses what the MPN state model cannot address
int32_t decode_delta(bzk_ctx *ctx, const bzk_mpn_state *s, const uint8_t *bytes, size_t len, std::vector<DeltaLeaf> &out) {
    wire::Reader r(bytes, len);
    const uint64_t n = r.u64();
    if (!r.ok) return refuse(ctx, "delta image of %zu bytes is truncated before its entry count", len);
    if (n > (len - 8) / 9) return refuse(ctx, "delta image of %zu bytes is truncated: it announces %llu entries", len, (unsigned long long)n);
    out.reserve(n);
    for (uint64_t e = 0; e < n; e++) {
        const unsigned long long ee = e;
        const uint64_t L = r.u64();
        if (r.ok && L != 2 && L != 4) return refuse(ctx, "entry %llu: a locator of %llu elements is not a scalar of the MPN state", ee, (unsigned long long)L);
        uint64_t loc[4] = {0, 0, 0, 0};
        for (uint64_t k = 0; k < L && r.ok; k++) loc[k] = r.u64();
        const uint8_t tag = r.u8();
        if (!r.ok) return refuse(ctx, "entry %llu: delta image truncated", ee);
        if (tag > 1) return refuse(ctx, "entry %llu: option tag %u is neither None (0) nor Some (1)", ee, tag);
        const std::string ls = loc_str(loc, L);
        Fr v = Fr::zero();
        if (tag == 1) {
            const uint8_t *p = r.take(32);
            if (!p) return refuse(ctx, "entry %llu: delta image truncated", ee);
            bzk_fr raw;
            memcpy(&raw, p, 32);
            if (!canonical(raw)) return refuse(ctx, "entry %llu: the scalar of locator %s is not canonical", ee, ls.c_str());
            memcpy(v.l, p, 32);
        }
        if (loc[0] >> (2 * s->A)) return refuse(ctx, "entry %llu: locator %s outside the state tree (4^%u accounts)", ee, ls.c_str(), s->A);
        uint32_t sub;
        if (L == 2) {
            if (loc[1] > 3) return refuse(ctx, "entry %llu: locator %s is not an account scalar", ee, ls.c_str());
            sub = (uint32_t)loc[1];
        } else {
            if (loc[1] != 4 || loc[3] > 1) return refuse(ctx, "entry %llu: locator %s is not a token leaf", ee, ls.c_str());
            if (loc[2] >> (2 * s->T)) return refuse(ctx, "entry %llu: locator %s outside the token tree", ee, ls.c_str());
            sub = 4 + 2 * (uint32_t)loc[2] + (uint32_t)loc[3];
        }
        out.push_back(DeltaLeaf{loc[0], sub, e, v});
    }
    if (r.o != len) return refuse(ctx, "delta image has %zu trailing bytes after its %llu entries", len - r.o, (unsigned long long)n);
    std::sort(out.begin(), out.end(), [](const DeltaLeaf &a, const DeltaLeaf &b) { return a.acc != b.acc ? a.acc < b.acc : a.sub < b.sub; });
    for (size_t k = 1; k < out.size(); k++)
        if (out[k].acc == out[k - 1].acc && out[k].sub == out[k - 1].sub) {
            const DeltaLeaf &a = out[k - 1].entry < out[k].entry ? out[k - 1] : out[k], &b = out[k - 1].entry < out[k].entry ? out[k] : out[k - 1];
            return refuse(ctx, "entry %llu: duplicate locator %s (entry %llu)", (unsigned long long)b.entry, loc_str(b.acc, b.sub).c_str(),
                          (unsigned long long)a.entry);
        }
    return BZK_OK;
}

// one account's leaves after the delta, as an Account; refuses values the account model cannot hold
int32_t fold_account(bzk_ctx *ctx, const Account &before, const DeltaLeaf *d, size_t n, Account *after, bool *has_x, bool *has_y) {
    const uint64_t acc = d[0].acc;
    Account a = before;
    std::map<uint32_t, std::pair<Fr, Fr>> slots;   // slot -> (id, balance) for every slot the old account or the delta holds
    for (auto &kv : before.tokens) slots[kv.first] = {kv.second.token_id, fr_from_u64(kv.second.amount)};
    *has_x = *has_y = false;
    for (size_t k = 0; k < n; k++) {
        const DeltaLeaf &l = d[k];
        uint64_t u = 0;
        if ((l.sub == 0 || l.sub == 1 || (l.sub >= 4 && (l.sub & 1))) && !fits_u64(l.v, &u))
            return refuse(ctx, "entry %llu: the value of locator %s does not fit in 64 bits", (unsigned long long)l.entry, loc_str(acc, l.sub).c_str());
        switch (l.sub) {
            case 0: a.tx_nonce = u; break;
            case 1: a.withdraw_nonce = u; break;
            case 2: a.ax = l.v; *has_x = true; break;
            case 3: a.ay = l.v; *has_y = true; break;
            default: {
                auto &sl = slots[(l.sub - 4) >> 1];
                ((l.sub & 1) ? sl.second : sl.first) = l.v;
            }
        }
    }
    a.tokens.clear();
    for (auto &kv : slots) {
        uint64_t amount = 0;
        fits_u64(kv.second.second, &amount);
        if (kv.second.first.is_zero()) {
            // `Account::tokens` drops a zero-id slot: a balance there could not be reproduced by the ledger
            if (amount) return refuse(ctx, "account %llu: token slot %u holds balance %llu under token id zero", (unsigned long long)acc, kv.first,
                                      (unsigned long long)amount);
            continue;
        }
        a.tokens[kv.first] = Money{kv.second.first, amount};
    }
    *after = a;
    return BZK_OK;
}

}  // namespace

extern "C" {

/* See include/bzk.h. */
int32_t bzk_mpn_state_apply_delta(bzk_ctx *ctx, bzk_mpn_state *s, const uint8_t *delta, size_t len, const bzk_fr *expect_hash,
                                  const uint64_t *expect_size, uint64_t *n_entries) {
    if (!ctx) return BZK_ERR_BAD_ARG;
    if (!s || (!delta && len)) return refuse(ctx, "null ledger or delta");
    if (!s->pending.empty())
        return refuse(ctx, "the ledger holds %zu accounts of an unapplied prepare_works fork: apply a block's delta to the chain's ledger", s->pending.size());
    if (expect_hash && !canonical(*expect_hash)) return refuse(ctx, "expect_hash is not canonical");
    const uint32_t A = s->A, T = s->T;
    // ---------------------------------------------------------------- decode, fold, index
    std::vector<DeltaLeaf> leaves;
    BZK_TRY(decode_delta(ctx, s, delta, len, leaves));
    struct Touched { uint64_t idx; const Account *before; Account after; };
    std::vector<Touched> touched;
    std::vector<std::pair<std::pair<FrKey, FrKey>, uint64_t>> addrs;   // `index_mpn_accounts`: (x, y) of every index whose x and y both change
    uint64_t size = s->state_size, count = s->account_count;
    static const Account kEmpty;
    for (size_t k = 0; k < leaves.size();) {
        size_t e = k;
        while (e < leaves.size() && leaves[e].acc == leaves[k].acc) e++;
        const uint64_t idx = leaves[k].acc;
        auto it = s->accounts.find(idx);
        Touched t{idx, it == s->accounts.end() ? &kEmpty : &it->second, Account()};
        bool hx = false, hy = false;
        BZK_TRY(fold_account(ctx, *t.before, leaves.data() + k, e - k, &t.after, &hx, &hy));
        if (hx != hy)
            return refuse(ctx, "account %llu: the delta sets its %s but not its %s (an inconsistent account index)", (unsigned long long)idx,
                          hx ? "x" : "y", hx ? "y" : "x");
        if (hx) {
            // ascending indices: one equal to the count extends it, one above it is a gap (apply_tx/mod.rs:43-51)
            if (idx == count) count++;
            else if (idx > count)
                return refuse(ctx, "account %llu: a new address above the account count %llu", (unsigned long long)idx, (unsigned long long)count);
            addrs.emplace_back(std::make_pair(key_of(t.after.ax), key_of(t.after.ay)), idx);
        }
        size += leaf_count(t.after) - leaf_count(*t.before);
        touched.push_back(std::move(t));
        k = e;
    }
    // ---------------------------------------------------------------- the plan: one step per tree level, values on the host
    // hv = tdefaults[0..T] ++ defaults[0..A] ++ the leaf scalars and clean siblings the plan reads
    std::vector<Fr> hv(s->tdefaults);
    hv.insert(hv.end(), s->defaults.begin(), s->defaults.end());
    auto host = [&](const Fr &v) { hv.push_back(v); return kPlanHost | (uint32_t)(hv.size() - 1); };
    struct Step { uint32_t arity; size_t ops_off, out_off, n; };
    std::vector<Step> steps;
    std::vector<uint32_t> ops;
    size_t n_out = 0;
    auto close_step = [&](uint32_t arity, size_t ops_off) {
        const size_t n = (ops.size() - ops_off) / arity;
        steps.push_back(Step{arity, ops_off, n_out, n});
        n_out += n;
    };
    using Node = std::pair<uint32_t, uint64_t>;   // (touched account, node index); level lists stay sorted
    // the parents of the nodes of `cur`, in order; a child not in `cur` is clean: clean(child) gives its operand
    auto level = [&](std::vector<Node> &cur, const std::function<uint32_t(const Node &)> &clean) {
        const size_t off = ops.size();
        std::vector<Node> next;
        for (size_t i = 0; i < cur.size();) {
            const Node p{cur[i].first, cur[i].second >> 2};
            for (uint64_t k = 0; k < 4; k++) {
                const Node c{p.first, p.second * 4 + k};
                ops.push_back(i < cur.size() && cur[i] == c ? (uint32_t)i++ : clean(c));
            }
            next.push_back(p);
        }
        close_step(4, off);
        cur.swap(next);
    };
    // token trees, rebuilt from the final slots: Poseidon-2 leaves, then T levels over default siblings
    std::vector<Node> cur;
    {
        const size_t off = ops.size();
        for (size_t o = 0; o < touched.size(); o++)
            for (auto &kv : touched[o].after.tokens) {
                ops.push_back(host(kv.second.token_id));
                ops.push_back(host(fr_from_u64(kv.second.amount)));
                cur.emplace_back((uint32_t)o, kv.first);
            }
        close_step(2, off);
    }
    for (uint32_t l = 1; l <= T; l++) level(cur, [&](const Node &) { return kPlanHost | (l - 1); });
    std::vector<uint32_t> troot(touched.size(), kPlanHost | T);
    for (size_t i = 0; i < cur.size(); i++) troot[cur[i].first] = (uint32_t)i;
    // account leaves: Poseidon-5(tx_nonce, withdraw_nonce, x, y, token root); an empty account hashes to defaults[0]
    cur.clear();
    {
        const size_t off = ops.size();
        for (size_t o = 0; o < touched.size(); o++) {
            const Account &a = touched[o].after;
            for (const Fr &v : {fr_from_u64(a.tx_nonce), fr_from_u64(a.withdraw_nonce), a.ax, a.ay}) ops.push_back(host(v));
            ops.push_back(troot[o]);
            cur.emplace_back(0u, touched[o].idx);
        }
        close_step(5, off);
    }
    const size_t first_state = steps.size() - 1;
    std::vector<std::vector<uint64_t>> lvl_idx(A + 1);
    for (auto &c : cur) lvl_idx[0].push_back(c.second);
    for (uint32_t l = 1; l <= A; l++) {
        level(cur, [&](const Node &c) {
            auto it = s->levels[l - 1].find(c.second);
            return it == s->levels[l - 1].end() ? kPlanHost | (T + l) : host(it->second);   // defaults[l - 1] sits at T + 1 + l - 1
        });
        for (auto &c : cur) lvl_idx[l].push_back(c.second);
    }
    if (hv.size() >= kPlanHost || n_out >= kPlanHost) return refuse(ctx, "delta of %zu leaves is too large for one plan", leaves.size());
    // ---------------------------------------------------------------- enqueue every step, then one copy back
    std::vector<Fr> res(n_out - steps[first_state].out_off);
    if (!touched.empty()) {
        BZK_CUDA(ctx, cudaSetDevice(ctx->device));
        const size_t o_hv = (ops.size() * 4 + 255) & ~(size_t)255, o_out = o_hv + ((hv.size() * sizeof(Fr) + 255) & ~(size_t)255),
                     total = o_out + n_out * sizeof(Fr);
        BZK_TRY(ensure_ws(ctx, &ctx->ws, &ctx->ws_bytes, total));
        char *b = (char *)ctx->ws;
        const uint32_t *d_ops = (const uint32_t *)b;
        const Fr *d_hv = (const Fr *)(b + o_hv);
        Fr *d_out = (Fr *)(b + o_out);
        BZK_CUDA(ctx, cudaMemcpyAsync(b, ops.data(), ops.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
        BZK_CUDA(ctx, cudaMemcpyAsync(b + o_hv, hv.data(), hv.size() * sizeof(Fr), cudaMemcpyHostToDevice, ctx->stream));
        for (size_t k = 0; k < steps.size(); k++)
            if (steps[k].n)
                BZK_TRY(poseidon_plan_step(ctx, steps[k].arity, d_ops + steps[k].ops_off, steps[k].n, k ? d_out + steps[k - 1].out_off : nullptr, d_hv,
                                           d_out + steps[k].out_off));
        BZK_CUDA(ctx, cudaMemcpyAsync(res.data(), d_out + steps[first_state].out_off, res.size() * sizeof(Fr), cudaMemcpyDeviceToHost, ctx->stream));
        BZK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
    // ---------------------------------------------------------------- check, then commit
    const Fr root = touched.empty() ? s->node(A, 0) : res.back();
    if ((expect_hash && !(root == fr_from_canon(expect_hash))) || (expect_size && size != *expect_size)) {
        const std::string got = fr_hex(root), want = expect_hash ? fr_hex(fr_from_canon(expect_hash)) : std::string("any");
        return refuse(ctx, "the delta gives state (%s, size %llu), expected (%s, size %s)", got.c_str(), (unsigned long long)size, want.c_str(),
                      expect_size ? std::to_string(*expect_size).c_str() : "any");
    }
    size_t r = 0;
    for (uint32_t l = 0; l <= A; l++)
        for (uint64_t idx : lvl_idx[l]) s->put(l, idx, res[r++]);
    for (auto &t : touched) {
        if (is_empty(t.after)) s->accounts.erase(t.idx);
        else s->accounts[t.idx] = std::move(t.after);
    }
    for (auto &a : addrs) {   // the reference's index is never pruned and `.first()` is the smallest index holding an address
        auto it = s->by_addr.find(a.first);
        if (it == s->by_addr.end()) s->by_addr.emplace(a.first, a.second);
        else it->second = std::min(it->second, a.second);
    }
    s->account_count = count;
    s->state_size = size;
    if (n_entries) *n_entries = leaves.size();
    return BZK_OK;
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------
// The three transition builders (DESIGN.md §3.7): each runs its own acceptance rules over the inputs, sequentially and without
// hashing, on a BatchCore; the core then hashes the token forest and the state tree of the whole batch in batched launches.
// Their output is the reference's transition structs plus what a circuit row needs besides them (bzk::Built); the rows
// themselves come from the writers of csrc/mpn_wire.cu.
// ---------------------------------------------------------------------------------------------
namespace {

wire::PointW null_key() { return wire::PointW{Fr::zero(), Fr::one().neg()}; }   // PublicKey::default().decompress() = (0, -1)

// The ledger side of one batch.  The acceptance loop looks accounts up (index_of, next_index, get) and records every accepted
// change as steps.  A step is one token-forest write (token `slot` of the account, as it is in `after`) and one state-tree write
// (the leaf of `after` over the token root that write leaves); reading an account after a step sees `after`.  hash() runs both
// trees over all steps; per step the core then gives the token root before it, its token proof, its state proof and the state
// root after it.
struct BatchCore {
    bzk_mpn_state *s;
    Fr prev_root;
    std::map<uint64_t, Account> mirror;                    // the accounts the batch has changed
    std::map<std::pair<FrKey, FrKey>, uint64_t> pending;   // s->pending and the accounts this batch creates
    struct Step { uint64_t acc; uint32_t slot; Account after; };
    std::vector<Step> steps;
    std::vector<uint64_t> touched;                         // the steps' accounts in first-seen order
    Forest forest;
    std::vector<Fr> tok_root, s_vals, s_proofs;

    explicit BatchCore(bzk_mpn_state *st) : s(st), prev_root(st->node(st->A, 0)), pending(st->pending) {}
    static std::pair<FrKey, FrKey> key(const Point &a) { return std::make_pair(key_of(a.x), key_of(a.y)); }
    // update.rs:47-70: the chain's index table first, then the accounts created earlier on this fork
    bool index_of(const Point &a, uint64_t *out) const {
        auto it = s->by_addr.find(key(a));
        if (it != s->by_addr.end()) { *out = it->second; return true; }
        auto jt = pending.find(key(a));
        if (jt != pending.end()) { *out = jt->second; return true; }
        return false;
    }
    // the index of an unknown address: mpn_account_count + |new_account_indices|; add_account records it
    uint64_t next_index() const { return s->account_count + pending.size(); }
    void add_account(const Point &a, uint64_t i) { pending.emplace(key(a), i); }
    Account get(uint64_t i) const {
        auto it = mirror.find(i);
        if (it != mirror.end()) return it->second;
        auto jt = s->accounts.find(i);
        return jt == s->accounts.end() ? Account() : jt->second;
    }
    void step(uint64_t acc, uint32_t slot, const Account &after) {
        mirror[acc] = after;
        steps.push_back(Step{acc, slot, after});
    }

    // the token forest (the touched accounts' pre-batch tokens enter as writes into empty trees, then one write per step), then
    // the accounts' leaves and the state tree
    int32_t hash(bzk_ctx *ctx) {
        const uint32_t A = s->A;
        forest.T = s->T;
        for (auto &st : steps)
            if (forest.tree_of.emplace(st.acc, (uint32_t)forest.tree_of.size()).second) touched.push_back(st.acc);
        for (uint64_t acc : touched) {
            auto it = s->accounts.find(acc);
            if (it != s->accounts.end())
                for (auto &kv : it->second.tokens) forest.write(acc, kv.first, kv.second);
        }
        forest.n_init = forest.idx.size();
        for (auto &st : steps) forest.write(st.acc, st.slot, st.after.tokens.at(st.slot));
        BZK_TRY(forest.run(ctx, s->tdefaults));
        std::vector<Fr> rows;
        rows.reserve(steps.size() * 5);
        for (size_t k = 0; k < steps.size(); k++) {
            const Account &a = steps[k].after;
            tok_root.push_back(forest.root(steps[k].acc));
            const Fr r = forest.applied(steps[k].acc, forest.n_init + k);
            for (const Fr &v : {fr_from_u64(a.tx_nonce), fr_from_u64(a.withdraw_nonce), a.ax, a.ay, r}) rows.push_back(v);
        }
        BZK_TRY(hash_rows(ctx, 5, rows, s_vals));
        const size_t ne = steps.size();
        std::vector<uint64_t> idx(ne);
        std::vector<Fr> init(ne * A * 3);
        for (size_t e = 0; e < ne; e++) {
            idx[e] = steps[e].acc;
            s->prove(idx[e], init.data() + e * A * 3);
        }
        return tree_update_host(ctx, A, std::vector<uint32_t>(ne, 0u), idx, s_vals, init, s_proofs);
    }
    Fr tok_before(size_t k) const { return tok_root[k]; }
    wire::Proof tok_proof(size_t k) const {
        const Fr *p = forest.proofs.data() + (forest.n_init + k) * s->T * 3;
        return wire::Proof(p, p + (size_t)s->T * 3);
    }
    wire::Proof state_proof(size_t k) const {
        const Fr *p = s_proofs.data() + k * s->A * 3;
        return wire::Proof(p, p + (size_t)s->A * 3);
    }
    Fr root_after(size_t k) const { return s_vals[(size_t)s->A * steps.size() + k]; }
    Fr root() const { return steps.empty() ? prev_root : root_after(steps.size() - 1); }
    // the state root entering each of `cap` slots when every transition made `per` steps; after the last one the state no longer moves
    std::vector<Fr> slot_roots(uint64_t cap, size_t per) const {
        std::vector<Fr> r(cap, root());
        for (size_t k = 0; k * per < steps.size(); k++) r[k] = k ? root_after(k * per - 1) : prev_root;
        return r;
    }
    // the ledger moves to the end of the batch; public3 = {state, aux_data, next_state}
    void commit(const Fr &aux, bzk_fr public3[3]) {
        const size_t ne = steps.size();
        for (size_t e = 0; e < ne; e++) {
            uint64_t node = steps[e].acc;
            for (uint32_t l = 0; l <= s->A; l++) { s->put(l, node, s_vals[(size_t)l * ne + e]); node >>= 2; }
        }
        for (uint64_t i : touched) {
            auto it = s->accounts.find(i);
            if (it != s->accounts.end()) s->state_size -= leaf_count(it->second);
            s->state_size += leaf_count(mirror[i]);
            s->accounts[i] = mirror[i];
        }
        s->pending = pending;
        fr_to_canon(public3 + 0, prev_root);
        fr_to_canon(public3 + 1, aux);
        fr_to_canon(public3 + 2, root());
    }
};

template <class Tr>
void report(const Built<Tr> &bt, uint64_t n_in, uint8_t *accepted, bzk_fr public3[3], uint64_t *n_accepted) {
    if (accepted) {
        memset(accepted, 0, n_in);
        for (uint64_t k : bt.from) accepted[k] = 1;
    }
    memcpy(public3, bt.public3, sizeof bt.public3);
    *n_accepted = bt.t.size();
}

}  // namespace

// `mpn::update::update` (/root/reference/src/mpn/update.rs:8-299): three steps per transaction (the source's amount, the source's
// fee, the destination)
int32_t bzk::mpn_update_build_impl(bzk_ctx *ctx, bzk_mpn_state *s, const bzk_mpn_tx *txs, uint64_t n_txs, uint32_t log4_batch,
                                   const bzk_fr *fee_token_canon, Built<wire::UpdateTransition> *out) {
    if (!ctx || !s || (n_txs && !txs) || !fee_token_canon || !out || log4_batch > 8) return BZK_ERR_BAD_ARG;
    BZK_CUDA(ctx, cudaSetDevice(ctx->device));
    const uint32_t A = s->A, T = s->T;
    const uint64_t cap = 1ull << (2 * log4_batch);
    const Fr fee_token = fr_from_canon(fee_token_canon);
    BatchCore b(s);
    *out = Built<wire::UpdateTransition>();
    out->d.keys.assign(cap, null_key());
    uint64_t fee_sum = 0;
    for (uint64_t k = 0; k < n_txs && out->t.size() < cap; k++) {
        const bzk_mpn_tx &tx = txs[k];
        // malformed field elements cannot be put into a witness row: such a transaction is simply not eligible
        if (!canonical(tx.src_pk_x) || !canonical(tx.dst_pk_x) || !canonical(tx.amount_token_id) || !canonical(tx.fee_token_id) ||
            !canonical(tx.sig_rx) || !canonical(tx.sig_ry) || !canonical(tx.sig_s))
            continue;
        const Fr fee_tok_id = fr_from_canon(&tx.fee_token_id), amt_tok_id = fr_from_canon(&tx.amount_token_id);
        // the reference's pre-filter (update.rs:31-38): fee token and both keys decompressible; filtered, not an error
        if (!(fee_tok_id == fee_token)) continue;
        Point src_addr, dst_addr;
        if (!jj_decompress(s, &tx.src_pk_x, tx.src_pk_odd != 0, &src_addr) || !jj_decompress(s, &tx.dst_pk_x, tx.dst_pk_odd != 0, &dst_addr))
            continue;
        // an unknown sender is rejected, an unknown receiver gets the next new index
        uint64_t src_index = 0, dst_index = 0;
        if (!b.index_of(src_addr, &src_index)) continue;
        const bool dst_new = !b.index_of(dst_addr, &dst_index);
        if (dst_new) dst_index = b.next_index();
        if (dst_index >> (2 * A)) continue;
        Account src_before = b.get(src_index), dst_before0 = b.get(dst_index);
        const int sti = find_token_index(src_before, T, amt_tok_id, false), dti = find_token_index(dst_before0, T, amt_tok_id, true),
                  sfi = find_token_index(src_before, T, fee_tok_id, false);
        if (sti < 0 || dti < 0 || sfi < 0) continue;
        const Money src_token = src_before.tokens[sti];
        const bool dst_has = dst_before0.tokens.count(dti) != 0;
        if (tx.nonce != src_before.tx_nonce + 1 || !(src_before.ax == src_addr.x) || !(src_before.ay == src_addr.y) ||
            (jj_on_curve(dst_before0.ax, dst_before0.ay, s->jj_d) && (!(dst_before0.ax == dst_addr.x) || !(dst_before0.ay == dst_addr.y))) ||
            (dst_has && !(src_token.token_id == dst_before0.tokens[dti].token_id)) || !(src_token.token_id == amt_tok_id) ||
            src_token.amount < tx.amount)
            continue;
        Account src_mid = src_before;
        src_mid.tx_nonce += 1;
        src_mid.tokens[sti].amount -= tx.amount;
        auto fit = src_mid.tokens.find(sfi);
        if (fit == src_mid.tokens.end() || !(fit->second.token_id == fee_tok_id) || fit->second.amount < tx.fee) continue;
        const Money src_fee_token = fit->second;
        Account src_after = src_mid;
        src_after.tokens[sfi].amount -= tx.fee;
        b.step(src_index, sti, src_mid);
        b.step(src_index, sfi, src_after);
        const Account dst_before = b.get(dst_index);   // after the source's steps: a transfer to oneself sees them
        Money dst_token{Fr::zero(), 0};
        if (dst_before.tokens.count(dti)) dst_token = dst_before.tokens.at(dti);
        Account dst_after = dst_before;
        dst_after.ax = dst_addr.x; dst_after.ay = dst_addr.y;
        if (!dst_after.tokens.count(dti)) dst_after.tokens[dti] = Money{amt_tok_id, 0};
        dst_after.tokens[dti].amount += tx.amount;
        b.step(dst_index, dti, dst_after);
        if (dst_new) b.add_account(dst_addr, dst_index);
        // `UpdateTransition` (update.rs:220-247); the hashes and proofs once the batch is hashed
        wire::UpdateTransition t;
        t.enabled = true;
        t.tx.nonce = tx.nonce;
        t.tx.src = wire::PubKey{src_addr.x, tx.src_pk_odd != 0}; t.tx.dst = wire::PubKey{dst_addr.x, tx.dst_pk_odd != 0};
        t.tx.amount = wire_money(Money{amt_tok_id, tx.amount}); t.tx.fee = wire_money(Money{fee_tok_id, tx.fee});
        t.tx.sig.r = wire::PointW{fr_from_canon(&tx.sig_rx), fr_from_canon(&tx.sig_ry)}; t.tx.sig.s = fr_from_canon(&tx.sig_s);
        t.src_before = wire_account(src_before); t.src_before_balance = wire_money(src_token); t.src_before_fee_balance = wire_money(src_fee_token);
        t.src_index = src_index; t.src_token_index = sti; t.src_fee_token_index = sfi;
        t.dst_before = wire_account(dst_before); t.dst_before_balance = wire_money(dst_token);
        t.dst_index = dst_index; t.dst_token_index = dti;
        out->d.keys[out->t.size()] = wire::PointW{dst_addr.x, dst_addr.y};
        out->t.push_back(std::move(t));
        out->from.push_back(k);
        fee_sum += tx.fee;
    }
    BZK_TRY(b.hash(ctx));
    for (size_t k = 0; k < out->t.size(); k++) {
        wire::UpdateTransition &t = out->t[k];
        t.src_before_balances_hash = b.tok_before(3 * k); t.dst_before_balances_hash = b.tok_before(3 * k + 2);
        t.src_balance_proof = b.tok_proof(3 * k); t.src_fee_balance_proof = b.tok_proof(3 * k + 1); t.dst_balance_proof = b.tok_proof(3 * k + 2);
        t.src_proof = b.state_proof(3 * k); t.dst_proof = b.state_proof(3 * k + 2);
    }
    out->d.roots = b.slot_roots(cap, 3);
    std::vector<Fr> aux_in = {fee_token, fr_from_u64(fee_sum)}, aux;
    BZK_TRY(hash_rows(ctx, 2, aux_in, aux));
    b.commit(aux[0], out->public3);
    return BZK_OK;
}

// `mpn::deposit::deposit` (/root/reference/src/mpn/deposit.rs:11-233) without the L1 balance bookkeeping (chain state): one step
// per deposit
int32_t bzk::mpn_deposit_build_impl(bzk_ctx *ctx, bzk_mpn_state *s, const bzk_mpn_deposit *deps, uint64_t n_deps, uint32_t log4_batch,
                                    Built<wire::DepositTransition> *out) {
    if (!ctx || !s || (n_deps && !deps) || !out || log4_batch > 8) return BZK_ERR_BAD_ARG;
    BZK_CUDA(ctx, cudaSetDevice(ctx->device));
    const uint32_t A = s->A, T = s->T;
    const uint64_t cap = 1ull << (2 * log4_batch);
    BatchCore b(s);
    *out = Built<wire::DepositTransition>();
    out->d.keys.assign(cap, null_key());
    std::vector<Fr> pk_rows;
    std::set<uint64_t> rejected_srcs;   // deposit.rs:33 `rejected_pub_keys`: a rejected deposit takes its L1 source's later ones with it
    for (uint64_t k = 0; k < n_deps && out->t.size() < cap; k++) {
        const bzk_mpn_deposit &d = deps[k];
        auto reject = [&] { if (d.src_id) rejected_srcs.insert(d.src_id); };
        if (!canonical(d.pk_x) || !canonical(d.token_id)) { reject(); continue; }
        Point addr;
        if (!jj_decompress(s, &d.pk_x, d.pk_odd != 0, &addr)) { reject(); continue; }
        uint64_t idx = 0;
        const bool is_new = !b.index_of(addr, &idx);
        if (is_new) idx = b.next_index();
        if (idx >> (2 * A)) { reject(); continue; }
        const Account before = b.get(idx);
        const Fr tok = fr_from_canon(&d.token_id);
        const int ti = find_token_index(before, T, tok, true);
        if (ti < 0 || (d.src_id && rejected_srcs.count(d.src_id)) ||
            (jj_on_curve(before.ax, before.ay, s->jj_d) && (!(before.ax == addr.x) || !(before.ay == addr.y)))) {
            reject();
            continue;
        }
        Account after = before;
        after.ax = addr.x; after.ay = addr.y;
        if (!after.tokens.count(ti)) after.tokens[ti] = Money{tok, 0};
        after.tokens[ti].amount += d.amount;
        b.step(idx, ti, after);
        if (is_new) b.add_account(addr, idx);
        // `DepositTransition` (deposit.rs:150-165)
        wire::DepositTransition t;
        t.enabled = true;
        t.tx.mpn_address = wire::PubKey{addr.x, d.pk_odd != 0};
        t.tx.payment.amount = wire_money(Money{tok, d.amount});
        t.before = wire_account(before);
        t.before_balance = wire_money(before.tokens.count(ti) ? before.tokens.at(ti) : Money{Fr::zero(), 0});
        t.account_index = idx; t.token_index = ti;
        out->d.keys[out->t.size()] = wire::PointW{addr.x, addr.y};
        pk_rows.push_back(addr.x); pk_rows.push_back(addr.y);
        out->t.push_back(std::move(t));
        out->from.push_back(k);
    }
    BZK_TRY(b.hash(ctx));
    std::vector<Fr> pk_hash;
    BZK_TRY(hash_rows(ctx, 2, pk_rows, pk_hash));
    pk_hash.resize(cap, Fr::zero());
    out->d.pk_hash = pk_hash;
    for (size_t k = 0; k < out->t.size(); k++) {
        wire::DepositTransition &t = out->t[k];
        t.before_balances_hash = b.tok_before(k); t.balance_proof = b.tok_proof(k); t.proof = b.state_proof(k);
    }
    out->d.roots = b.slot_roots(cap, 1);
    std::vector<wire::DepositTransition> slots;
    padded(out->t, log4_batch, null_deposit(A, T), slots);
    std::vector<Fr> rev(cap * 4);
    for (uint64_t k = 0; k < cap; k++) deposit_reveal(slots[k], out->d, k, rev.data() + k * 4);
    Fr aux;
    BZK_TRY(list_root(ctx, 4, rev, &aux));
    b.commit(aux, out->public3);
    return BZK_OK;
}

// `mpn::withdraw::withdraw` (/root/reference/src/mpn/withdraw.rs:10-259): nonce, balances and the EdDSA signature over
// Poseidon(fingerprint, nonce) are checked here (the hashes of a batch in two launches, the scalar multiplications on the host);
// two steps per withdrawal (amount, then fee).  A withdrawal creates no account.
int32_t bzk::mpn_withdraw_build_impl(bzk_ctx *ctx, bzk_mpn_state *s, const bzk_mpn_withdraw *wds, uint64_t n_wds, uint32_t log4_batch,
                                     Built<wire::WithdrawTransition> *out) {
    if (!ctx || !s || (n_wds && !wds) || !out || log4_batch > 8) return BZK_ERR_BAD_ARG;
    BZK_CUDA(ctx, cudaSetDevice(ctx->device));
    const uint32_t A = s->A, T = s->T;
    const uint64_t cap = 1ull << (2 * log4_batch);
    // signature material of every candidate in two batched launches: msg = H(fingerprint, nonce), h = H(R.x, R.y, A.x, A.y, msg)
    std::vector<Point> addr(n_wds);
    std::vector<uint8_t> ok(n_wds, 0);
    std::vector<Fr> msg_rows, h_rows, msgs, hs;
    for (uint64_t k = 0; k < n_wds; k++) {
        const bzk_mpn_withdraw &w = wds[k];
        ok[k] = canonical(w.pk_x) && canonical(w.amount_token_id) && canonical(w.fee_token_id) && canonical(w.fingerprint) && canonical(w.sig_rx) &&
                canonical(w.sig_ry) && canonical(w.sig_s) && jj_decompress(s, &w.pk_x, w.pk_odd != 0, &addr[k]);
        msg_rows.push_back(ok[k] ? fr_from_canon(&w.fingerprint) : Fr::zero());
        msg_rows.push_back(fr_from_u64(w.nonce));
    }
    BZK_TRY(hash_rows(ctx, 2, msg_rows, msgs));
    for (uint64_t k = 0; k < n_wds; k++) {
        const bzk_mpn_withdraw &w = wds[k];
        h_rows.push_back(ok[k] ? fr_from_canon(&w.sig_rx) : Fr::zero()); h_rows.push_back(ok[k] ? fr_from_canon(&w.sig_ry) : Fr::zero());
        h_rows.push_back(ok[k] ? addr[k].x : Fr::zero()); h_rows.push_back(ok[k] ? addr[k].y : Fr::zero()); h_rows.push_back(msgs[k]);
    }
    BZK_TRY(hash_rows(ctx, 5, h_rows, hs));
    // `verify_calldata` (src/core/transaction.rs:177-182, withdraw.rs:77) for the entries that carry the payment's calldata
    bool any_calldata = false;
    for (uint64_t k = 0; k < n_wds; k++) any_calldata |= wds[k].check_calldata != 0;
    if (any_calldata) {
        std::vector<Fr> rows, cd;
        for (uint64_t k = 0; k < n_wds; k++) {
            const bzk_mpn_withdraw &w = wds[k];
            const bool on = ok[k] && w.check_calldata;
            rows.push_back(on ? addr[k].x : Fr::zero()); rows.push_back(on ? addr[k].y : Fr::zero()); rows.push_back(fr_from_u64(w.nonce));
            rows.push_back(on ? fr_from_canon(&w.sig_rx) : Fr::zero()); rows.push_back(on ? fr_from_canon(&w.sig_ry) : Fr::zero());
            rows.push_back(on ? fr_from_canon(&w.sig_s) : Fr::zero());
        }
        BZK_TRY(hash_rows(ctx, 6, rows, cd));
        for (uint64_t k = 0; k < n_wds; k++)
            if (ok[k] && wds[k].check_calldata && (!canonical(wds[k].calldata) || !(cd[k] == fr_from_canon(&wds[k].calldata)))) ok[k] = 0;
    }
    BatchCore b(s);
    *out = Built<wire::WithdrawTransition>();
    out->d.keys.assign(cap, null_key());
    out->d.fingerprint.assign(cap, Fr::zero());
    std::vector<Fr> cd_rows;
    for (uint64_t k = 0; k < n_wds && out->t.size() < cap; k++) {
        if (!ok[k]) continue;
        const bzk_mpn_withdraw &w = wds[k];
        uint64_t idx = 0;
        if (!b.index_of(addr[k], &idx)) continue;
        const Account before = b.get(idx);
        const Fr tok = fr_from_canon(&w.amount_token_id), ftok = fr_from_canon(&w.fee_token_id);
        const int ti = find_token_index(before, T, tok, false), fi = find_token_index(before, T, ftok, false);
        if (ti < 0 || fi < 0 || w.nonce != before.withdraw_nonce + 1) continue;
        if (before.tokens.at(ti).amount < w.amount) continue;
        Fr sig_s;
        memcpy(sig_s.l, &w.sig_s, 32);
        const Point sig_r{fr_from_canon(&w.sig_rx), fr_from_canon(&w.sig_ry)};
        if (!eddsa_verify_with_h(s, addr[k], sig_r, sig_s, hs[k])) continue;
        Account mid = before;
        mid.tokens[ti].amount -= w.amount;
        if (mid.tokens.at(fi).amount < w.fee) continue;
        Account after = mid;
        after.tokens[fi].amount -= w.fee;
        after.withdraw_nonce += 1;
        b.step(idx, ti, mid);
        b.step(idx, fi, after);
        // `WithdrawTransition` (withdraw.rs:160-178)
        wire::WithdrawTransition t;
        t.enabled = true;
        t.tx.mpn_address = wire::PubKey{addr[k].x, w.pk_odd != 0};
        t.tx.nonce = w.nonce;
        t.tx.sig.r = wire::PointW{sig_r.x, sig_r.y}; t.tx.sig.s = fr_from_canon(&w.sig_s);
        t.tx.payment.amount = wire_money(Money{tok, w.amount}); t.tx.payment.fee = wire_money(Money{ftok, w.fee});
        t.before = wire_account(before); t.before_token_balance = wire_money(before.tokens.at(ti)); t.before_fee_balance = wire_money(mid.tokens.at(fi));
        t.account_index = idx; t.token_index = ti; t.fee_token_index = fi;
        const size_t slot = out->t.size();
        out->d.keys[slot] = wire::PointW{addr[k].x, addr[k].y};
        out->d.fingerprint[slot] = fr_from_canon(&w.fingerprint);
        for (const Fr &v : {addr[k].x, addr[k].y, fr_from_u64(w.nonce), sig_r.x, sig_r.y, t.tx.sig.s}) cd_rows.push_back(v);
        out->t.push_back(std::move(t));
        out->from.push_back(k);
    }
    BZK_TRY(b.hash(ctx));
    std::vector<Fr> cds;
    BZK_TRY(hash_rows(ctx, 6, cd_rows, cds));
    cds.resize(cap, Fr::zero());
    out->d.calldata = cds;
    for (size_t k = 0; k < out->t.size(); k++) {
        wire::WithdrawTransition &t = out->t[k];
        t.before_token_hash = b.tok_before(2 * k); t.token_balance_proof = b.tok_proof(2 * k); t.fee_balance_proof = b.tok_proof(2 * k + 1);
        t.proof = b.state_proof(2 * k);
    }
    out->d.roots = b.slot_roots(cap, 2);
    std::vector<wire::WithdrawTransition> slots;
    padded(out->t, log4_batch, null_withdraw(A, T), slots);
    std::vector<Fr> rev(cap * 7);
    for (uint64_t k = 0; k < cap; k++) withdraw_reveal(slots[k], out->d, k, rev.data() + k * 7);
    Fr aux;
    BZK_TRY(list_root(ctx, 7, rev, &aux));
    b.commit(aux, out->public3);
    return BZK_OK;
}

extern "C" {

/* The builders' C ABI (include/bzk.h): the rows of the padded batch by the circuit's writer (csrc/mpn_wire.cu).  The ledger
 * advances (build on a clone, see bzk_mpn_state_clone). */
int32_t bzk_mpn_update_build(bzk_ctx *ctx, bzk_mpn_state *s, const bzk_mpn_tx *txs, uint64_t n_txs, uint32_t log4_batch,
                             const bzk_fr *fee_token_canon, bzk_fr *raws, bzk_fr *ext, uint8_t *accepted, bzk_fr public3[3],
                             uint64_t *n_accepted) {
    if (!raws || !ext || !public3 || !n_accepted) return BZK_ERR_BAD_ARG;
    Built<wire::UpdateTransition> bt;
    BZK_TRY(mpn_update_build_impl(ctx, s, txs, n_txs, log4_batch, fee_token_canon, &bt));
    std::vector<wire::UpdateTransition> slots;
    padded(bt.t, log4_batch, null_update(s->A, s->T), slots);
    BZK_TRY(write_update_rows(slots, bt.d, s->A, s->T, fr_from_canon(fee_token_canon), raws, ext));
    report(bt, n_txs, accepted, public3, n_accepted);
    return BZK_OK;
}

int32_t bzk_mpn_deposit_build(bzk_ctx *ctx, bzk_mpn_state *s, const bzk_mpn_deposit *deps, uint64_t n_deps, uint32_t log4_batch, bzk_fr *raws1,
                              bzk_fr *raws2, bzk_fr *roots, bzk_fr *reveal, uint8_t *accepted, bzk_fr public3[3], uint64_t *n_accepted) {
    if (!raws1 || !raws2 || !roots || !reveal || !public3 || !n_accepted) return BZK_ERR_BAD_ARG;
    Built<wire::DepositTransition> bt;
    BZK_TRY(mpn_deposit_build_impl(ctx, s, deps, n_deps, log4_batch, &bt));
    std::vector<wire::DepositTransition> slots;
    padded(bt.t, log4_batch, null_deposit(s->A, s->T), slots);
    BZK_TRY(write_deposit_rows(slots, bt.d, s->A, s->T, raws1, raws2, roots, reveal));
    report(bt, n_deps, accepted, public3, n_accepted);
    return BZK_OK;
}

int32_t bzk_mpn_withdraw_build(bzk_ctx *ctx, bzk_mpn_state *s, const bzk_mpn_withdraw *wds, uint64_t n_wds, uint32_t log4_batch, bzk_fr *raws1,
                               bzk_fr *raws2, bzk_fr *roots, bzk_fr *reveal, uint8_t *accepted, bzk_fr public3[3], uint64_t *n_accepted) {
    if (!raws1 || !raws2 || !roots || !reveal || !public3 || !n_accepted) return BZK_ERR_BAD_ARG;
    Built<wire::WithdrawTransition> bt;
    BZK_TRY(mpn_withdraw_build_impl(ctx, s, wds, n_wds, log4_batch, &bt));
    std::vector<wire::WithdrawTransition> slots;
    padded(bt.t, log4_batch, null_withdraw(s->A, s->T), slots);
    BZK_TRY(write_withdraw_rows(slots, bt.d, s->A, s->T, raws1, raws2, roots, reveal));
    report(bt, n_wds, accepted, public3, n_accepted);
    return BZK_OK;
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------
// witness of a whole deposit / withdraw batch from the builder's rows: what `{Deposit,Withdraw}Circuit::synthesize`
// assigns (/root/reference/src/mpn/circuits/deposit_circuit.rs:47-293, withdraw_circuit.rs:49-413), laid out as
//   inputs = [1, commitment, height, state, aux_data, next_state]
//   aux    = [the five public values] ++ phase-1 program x n_slots ++ reveal program ++ phase-2 program x n_slots
// phase 2's externals per slot: ext_src[e] < 0 -> the state root entering the slot, else phase-1 raw ext_src[e] of the slot
// (bzk_mpn_circuit_two_phase_info); the reveal program's externals are the builder's reveal rows, slot-major.
// ---------------------------------------------------------------------------------------------
extern "C" int32_t bzk_mpn_dw_witness(bzk_ctx *ctx, const bzk_witness_program *phase1, const bzk_witness_program *phase2,
                                      const bzk_witness_program *reveal_prog, uint64_t n_slots, const bzk_fr *raws1, const bzk_fr *raws2,
                                      const bzk_fr *roots, const int32_t *ext_src, uint32_t n_ext_src, const bzk_fr *reveal_rows,
                                      const bzk_fr public5[5], void *d_inputs, void *d_aux) {
    if (!ctx || !phase1 || !phase2 || !reveal_prog || !n_slots || !raws1 || !raws2 || !roots || (n_ext_src && !ext_src) || !reveal_rows || !public5 ||
        !d_inputs || !d_aux)
        return BZK_ERR_BAD_ARG;
    uint64_t n1 = 0, n2 = 0, nr = 0;
    uint32_t raw1 = 0, ext1 = 0, raw2 = 0, ext2 = 0, rawr = 0, extr = 0;
    witness_program_shape(phase1, &n1, &raw1, &ext1);
    witness_program_shape(phase2, &n2, &raw2, &ext2);
    witness_program_shape(reveal_prog, &nr, &rawr, &extr);
    if (ext1 != 0 || ext2 != n_ext_src || extr % n_slots != 0) return BZK_ERR_BAD_ARG;
    for (uint32_t e = 0; e < n_ext_src; e++)
        if (ext_src[e] >= (int32_t)raw1) return BZK_ERR_BAD_ARG;
    BZK_CUDA(ctx, cudaSetDevice(ctx->device));
    Fr head[11];
    head[0] = Fr::one();
    for (int k = 0; k < 5; k++) { head[1 + k] = fr_from_canon(public5 + k); head[6 + k] = head[1 + k]; }
    Fr *z_in = (Fr *)d_inputs, *z_aux = (Fr *)d_aux;
    BZK_CUDA(ctx, cudaMemcpyAsync(z_in, head, 6 * sizeof(Fr), cudaMemcpyHostToDevice, ctx->stream));
    BZK_CUDA(ctx, cudaMemcpyAsync(z_aux, head + 6, 5 * sizeof(Fr), cudaMemcpyHostToDevice, ctx->stream));
    BZK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // `head` is a stack buffer
    BZK_TRY(bzk_witness_run_dev(ctx, phase1, raws1, nullptr, n_slots, z_aux + 5));
    BZK_TRY(bzk_witness_run_dev(ctx, reveal_prog, nullptr, reveal_rows, 1, z_aux + 5 + n_slots * n1));
    std::vector<bzk_fr> ext((size_t)n_slots * n_ext_src);
    for (uint64_t k = 0; k < n_slots; k++)
        for (uint32_t e = 0; e < n_ext_src; e++) ext[k * n_ext_src + e] = ext_src[e] < 0 ? roots[k] : raws1[k * raw1 + ext_src[e]];
    BZK_TRY(bzk_witness_run_dev(ctx, phase2, raws2, ext.data(), n_slots, z_aux + 5 + n_slots * n1 + nr));
    return BZK_OK;
}

// ---------------------------------------------------------------------------------------------
// witness of a whole update batch from the builder's rows: what `UpdateCircuit::synthesize` assigns
// (/root/reference/src/mpn/circuits/update_circuit.rs:49-494), laid out as z = inputs ++ aux:
//   inputs  = [1, commitment, height, state, aux_data, next_state]
//   aux     = [commitment, height, state, fee_token, aux_data, next_state]      (the six prologue allocations)
//             ++ slot program x n_slots                                          (bzk_witness_run_dev)
//             ++ epilogue program (the Poseidon(fee_token, sum of accepted fees) gadget; externals =
//                fee_token, then every slot's accepted fee)
// ---------------------------------------------------------------------------------------------
extern "C" int32_t bzk_mpn_update_witness(bzk_ctx *ctx, const bzk_witness_program *slot_prog, const bzk_witness_program *epilogue_prog,
                                          uint64_t n_slots, uint32_t log4_token, uint64_t slot_vars, uint64_t epilogue_vars, const bzk_fr *raws,
                                          const bzk_fr *ext, uint32_t n_raw, const bzk_fr prologue[6], void *d_inputs, void *d_aux) {
    if (!ctx || !slot_prog || !epilogue_prog || !n_slots || !raws || !ext || !prologue || !d_inputs || !d_aux || n_raw < 16 + 3 * log4_token)
        return BZK_ERR_BAD_ARG;
    {   // the rows must have the shape the two programs were compiled for (a mismatch would read / write out of bounds)
        uint64_t s_ops = 0, e_ops = 0;
        uint32_t s_raw = 0, s_ext = 0, e_raw = 0, e_ext = 0;
        witness_program_shape(slot_prog, &s_ops, &s_raw, &s_ext);
        witness_program_shape(epilogue_prog, &e_ops, &e_raw, &e_ext);
        if (s_raw != n_raw || s_ext != 2 || s_ops != slot_vars || e_ext != 1 + n_slots || e_ops != epilogue_vars) return BZK_ERR_BAD_ARG;
    }
    BZK_CUDA(ctx, cudaSetDevice(ctx->device));
    Fr head[12];  // 6 inputs, 6 prologue aux (Montgomery)
    const Fr commitment = fr_from_canon(prologue + 0), height = fr_from_canon(prologue + 1), state = fr_from_canon(prologue + 2),
             fee_token = fr_from_canon(prologue + 3), aux_data = fr_from_canon(prologue + 4), next_state = fr_from_canon(prologue + 5);
    head[0] = Fr::one(); head[1] = commitment; head[2] = height; head[3] = state; head[4] = aux_data; head[5] = next_state;
    head[6] = commitment; head[7] = height; head[8] = state; head[9] = fee_token; head[10] = aux_data; head[11] = next_state;
    Fr *z_in = (Fr *)d_inputs, *z_aux = (Fr *)d_aux;
    BZK_CUDA(ctx, cudaMemcpyAsync(z_in, head, 6 * sizeof(Fr), cudaMemcpyHostToDevice, ctx->stream));
    BZK_CUDA(ctx, cudaMemcpyAsync(z_aux, head + 6, 6 * sizeof(Fr), cudaMemcpyHostToDevice, ctx->stream));
    BZK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // `head` is a stack buffer
    BZK_TRY(bzk_witness_run_dev(ctx, slot_prog, raws, ext, n_slots, z_aux + 6));
    // accepted fee of a slot = enabled ? tx.fee : 0; both are raw inputs (positions 0 and 15 + 3T of a row)
    std::vector<bzk_fr> epi_ext(1 + n_slots);
    epi_ext[0] = prologue[3];
    const bzk_fr zero{};
    for (uint64_t k = 0; k < n_slots; k++) {
        const bzk_fr *row = raws + k * n_raw;
        epi_ext[1 + k] = row[0].l[0] ? row[15 + 3 * log4_token] : zero;
    }
    BZK_TRY(bzk_witness_run_dev(ctx, epilogue_prog, nullptr, epi_ext.data(), 1, z_aux + 6 + n_slots * slot_vars));
    return BZK_OK;
}

// `PublicKey::decompress` as a stand-alone host call (no context): x canonical, y parity flag -> affine point
// (canonical); BZK_ERR_NOT_ON_CURVE when x is not the abscissa of a curve point.
extern "C" int32_t bzk_jubjub_decompress(const bzk_fr *jubjub_d, const bzk_fr *x, int32_t y_is_odd, bzk_fr out_xy[2]) {
    if (!jubjub_d || !x || !out_xy) return BZK_ERR_BAD_ARG;
    bzk_mpn_state tmp;
    tmp.jj_d = fr_from_canon(jubjub_d);
    Point p;
    if (!jj_decompress(&tmp, x, y_is_odd != 0, &p) || !jj_on_curve(p.x, p.y, tmp.jj_d)) return BZK_ERR_NOT_ON_CURVE;
    fr_to_canon(out_xy + 0, p.x);
    fr_to_canon(out_xy + 1, p.y);
    return BZK_OK;
}
