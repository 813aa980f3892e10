// bazuka_b200 — the worker protocol natively: bincode of MpnWork and the three messages, MpnWork::verify's commitment, and
// the rows a work's transitions put into the witness programs (host code; the GPU work is in witness.cu / groth16.cu).
//
// This is the external prover's side of the boundary (SURVEY §8b): a Rust node hands `bincode::serialize(&work)` across the
// FFI and gets the 391-byte `ZkProof` back — the types of mpn_wire.cuh mirror the reference's field for field, the codec is
// checked byte for byte against the Python restatement (bazuka_b200/mpn/wire.py) in tests/test_wire_native_cpu.py.
#include "mpn_wire.cuh"

#include <functional>
#include <map>

namespace bzk {
namespace wire {

// ---------------------------------------------------------------- sha3-256
namespace {
inline uint64_t rotl64(uint64_t x, int s) { return s ? (x << s) | (x >> (64 - s)) : x; }
void keccak_f(uint64_t st[25]) {
    static const uint64_t RC[24] = {0x0000000000000001ULL, 0x0000000000008082ULL, 0x800000000000808aULL, 0x8000000080008000ULL, 0x000000000000808bULL,
                                    0x0000000080000001ULL, 0x8000000080008081ULL, 0x8000000000008009ULL, 0x000000000000008aULL, 0x0000000000000088ULL,
                                    0x0000000080008009ULL, 0x000000008000000aULL, 0x000000008000808bULL, 0x800000000000008bULL, 0x8000000000008089ULL,
                                    0x8000000000008003ULL, 0x8000000000008002ULL, 0x8000000000000080ULL, 0x000000000000800aULL, 0x800000008000000aULL,
                                    0x8000000080008081ULL, 0x8000000000008080ULL, 0x0000000080000001ULL, 0x8000000080008008ULL};
    static const int ROT[25] = {0, 1, 62, 28, 27, 36, 44, 6, 55, 20, 3, 10, 43, 25, 39, 41, 45, 15, 21, 8, 18, 2, 61, 56, 14};  // [x + 5y]
    for (int rnd = 0; rnd < 24; rnd++) {
        uint64_t c[5], d[5], b[25];
        for (int x = 0; x < 5; x++) c[x] = st[x] ^ st[x + 5] ^ st[x + 10] ^ st[x + 15] ^ st[x + 20];
        for (int x = 0; x < 5; x++) d[x] = c[(x + 4) % 5] ^ rotl64(c[(x + 1) % 5], 1);
        for (int i = 0; i < 25; i++) st[i] ^= d[i % 5];
        for (int x = 0; x < 5; x++)
            for (int y = 0; y < 5; y++) b[y + 5 * ((2 * x + 3 * y) % 5)] = rotl64(st[x + 5 * y], ROT[x + 5 * y]);
        for (int x = 0; x < 5; x++)
            for (int y = 0; y < 5; y++) st[x + 5 * y] = b[x + 5 * y] ^ (~b[(x + 1) % 5 + 5 * y] & b[(x + 2) % 5 + 5 * y]);
        st[0] ^= RC[rnd];
    }
}
}  // namespace

void sha3_256(const uint8_t *data, size_t len, uint8_t out[32]) {
    constexpr size_t rate = 136;
    uint64_t st[25] = {0};
    uint8_t block[rate];
    while (len >= rate) {
        for (size_t i = 0; i < rate / 8; i++) { uint64_t v; memcpy(&v, data + 8 * i, 8); st[i] ^= v; }
        keccak_f(st);
        data += rate; len -= rate;
    }
    memset(block, 0, rate);
    if (len) memcpy(block, data, len);
    block[len] ^= 0x06;
    block[rate - 1] ^= 0x80;
    for (size_t i = 0; i < rate / 8; i++) { uint64_t v; memcpy(&v, block + 8 * i, 8); st[i] ^= v; }
    keccak_f(st);
    memcpy(out, st, 32);
}

Fr fr_from_le_bytes_mod_r(const uint8_t bytes[32]) {
    Fr v;
    memcpy(v.l, bytes, 32);
    // 2^256 < 5r: a few conditional subtractions (compare-and-subtract, as in common.cuh's splitmix_fr_canonical)
    for (int k = 0; k < 4; k++) v = Fr::reduce_once(v);
    return v.to_mont();
}

Fr commitment(const uint8_t prover[32], uint64_t reward) {
    Writer w;
    w.bytes(prover, 32);
    w.u64(reward);
    uint8_t h[32];
    sha3_256(w.b.data(), w.b.size(), h);
    return fr_from_le_bytes_mod_r(h);
}

Fr withdraw_fingerprint(const ContractWithdraw &p) {
    ContractWithdraw q = p;
    q.calldata = Fr::zero();
    Writer w;
    enc_contract_withdraw(w, q);
    uint8_t h[32];
    sha3_256(w.b.data(), w.b.size(), h);
    return fr_from_le_bytes_mod_r(h);
}

// ---------------------------------------------------------------- leaves
namespace {
constexpr uint64_t kMaxLevels = 64, kMaxTokens = 1u << 16, kMaxBlob = 1u << 24, kMaxTransitions = 1u << 16, kMaxVkInputs = 4096;

void enc_contract_id(Writer &w, const ContractId &c) {
    w.u32(c.tag);
    if (c.tag == 2) w.fr(c.custom);
}
void dec_contract_id(Reader &r, ContractId &c) {
    c.tag = r.u32();
    if (c.tag > 2) r.ok = false;
    c.custom = c.tag == 2 ? r.fr() : Fr::zero();
}
void enc_money(Writer &w, const Money &m) { enc_contract_id(w, m.token); w.u64(m.amount); }
void dec_money(Reader &r, Money &m) { dec_contract_id(r, m.token); m.amount = r.u64(); }
void enc_point(Writer &w, const PointW &p) { w.fr(p.x); w.fr(p.y); }
void dec_point(Reader &r, PointW &p) { p.x = r.fr(); p.y = r.fr(); }
void enc_pubkey(Writer &w, const PubKey &k) { w.fr(k.x); w.boolean(k.odd); }
void dec_pubkey(Reader &r, PubKey &k) { k.x = r.fr(); k.odd = r.boolean(); }
void enc_sig(Writer &w, const Sig &s) { enc_point(w, s.r); w.fr(s.s); }
void dec_sig(Reader &r, Sig &s) { dec_point(r, s.r); s.s = r.fr(); }
void enc_proof(Writer &w, const Proof &p) {
    w.u64(p.size() / 3);
    for (const Fr &v : p) w.fr(v);
}
void dec_proof(Reader &r, Proof &p) {
    const uint64_t n = r.len(kMaxLevels);
    p.resize(r.ok ? n * 3 : 0);
    for (Fr &v : p) v = r.fr();
}
void enc_account(Writer &w, const Account &a) {
    w.u32((uint32_t)a.tx_nonce); w.u32((uint32_t)a.withdraw_nonce); enc_point(w, a.address);
    w.u64(a.tokens.size());
    for (auto &kv : a.tokens) { w.u64(kv.first); enc_money(w, kv.second); }
}
void dec_account(Reader &r, Account &a) {
    a.tx_nonce = r.u32(); a.withdraw_nonce = r.u32(); dec_point(r, a.address);
    const uint64_t n = r.len(kMaxTokens);
    a.tokens.clear();
    for (uint64_t i = 0; r.ok && i < n; i++) {
        std::pair<uint64_t, Money> kv;
        kv.first = r.u64();
        dec_money(r, kv.second);
        a.tokens.push_back(kv);
    }
}
void enc_mpn_tx(Writer &w, const MpnTx &t) {
    w.u32((uint32_t)t.nonce); enc_pubkey(w, t.src); enc_pubkey(w, t.dst); enc_money(w, t.amount); enc_money(w, t.fee); enc_sig(w, t.sig);
}
void dec_mpn_tx(Reader &r, MpnTx &t) {
    t.nonce = r.u32(); dec_pubkey(r, t.src); dec_pubkey(r, t.dst); dec_money(r, t.amount); dec_money(r, t.fee); dec_sig(r, t.sig);
}
void dec_string(Reader &r, std::string &s) {
    const uint64_t n = r.len(kMaxBlob);
    const uint8_t *p = r.take(n);
    s.assign(p ? (const char *)p : "", p ? n : 0);
}
void dec_address(Reader &r, uint8_t out[32]) {   // ed25519 key (ext): serialize_bytes of 32 bytes
    const uint64_t n = r.u64();
    if (n != 32) { r.ok = false; return; }
    const uint8_t *p = r.take(32);
    if (p) memcpy(out, p, 32);
}
// the fields before the Option<Signature> tag
void enc_contract_deposit_head(Writer &w, const ContractDeposit &p) {
    w.bytes(p.memo.data(), p.memo.size()); enc_contract_id(w, p.contract_id); w.u32(p.circuit_id); w.fr(p.calldata);
    w.bytes(p.src, 32); enc_money(w, p.amount); enc_money(w, p.fee); w.u32(p.nonce);
}
void enc_contract_deposit(Writer &w, const ContractDeposit &p) {
    enc_contract_deposit_head(w, p);
    w.u8(p.has_sig ? 1 : 0);
    if (p.has_sig) w.bytes(p.sig.data(), p.sig.size());
}
void dec_contract_deposit(Reader &r, ContractDeposit &p) {
    dec_string(r, p.memo); dec_contract_id(r, p.contract_id); p.circuit_id = r.u32(); p.calldata = r.fr();
    dec_address(r, p.src); dec_money(r, p.amount); dec_money(r, p.fee); p.nonce = r.u32();
    const uint8_t tag = r.u8();
    if (tag > 1) r.ok = false;
    p.has_sig = tag == 1;
    p.sig.clear();
    if (p.has_sig) {
        const uint64_t n = r.len(128);
        const uint8_t *q = r.take(n);
        if (q) p.sig.assign(q, q + n);
    }
}
void dec_contract_withdraw(Reader &r, ContractWithdraw &p) {
    dec_string(r, p.memo); dec_contract_id(r, p.contract_id); p.circuit_id = r.u32(); p.calldata = r.fr();
    dec_address(r, p.dst); dec_money(r, p.amount); dec_money(r, p.fee);
}
void enc_mpn_deposit(Writer &w, const MpnDeposit &d) { enc_pubkey(w, d.mpn_address); enc_contract_deposit(w, d.payment); }
void dec_mpn_deposit(Reader &r, MpnDeposit &d) { dec_pubkey(r, d.mpn_address); dec_contract_deposit(r, d.payment); }
void enc_mpn_withdraw(Writer &w, const MpnWithdraw &d) {
    enc_pubkey(w, d.mpn_address); w.u32(d.nonce); enc_sig(w, d.sig); enc_contract_withdraw(w, d.payment);
}
void dec_mpn_withdraw(Reader &r, MpnWithdraw &d) {
    dec_pubkey(r, d.mpn_address); d.nonce = r.u32(); dec_sig(r, d.sig); dec_contract_withdraw(r, d.payment);
}

// ---------------------------------------------------------------- transitions (field order = the Rust structs')
void enc_update(Writer &w, const UpdateTransition &t) {
    w.boolean(t.enabled); enc_mpn_tx(w, t.tx); enc_account(w, t.src_before); w.fr(t.src_before_balances_hash); enc_money(w, t.src_before_balance);
    enc_money(w, t.src_before_fee_balance); enc_proof(w, t.src_proof); w.u64(t.src_index); w.u64(t.src_token_index); enc_proof(w, t.src_balance_proof);
    w.u64(t.src_fee_token_index); enc_proof(w, t.src_fee_balance_proof); enc_account(w, t.dst_before); w.fr(t.dst_before_balances_hash);
    enc_money(w, t.dst_before_balance); enc_proof(w, t.dst_proof); w.u64(t.dst_index); w.u64(t.dst_token_index); enc_proof(w, t.dst_balance_proof);
}
void dec_update(Reader &r, UpdateTransition &t) {
    t.enabled = r.boolean(); dec_mpn_tx(r, t.tx); dec_account(r, t.src_before); t.src_before_balances_hash = r.fr(); dec_money(r, t.src_before_balance);
    dec_money(r, t.src_before_fee_balance); dec_proof(r, t.src_proof); t.src_index = r.u64(); t.src_token_index = r.u64(); dec_proof(r, t.src_balance_proof);
    t.src_fee_token_index = r.u64(); dec_proof(r, t.src_fee_balance_proof); dec_account(r, t.dst_before); t.dst_before_balances_hash = r.fr();
    dec_money(r, t.dst_before_balance); dec_proof(r, t.dst_proof); t.dst_index = r.u64(); t.dst_token_index = r.u64(); dec_proof(r, t.dst_balance_proof);
}
void enc_deposit(Writer &w, const DepositTransition &t) {
    w.boolean(t.enabled); enc_mpn_deposit(w, t.tx); enc_account(w, t.before); w.fr(t.before_balances_hash); enc_money(w, t.before_balance);
    enc_proof(w, t.proof); w.u64(t.account_index); w.u64(t.token_index); enc_proof(w, t.balance_proof);
}
void dec_deposit(Reader &r, DepositTransition &t) {
    t.enabled = r.boolean(); dec_mpn_deposit(r, t.tx); dec_account(r, t.before); t.before_balances_hash = r.fr(); dec_money(r, t.before_balance);
    dec_proof(r, t.proof); t.account_index = r.u64(); t.token_index = r.u64(); dec_proof(r, t.balance_proof);
}
void enc_withdraw(Writer &w, const WithdrawTransition &t) {
    w.boolean(t.enabled); enc_mpn_withdraw(w, t.tx); enc_account(w, t.before); enc_money(w, t.before_token_balance); enc_money(w, t.before_fee_balance);
    enc_proof(w, t.proof); w.u64(t.account_index); w.u64(t.token_index); enc_proof(w, t.token_balance_proof); w.fr(t.before_token_hash);
    w.u64(t.fee_token_index); enc_proof(w, t.fee_balance_proof);
}
void dec_withdraw(Reader &r, WithdrawTransition &t) {
    t.enabled = r.boolean(); dec_mpn_withdraw(r, t.tx); dec_account(r, t.before); dec_money(r, t.before_token_balance); dec_money(r, t.before_fee_balance);
    dec_proof(r, t.proof); t.account_index = r.u64(); t.token_index = r.u64(); dec_proof(r, t.token_balance_proof); t.before_token_hash = r.fr();
    t.fee_token_index = r.u64(); dec_proof(r, t.fee_balance_proof);
}

// ZkVerifierKey::Groth16(Box<Groth16VerifyingKey>): u32 tag 0 + 870 bytes (alpha_g1, beta_g1, beta_g2, gamma_g2, delta_g1,
// delta_g2) + u64 count + 97 bytes per input point (/root/reference/src/zk/groth16/mod.rs:28-32)
void enc_vk(Writer &w, const std::vector<uint8_t> &blob) { w.u32(0); w.raw(blob.data(), blob.size()); }
void dec_vk(Reader &r, std::vector<uint8_t> &blob) {
    if (r.u32() != 0) r.ok = false;
    const uint8_t *head = r.take(870);
    const uint64_t n = r.len(kMaxVkInputs);
    const uint8_t *ic = r.take(97 * n);
    blob.clear();
    if (!r.ok || !head || (n && !ic)) return;
    blob.insert(blob.end(), head, head + 870);
    for (int i = 0; i < 8; i++) blob.push_back((uint8_t)(n >> (8 * i)));
    if (n) blob.insert(blob.end(), ic, ic + 97 * n);
}
void enc_config(Writer &w, const Config &c) {
    w.u8(c.log4_tree); w.u8(c.log4_token); w.u8(c.log4_deposit_batch); w.u8(c.log4_withdraw_batch); w.u8(c.log4_update_batch);
    enc_contract_id(w, c.contract_id);
    w.u64(c.n_update_batches); w.u64(c.n_deposit_batches); w.u64(c.n_withdraw_batches);
    for (int k = 0; k < 3; k++) enc_vk(w, c.vk[k]);
}
void dec_config(Reader &r, Config &c) {
    c.log4_tree = r.u8(); c.log4_token = r.u8(); c.log4_deposit_batch = r.u8(); c.log4_withdraw_batch = r.u8(); c.log4_update_batch = r.u8();
    dec_contract_id(r, c.contract_id);
    c.n_update_batches = r.u64(); c.n_deposit_batches = r.u64(); c.n_withdraw_batches = r.u64();
    for (int k = 0; k < 3; k++) dec_vk(r, c.vk[k]);
}
}  // namespace

void enc_contract_deposit_unsigned(Writer &w, const ContractDeposit &p) {
    enc_contract_deposit_head(w, p);
    w.u8(0);
}

void enc_contract_withdraw(Writer &w, const ContractWithdraw &p) {
    w.bytes(p.memo.data(), p.memo.size()); enc_contract_id(w, p.contract_id); w.u32(p.circuit_id); w.fr(p.calldata);
    w.bytes(p.dst, 32); enc_money(w, p.amount); enc_money(w, p.fee);
}

void enc_work(Writer &w, const Work &k) {
    enc_config(w, k.config);
    w.u64(k.height); w.fr(k.state); w.fr(k.aux_data); w.fr(k.next_state);
    w.u32(k.kind);
    w.u64(k.n_transitions());
    if (k.kind == KIND_DEPOSIT) for (auto &t : k.deposits) enc_deposit(w, t);
    else if (k.kind == KIND_WITHDRAW) for (auto &t : k.withdraws) enc_withdraw(w, t);
    else for (auto &t : k.updates) enc_update(w, t);
    w.fr(k.new_root_hash); w.u64(k.new_root_size);
    w.u64(k.reward);
}

bool dec_work(Reader &r, Work &k) {
    dec_config(r, k.config);
    k.height = r.u64(); k.state = r.fr(); k.aux_data = r.fr(); k.next_state = r.fr();
    k.kind = r.u32();
    if (k.kind > 2) r.ok = false;
    const uint64_t n = r.len(kMaxTransitions);
    k.deposits.clear(); k.withdraws.clear(); k.updates.clear();
    for (uint64_t i = 0; r.ok && i < n; i++) {
        if (k.kind == KIND_DEPOSIT) { k.deposits.emplace_back(); dec_deposit(r, k.deposits.back()); }
        else if (k.kind == KIND_WITHDRAW) { k.withdraws.emplace_back(); dec_withdraw(r, k.withdraws.back()); }
        else { k.updates.emplace_back(); dec_update(r, k.updates.back()); }
    }
    k.new_root_hash = r.fr(); k.new_root_size = r.u64();
    k.reward = r.u64();
    return r.ok;
}

bool dec_config_bytes(const uint8_t *b, size_t n, Config &c) {
    Reader r(b, n);
    dec_config(r, c);
    return r.ok && r.o == n;
}
// `bincode::serialize(&Vec<T>)`: u64 count, then the elements
bool dec_deposits(const uint8_t *b, size_t n, std::vector<MpnDeposit> &out) {
    Reader r(b, n);
    const uint64_t k = r.len(kMaxTransitions * 16);
    out.clear();
    for (uint64_t i = 0; r.ok && i < k; i++) { out.emplace_back(); dec_mpn_deposit(r, out.back()); }
    return r.ok && r.o == n;
}
bool dec_withdraws(const uint8_t *b, size_t n, std::vector<MpnWithdraw> &out) {
    Reader r(b, n);
    const uint64_t k = r.len(kMaxTransitions * 16);
    out.clear();
    for (uint64_t i = 0; r.ok && i < k; i++) { out.emplace_back(); dec_mpn_withdraw(r, out.back()); }
    return r.ok && r.o == n;
}
bool dec_txs(const uint8_t *b, size_t n, std::vector<MpnTx> &out) {
    Reader r(b, n);
    const uint64_t k = r.len(kMaxTransitions * 16);
    out.clear();
    for (uint64_t i = 0; r.ok && i < k; i++) { out.emplace_back(); dec_mpn_tx(r, out.back()); }
    return r.ok && r.o == n;
}

}  // namespace wire
}  // namespace bzk

// ------------------------------------------------------------------------------------------------ C ABI
using namespace bzk;
using namespace bzk::wire;

struct bzk_mpn_work { Work w; };

namespace {
inline void put_u(bzk_fr *out, uint64_t v) { memset(out, 0, 32); memcpy(out, &v, 8); }

// batched Poseidon, in[n][arity] -> out[n] (Montgomery images): the host hasher, or a context's batched launch
using HashBatch = std::function<int32_t(uint32_t arity, const Fr *in, size_t n, Fr *out)>;

struct RootJob {   // one enabled transition: its account before, the balances hash in its leaf, its index and Merkle proof
    const Account *account;
    Fr balances_hash;
    uint64_t index;
    const Proof *proof;
};

struct RowCtx {
    HashBatch hash;
    const bzk_fr *jj_d;
    // PublicKey::decompress -> affine point
    int32_t decompress(const PubKey &k, PointW *out) const {
        bzk_fr x, xy[2];
        fr_to_canon(&x, k.x);
        BZK_TRY(bzk_jubjub_decompress(jj_d, &x, k.odd ? 1 : 0, xy));
        memcpy(out->x.l, xy + 0, 32); memcpy(out->y.l, xy + 1, 32);
        out->x = out->x.to_mont(); out->y = out->y.to_mont();
        return BZK_OK;
    }
    // The state root each job's transition was built against: leaf H(tx_nonce, withdraw_nonce, addr, balances hash), then
    // `calc_root_poseidon4` (/root/reference/src/zk/groth16/gadgets/merkle/mod.rs:53-65) under the transition's own proof —
    // level-synchronously over all jobs: one batch for the leaves, one per tree level (1 + depth launches for a whole batch
    // instead of (1 + depth) dependent hashes per transaction).
    int32_t entering_roots(const std::vector<RootJob> &jobs, uint32_t depth, std::vector<Fr> &out) const {
        const size_t n = jobs.size();
        out.assign(n, Fr::zero());
        if (n == 0) return BZK_OK;
        std::vector<Fr> in(n * 5), cur(n);
        for (size_t j = 0; j < n; j++) {
            const Account &a = *jobs[j].account;
            Fr *row = in.data() + j * 5;
            row[0] = fr_from_u64(a.tx_nonce); row[1] = fr_from_u64(a.withdraw_nonce); row[2] = a.address.x; row[3] = a.address.y;
            row[4] = jobs[j].balances_hash;
        }
        BZK_TRY(hash(5, in.data(), n, cur.data()));
        in.resize(n * 4);
        for (uint32_t l = 0; l < depth; l++) {
            for (size_t j = 0; j < n; j++) {
                const uint64_t pos = (jobs[j].index >> (2 * l)) & 3;
                const Fr *sib = jobs[j].proof->data() + (size_t)l * 3;
                int w = 0;
                for (uint64_t k = 0; k < 4; k++) in[j * 4 + k] = (k == pos) ? cur[j] : sib[w++];
            }
            BZK_TRY(hash(4, in.data(), n, cur.data()));
        }
        out = cur;
        return BZK_OK;
    }
};

// the state root entering every slot: an enabled transition's own (roots[] of the enabled ones, in slot order); a disabled one
// takes the next enabled slot's, or — after the last enabled slot — where the batch ends (`next_state`; `state` when nothing is
// enabled)
template <class T>
void slot_roots(const std::vector<T> &ts, const Fr &state, const Fr &next_state, const std::vector<Fr> &enabled_roots, std::vector<Fr> &out) {
    const size_t n = ts.size();
    out.assign(n, Fr::zero());
    size_t e = enabled_roots.size();
    Fr carry = e ? next_state : state;
    for (size_t k = n; k-- > 0;) {
        if (ts[k].enabled) carry = enabled_roots[--e];
        out[k] = carry;
    }
}
bool proofs_shaped(const Proof &p, uint32_t levels) { return p.size() == (size_t)levels * 3; }

}  // namespace

extern "C" {

int32_t bzk_mpn_work_decode(const uint8_t *bytes, size_t len, bzk_mpn_work **out, size_t *consumed) {
    if (!bytes || !out) return BZK_ERR_BAD_ARG;
    auto *w = new (std::nothrow) bzk_mpn_work;
    if (!w) return BZK_ERR_OOM;
    Reader r(bytes, len);
    if (!dec_work(r, w->w) || (!consumed && r.o != len)) { delete w; return BZK_ERR_BAD_ARG; }
    if (consumed) *consumed = r.o;
    *out = w;
    return BZK_OK;
}

int32_t bzk_mpn_work_free(bzk_mpn_work *w) {
    delete w;
    return BZK_OK;
}

int32_t bzk_mpn_work_encode(const bzk_mpn_work *w, uint8_t *out, size_t cap, size_t *len) {
    if (!w || !len) return BZK_ERR_BAD_ARG;
    Writer wr;
    enc_work(wr, w->w);
    *len = wr.b.size();
    if (!out) return BZK_OK;
    if (cap < wr.b.size()) return BZK_ERR_BAD_ARG;
    memcpy(out, wr.b.data(), wr.b.size());
    return BZK_OK;
}

int32_t bzk_mpn_work_get_info(const bzk_mpn_work *w, bzk_mpn_work_info *out) {
    if (!w || !out) return BZK_ERR_BAD_ARG;
    const Work &k = w->w;
    memset(out, 0, sizeof *out);
    out->kind = k.kind; out->log4_tree = k.config.log4_tree; out->log4_token = k.config.log4_token; out->log4_batch = k.log4_batch();
    out->n_transitions = k.n_transitions(); out->height = k.height; out->reward = k.reward; out->new_root_size = k.new_root_size;
    fr_to_canon(&out->state, k.state); fr_to_canon(&out->aux_data, k.aux_data); fr_to_canon(&out->next_state, k.next_state);
    fr_to_canon(&out->new_root_hash, k.new_root_hash);
    return BZK_OK;
}

int32_t bzk_mpn_work_vk(const bzk_mpn_work *w, const uint8_t **vk, size_t *len) {
    if (!w || !vk || !len) return BZK_ERR_BAD_ARG;
    const auto &b = w->w.config.vk[w->w.kind];
    *vk = b.data(); *len = b.size();
    return BZK_OK;
}

int32_t bzk_mpn_commitment(const uint8_t prover[32], uint64_t reward, bzk_fr *out) {
    if (!prover || !out) return BZK_ERR_BAD_ARG;
    fr_to_canon(out, commitment(prover, reward));
    return BZK_OK;
}

int32_t bzk_sha3_256(const uint8_t *data, size_t len, uint8_t out[32]) {
    if ((len && !data) || !out) return BZK_ERR_BAD_ARG;
    sha3_256(data, len, out);
    return BZK_OK;
}

/* the five public inputs of `check_proof` for this work and prover (/root/reference/src/mpn/mod.rs:281-295), Montgomery
 * images as bzk_groth16_verify_bytes takes them */
int32_t bzk_mpn_work_public_inputs(const bzk_mpn_work *w, const uint8_t prover[32], bzk_fr out[5]) {
    if (!w || !prover || !out) return BZK_ERR_BAD_ARG;
    const Fr v[5] = {commitment(prover, w->w.reward), fr_from_u64(w->w.height), w->w.state, w->w.aux_data, w->w.next_state};
    memcpy(out, v, sizeof v);
    return BZK_OK;
}

/* `MpnWork::verify` */
int32_t bzk_mpn_work_verify(const bzk_mpn_work *w, const uint8_t prover[32], const uint8_t *proof387) {
    if (!w || !prover || !proof387) return BZK_ERR_BAD_ARG;
    bzk_fr inputs[5];
    BZK_TRY(bzk_mpn_work_public_inputs(w, prover, inputs));
    const auto &vk = w->w.config.vk[w->w.kind];
    return bzk_groth16_verify_bytes(vk.data(), vk.size(), inputs, 5, proof387);
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------ circuit rows
namespace bzk {

UpdateTransition null_update(uint32_t A, uint32_t T) {
    UpdateTransition t;
    t.src_proof.assign(3 * A, Fr::zero()); t.dst_proof.assign(3 * A, Fr::zero());
    t.src_balance_proof.assign(3 * T, Fr::zero()); t.src_fee_balance_proof.assign(3 * T, Fr::zero()); t.dst_balance_proof.assign(3 * T, Fr::zero());
    return t;
}
DepositTransition null_deposit(uint32_t A, uint32_t T) {
    DepositTransition t;
    t.proof.assign(3 * A, Fr::zero()); t.balance_proof.assign(3 * T, Fr::zero());
    return t;
}
WithdrawTransition null_withdraw(uint32_t A, uint32_t T) {
    WithdrawTransition t;
    t.proof.assign(3 * A, Fr::zero()); t.token_balance_proof.assign(3 * T, Fr::zero()); t.fee_balance_proof.assign(3 * T, Fr::zero());
    return t;
}

void deposit_reveal(const DepositTransition &t, const SlotData &d, size_t slot, Fr out[4]) {
    out[0] = t.enabled ? Fr::one() : Fr::zero(); out[1] = t.tx.payment.amount.token.scalar(); out[2] = fr_from_u64(t.tx.payment.amount.amount);
    out[3] = d.pk_hash[slot];   // deposit_circuit.rs: the calldata of a deposit is the hash of its MPN key
}
void withdraw_reveal(const WithdrawTransition &t, const SlotData &d, size_t slot, Fr out[7]) {
    const ContractWithdraw &p = t.tx.payment;
    out[0] = t.enabled ? Fr::one() : Fr::zero(); out[1] = p.amount.token.scalar(); out[2] = fr_from_u64(p.amount.amount);
    out[3] = p.fee.token.scalar(); out[4] = fr_from_u64(p.fee.amount); out[5] = d.fingerprint[slot]; out[6] = d.calldata[slot];
}

namespace {
// appends scalars to one row of a circuit's inputs, canonical
struct RowWriter {
    bzk_fr *row;
    size_t w = 0;
    void fr(const Fr &v) { fr_to_canon(row + (w++), v); }
    void u(uint64_t v) { put_u(row + (w++), v); }
    void proof(const Proof &p) { for (const Fr &v : p) fr(v); }
    void account(const Account &a) { u(a.tx_nonce); u(a.withdraw_nonce); fr(a.address.x); fr(a.address.y); }
    void money(const Money &m) { fr(m.token.scalar()); u(m.amount); }
};
}  // namespace

// the order of UpdateCircuit's allocations (`bazuka_b200/mpn/witness_program.py::raw_values`)
int32_t write_update_rows(const std::vector<UpdateTransition> &ts, const SlotData &d, uint32_t A, uint32_t T, const Fr &fee_token, bzk_fr *raws,
                          bzk_fr *ext) {
    const uint32_t n_raw = update_raw_width(A, T);
    for (size_t s = 0; s < ts.size(); s++) {
        const UpdateTransition &t = ts[s];
        RowWriter r{raws + s * n_raw};
        r.u(t.enabled ? 1 : 0); r.u(t.src_token_index); r.u(t.src_fee_token_index); r.u(t.dst_token_index);
        r.account(t.src_before);
        r.fr(t.src_before_balances_hash); r.fr(t.dst_before_balances_hash);
        r.money(t.src_before_balance); r.money(t.src_before_fee_balance);
        r.proof(t.src_balance_proof);
        r.u(t.tx.amount.amount); r.u(t.tx.fee.amount);
        r.proof(t.src_fee_balance_proof);
        r.u(t.tx.nonce); r.u(t.src_index); r.fr(t.tx.amount.token.scalar()); r.fr(t.tx.fee.token.scalar());
        r.money(t.dst_before_balance);
        r.proof(t.dst_balance_proof);
        r.proof(t.src_proof);
        r.fr(d.keys[s].x); r.fr(d.keys[s].y); r.u(t.dst_index);
        r.account(t.dst_before);
        r.proof(t.dst_proof);
        r.fr(t.tx.sig.r.x); r.fr(t.tx.sig.r.y); r.fr(t.tx.sig.s);
        if (r.w != n_raw) return BZK_ERR_BAD_ARG;
        fr_to_canon(ext + 2 * s, fee_token);
        fr_to_canon(ext + 2 * s + 1, d.roots[s]);
    }
    return BZK_OK;
}

// raws1 {enabled, token, amount, pk.x, pk.y}; raws2 {account index, token index, account before (4), balances hash, balance
// before (2), balance proof, account proof}
int32_t write_deposit_rows(const std::vector<DepositTransition> &ts, const SlotData &d, uint32_t A, uint32_t T, bzk_fr *raws1, bzk_fr *raws2,
                           bzk_fr *roots, bzk_fr *reveal) {
    const DwWidths wd = deposit_widths(A, T);
    for (size_t s = 0; s < ts.size(); s++) {
        const DepositTransition &t = ts[s];
        RowWriter r1{raws1 + s * wd.raw1}, r2{raws2 + s * wd.raw2};
        r1.u(t.enabled ? 1 : 0); r1.money(t.tx.payment.amount); r1.fr(d.keys[s].x); r1.fr(d.keys[s].y);
        r2.u(t.account_index); r2.u(t.token_index); r2.account(t.before);
        r2.fr(t.before_balances_hash); r2.money(t.before_balance);
        r2.proof(t.balance_proof);
        r2.proof(t.proof);
        if (r2.w != wd.raw2) return BZK_ERR_BAD_ARG;
        Fr rv[4];
        deposit_reveal(t, d, s, rv);
        for (int i = 0; i < 4; i++) fr_to_canon(reveal + s * wd.reveal + i, rv[i]);
        fr_to_canon(roots + s, d.roots[s]);
    }
    return BZK_OK;
}

// raws1 {enabled, token, amount, fee token, fee, fingerprint, pk.x, pk.y, nonce, sig.r.x, sig.r.y, sig.s}; raws2 {account index,
// token index, fee token index, account before (4), token-tree hash, balance before (2), its proof, fee balance before (2), its
// proof, account proof}
int32_t write_withdraw_rows(const std::vector<WithdrawTransition> &ts, const SlotData &d, uint32_t A, uint32_t T, bzk_fr *raws1, bzk_fr *raws2,
                            bzk_fr *roots, bzk_fr *reveal) {
    const DwWidths wd = withdraw_widths(A, T);
    for (size_t s = 0; s < ts.size(); s++) {
        const WithdrawTransition &t = ts[s];
        const ContractWithdraw &p = t.tx.payment;
        RowWriter r1{raws1 + s * wd.raw1}, r2{raws2 + s * wd.raw2};
        r1.u(t.enabled ? 1 : 0); r1.money(p.amount); r1.money(p.fee); r1.fr(d.fingerprint[s]);
        r1.fr(d.keys[s].x); r1.fr(d.keys[s].y); r1.u(t.tx.nonce);
        r1.fr(t.tx.sig.r.x); r1.fr(t.tx.sig.r.y); r1.fr(t.tx.sig.s);
        r2.u(t.account_index); r2.u(t.token_index); r2.u(t.fee_token_index); r2.account(t.before);
        r2.fr(t.before_token_hash); r2.money(t.before_token_balance);
        r2.proof(t.token_balance_proof);
        r2.money(t.before_fee_balance);
        r2.proof(t.fee_balance_proof);
        r2.proof(t.proof);
        if (r2.w != wd.raw2) return BZK_ERR_BAD_ARG;
        Fr rv[7];
        withdraw_reveal(t, d, s, rv);
        for (int i = 0; i < 7; i++) fr_to_canon(reveal + s * wd.reveal + i, rv[i]);
        fr_to_canon(roots + s, d.roots[s]);
    }
    return BZK_OK;
}

}  // namespace bzk

namespace {

// An update work's rows (write_update_rows).  The entering roots are not on the wire: recomputed from each transition's own
// account, proof and index.
int32_t update_rows(const Work &k, const RowCtx &rc, const bzk_fr *fee_token, bzk_fr *raws, bzk_fr *ext) {
    const uint32_t A = k.config.log4_tree, T = k.config.log4_token;
    std::vector<UpdateTransition> updates;
    if (!padded(k.updates, k.config.log4_update_batch, null_update(A, T), updates)) return BZK_ERR_BAD_ARG;
    SlotData d;
    d.keys.resize(updates.size());
    std::vector<RootJob> jobs;
    for (size_t s = 0; s < updates.size(); s++) {
        const UpdateTransition &t = updates[s];
        if (!proofs_shaped(t.src_proof, A) || !proofs_shaped(t.dst_proof, A) || !proofs_shaped(t.src_balance_proof, T) ||
            !proofs_shaped(t.src_fee_balance_proof, T) || !proofs_shaped(t.dst_balance_proof, T))
            return BZK_ERR_BAD_ARG;
        BZK_TRY(rc.decompress(t.tx.dst, &d.keys[s]));
        if (t.enabled) jobs.push_back(RootJob{&t.src_before, t.src_before_balances_hash, t.src_index, &t.src_proof});
    }
    std::vector<Fr> enabled_roots;
    BZK_TRY(rc.entering_roots(jobs, A, enabled_roots));
    slot_roots(updates, k.state, k.next_state, enabled_roots, d.roots);
    Fr fee;
    memcpy(fee.l, fee_token, 32);
    return write_update_rows(updates, d, A, T, fee.to_mont(), raws, ext);
}

// A deposit / withdraw work's rows (write_deposit_rows / write_withdraw_rows).  The calldata hash of every enabled slot's
// revealed row in ONE batched hash.
int32_t dw_rows(const Work &k, const RowCtx &rc, bzk_fr *raws1, bzk_fr *raws2, bzk_fr *roots_out, bzk_fr *reveal) {
    const uint32_t A = k.config.log4_tree, T = k.config.log4_token;
    std::vector<Fr> enabled_roots, cd_in, cd;
    std::vector<RootJob> jobs;
    std::vector<size_t> enabled;
    SlotData d;
    auto finish = [&](uint32_t arity, std::vector<Fr> &per_slot) -> int32_t {   // the calldata hashes, spread over the slots
        BZK_TRY(rc.entering_roots(jobs, A, enabled_roots));
        cd.assign(jobs.size(), Fr::zero());
        if (!jobs.empty()) BZK_TRY(rc.hash(arity, cd_in.data(), jobs.size(), cd.data()));
        per_slot.assign(d.keys.size(), Fr::zero());
        for (size_t e = 0; e < enabled.size(); e++) per_slot[enabled[e]] = cd[e];
        return BZK_OK;
    };
    if (k.kind == KIND_DEPOSIT) {
        std::vector<DepositTransition> deposits;
        if (!padded(k.deposits, k.config.log4_deposit_batch, null_deposit(A, T), deposits)) return BZK_ERR_BAD_ARG;
        d.keys.resize(deposits.size());
        for (size_t s = 0; s < deposits.size(); s++) {
            const DepositTransition &t = deposits[s];
            if (!proofs_shaped(t.proof, A) || !proofs_shaped(t.balance_proof, T)) return BZK_ERR_BAD_ARG;
            BZK_TRY(rc.decompress(t.tx.mpn_address, &d.keys[s]));
            if (!t.enabled) continue;
            jobs.push_back(RootJob{&t.before, t.before_balances_hash, t.account_index, &t.proof});
            enabled.push_back(s);
            cd_in.push_back(d.keys[s].x); cd_in.push_back(d.keys[s].y);
        }
        BZK_TRY(finish(2, d.pk_hash));
        slot_roots(deposits, k.state, k.next_state, enabled_roots, d.roots);
        return write_deposit_rows(deposits, d, A, T, raws1, raws2, roots_out, reveal);
    }
    std::vector<WithdrawTransition> withdraws;
    if (!padded(k.withdraws, k.config.log4_withdraw_batch, null_withdraw(A, T), withdraws)) return BZK_ERR_BAD_ARG;
    d.keys.resize(withdraws.size());
    d.fingerprint.assign(withdraws.size(), Fr::zero());
    for (size_t s = 0; s < withdraws.size(); s++) {
        const WithdrawTransition &t = withdraws[s];
        if (!proofs_shaped(t.proof, A) || !proofs_shaped(t.token_balance_proof, T) || !proofs_shaped(t.fee_balance_proof, T)) return BZK_ERR_BAD_ARG;
        BZK_TRY(rc.decompress(t.tx.mpn_address, &d.keys[s]));
        if (!t.enabled) continue;
        jobs.push_back(RootJob{&t.before, t.before_token_hash, t.account_index, &t.proof});
        enabled.push_back(s);
        d.fingerprint[s] = withdraw_fingerprint(t.tx.payment);
        // calldata = H(pk, nonce, sig) (`verify_calldata`, /root/reference/src/core/transaction.rs:177-182)
        cd_in.push_back(d.keys[s].x); cd_in.push_back(d.keys[s].y); cd_in.push_back(Fr::from_u32(t.tx.nonce));
        cd_in.push_back(t.tx.sig.r.x); cd_in.push_back(t.tx.sig.r.y); cd_in.push_back(t.tx.sig.s);
    }
    BZK_TRY(finish(6, d.calldata));
    slot_roots(withdraws, k.state, k.next_state, enabled_roots, d.roots);
    return write_withdraw_rows(withdraws, d, A, T, raws1, raws2, roots_out, reveal);
}

RowCtx host_rows(const bzk_poseidon_host *hasher, const bzk_fr *jj_d) {
    return RowCtx{[hasher](uint32_t arity, const Fr *in, size_t n, Fr *out) { return bzk_poseidon_host_hash(hasher, arity, (const bzk_fr *)in, n, (bzk_fr *)out); },
                  jj_d};
}
RowCtx ctx_rows(bzk_ctx *ctx, const bzk_fr *jj_d) {
    return RowCtx{[ctx](uint32_t arity, const Fr *in, size_t n, Fr *out) { return bzk_poseidon_hash(ctx, arity, (const bzk_fr *)in, n, (bzk_fr *)out); }, jj_d};
}
}  // namespace

extern "C" {

/* host variants: the hashes on the host Poseidon (no GPU context; a node that only wants to LOOK at a work) */
int32_t bzk_mpn_work_update_rows(const bzk_mpn_work *work, const bzk_poseidon_host *hasher, const bzk_fr *jubjub_d, const bzk_fr *fee_token,
                                 bzk_fr *raws, bzk_fr *ext) {
    if (!work || !hasher || !jubjub_d || !fee_token || !raws || !ext || work->w.kind != KIND_UPDATE) return BZK_ERR_BAD_ARG;
    return update_rows(work->w, host_rows(hasher, jubjub_d), fee_token, raws, ext);
}
int32_t bzk_mpn_work_dw_rows(const bzk_mpn_work *work, const bzk_poseidon_host *hasher, const bzk_fr *jubjub_d, bzk_fr *raws1, bzk_fr *raws2,
                             bzk_fr *roots_out, bzk_fr *reveal) {
    if (!work || !hasher || !jubjub_d || !raws1 || !raws2 || !roots_out || !reveal || work->w.kind == KIND_UPDATE) return BZK_ERR_BAD_ARG;
    return dw_rows(work->w, host_rows(hasher, jubjub_d), raws1, raws2, roots_out, reveal);
}
/* the prover's variants: the same rows with every hash in batched launches on the context (1 + A launches for the entering roots
 * of a whole batch, one for the calldata hashes) — what bzk_mpn_prover_prove_work uses */
int32_t bzk_mpn_work_update_rows_ctx(bzk_ctx *ctx, const bzk_mpn_work *work, const bzk_fr *jubjub_d, const bzk_fr *fee_token, bzk_fr *raws, bzk_fr *ext) {
    if (!ctx || !work || !jubjub_d || !fee_token || !raws || !ext || work->w.kind != KIND_UPDATE) return BZK_ERR_BAD_ARG;
    return update_rows(work->w, ctx_rows(ctx, jubjub_d), fee_token, raws, ext);
}
int32_t bzk_mpn_work_dw_rows_ctx(bzk_ctx *ctx, const bzk_mpn_work *work, const bzk_fr *jubjub_d, bzk_fr *raws1, bzk_fr *raws2, bzk_fr *roots_out,
                                 bzk_fr *reveal) {
    if (!ctx || !work || !jubjub_d || !raws1 || !raws2 || !roots_out || !reveal || work->w.kind == KIND_UPDATE) return BZK_ERR_BAD_ARG;
    return dw_rows(work->w, ctx_rows(ctx, jubjub_d), raws1, raws2, roots_out, reveal);
}

/* `GetMpnWorkResponse { works: HashMap<usize, MpnWork> }` (/root/reference/src/client/messages.rs:371-376): up to `cap` works
 * are decoded into ids[] / works[] (free each with bzk_mpn_work_free); *n = the number on the wire. */
int32_t bzk_mpn_get_work_response_decode(const uint8_t *bytes, size_t len, uint64_t *ids, bzk_mpn_work **works, uint64_t cap, uint64_t *n) {
    if (!bytes || !n || (cap && (!ids || !works))) return BZK_ERR_BAD_ARG;
    Reader r(bytes, len);
    const uint64_t count = r.len(1u << 16);
    if (!r.ok) return BZK_ERR_BAD_ARG;
    std::vector<bzk_mpn_work *> got;
    int32_t st = BZK_OK;
    for (uint64_t i = 0; i < count && st == BZK_OK; i++) {
        const uint64_t id = r.u64();
        auto *w = new (std::nothrow) bzk_mpn_work;
        if (!w) { st = BZK_ERR_OOM; break; }
        if (!dec_work(r, w->w)) { delete w; st = BZK_ERR_BAD_ARG; break; }
        if (i < cap) { ids[i] = id; got.push_back(w); }
        else delete w;
    }
    if (st == BZK_OK && r.o != len) st = BZK_ERR_BAD_ARG;
    if (st != BZK_OK) {
        for (auto *w : got) delete w;
        return st;
    }
    for (size_t i = 0; i < got.size(); i++) works[i] = got[i];
    *n = count;
    return BZK_OK;
}

/* `GetMpnWorkRequest { address }` = `PostMpnWorkerRequest`'s body: the 40-byte image of an ed25519 address */
int32_t bzk_mpn_get_work_request_encode(const uint8_t address[32], uint8_t out[40]) {
    if (!address || !out) return BZK_ERR_BAD_ARG;
    Writer w;
    w.bytes(address, 32);
    memcpy(out, w.b.data(), 40);
    return BZK_OK;
}

/* `PostMpnSolutionRequest { prover, proofs: HashMap<usize, ZkProof> }` (messages.rs:378-382); proofs387 = n x 387-byte
 * Groth16Proof images (each goes out as the 391-byte ZkProof::Groth16).  out == NULL sizes the buffer. */
int32_t bzk_mpn_post_solution_request_encode(const uint8_t prover[32], const uint64_t *ids, const uint8_t *proofs387, uint64_t n, uint8_t *out, size_t cap,
                                             size_t *len) {
    if (!prover || !len || (n && (!ids || !proofs387))) return BZK_ERR_BAD_ARG;
    Writer w;
    w.bytes(prover, 32);
    w.u64(n);
    for (uint64_t i = 0; i < n; i++) { w.u64(ids[i]); w.u32(0); w.raw(proofs387 + 387 * i, 387); }
    *len = w.b.size();
    if (!out) return BZK_OK;
    if (cap < w.b.size()) return BZK_ERR_BAD_ARG;
    memcpy(out, w.b.data(), w.b.size());
    return BZK_OK;
}

/* `PostMpnSolutionResponse { accepted: usize }` */
int32_t bzk_mpn_post_solution_response_decode(const uint8_t *bytes, size_t len, uint64_t *accepted) {
    if (!bytes || !accepted || len != 8) return BZK_ERR_BAD_ARG;
    memcpy(accepted, bytes, 8);
    return BZK_OK;
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------ prepare_works
extern "C" {

/* `mpn::prepare_works` (/root/reference/src/mpn/mod.rs:298-424) over the native ledger: on ONE fork of `state` (which is not
 * modified), `mpn_num_deposit_batches` deposit batches, then the withdraw batches, then the update batches — every batch is
 * offered the whole list again (what an earlier batch took is stale for the next), the accounts created on the way are found by
 * the later batches (`new_account_indices`) — and every batch becomes an `MpnWork {config, public_inputs, data, new_root, reward}`.
 * Inputs are the reference's own wire images: `bincode::serialize(&config)`, `&Vec<MpnDeposit>`, `&Vec<MpnWithdraw>`,
 * `&Vec<MpnTransaction>`; rewards = {deposit, withdraw, update}.  What the builders check of the L1 side comes from the payments:
 * a deposit's source (`rejected_pub_keys`), a withdrawal's calldata (`verify_calldata`) and fingerprint.  Output: the bincode of
 * `HashMap<usize, MpnWork>` numbered in building order — the body of `GetMpnWorkResponse` — in a buffer to release with
 * bzk_buffer_free, and the fork (bzk_mpn_state_free it, or bzk_mpn_state_commit_accounts + keep it when the block is applied).
 * The validator's own reward deposit and the L1 balance bookkeeping of that function are chain state: the caller prepends that
 * deposit to the list like the reference does (mod.rs:338-351). */
int32_t bzk_mpn_prepare_works(bzk_ctx *ctx, const bzk_mpn_state *state, const uint8_t *config_bytes, size_t config_len, const uint8_t *deposits_bytes,
                              size_t deposits_len, const uint8_t *withdraws_bytes, size_t withdraws_len, const uint8_t *updates_bytes, size_t updates_len,
                              const uint64_t rewards[3], uint64_t height, const bzk_fr *fee_token, bzk_mpn_state **fork_out, uint8_t **works_bytes,
                              size_t *works_len, uint64_t *n_works) {
    if (!ctx || !state || !config_bytes || !rewards || !fee_token || !fork_out || !works_bytes || !works_len || !n_works) return BZK_ERR_BAD_ARG;
    Config config;
    std::vector<MpnDeposit> deposits;
    std::vector<MpnWithdraw> withdraws;
    std::vector<MpnTx> updates;
    if (!dec_config_bytes(config_bytes, config_len, config)) return BZK_ERR_BAD_ARG;
    if (deposits_bytes && !dec_deposits(deposits_bytes, deposits_len, deposits)) return BZK_ERR_BAD_ARG;
    if (withdraws_bytes && !dec_withdraws(withdraws_bytes, withdraws_len, withdraws)) return BZK_ERR_BAD_ARG;
    if (updates_bytes && !dec_txs(updates_bytes, updates_len, updates)) return BZK_ERR_BAD_ARG;
    {
        bzk_fr root;
        uint64_t sz, cnt, pend;
        BZK_TRY(bzk_mpn_state_info(state, &root, &sz, &cnt, &pend));
        uint32_t shape[2] = {0, 0};
        // the ledger must have the config's shape: the builders size their proofs from the ledger's (A, T), a work's rows from the config's
        if (bzk_mpn_state_shape(state, shape) != BZK_OK || shape[0] != config.log4_tree || shape[1] != config.log4_token || config.log4_deposit_batch > 8 ||
            config.log4_withdraw_batch > 8 || config.log4_update_batch > 8)
            return BZK_ERR_BAD_ARG;
    }
    // ---- the builders' flat inputs
    std::vector<bzk_mpn_deposit> dep_in(deposits.size());
    {
        std::map<std::vector<uint8_t>, uint64_t> src_ids;   // L1 source -> non-zero id (deposit.rs:33 `rejected_pub_keys`)
        for (size_t k = 0; k < deposits.size(); k++) {
            const MpnDeposit &d = deposits[k];
            bzk_mpn_deposit &o = dep_in[k];
            memset(&o, 0, sizeof o);
            fr_to_canon(&o.pk_x, d.mpn_address.x); o.pk_odd = d.mpn_address.odd ? 1 : 0;
            fr_to_canon(&o.token_id, d.payment.amount.token.scalar()); o.amount = d.payment.amount.amount;
            const std::vector<uint8_t> src(d.payment.src, d.payment.src + 32);
            o.src_id = src_ids.emplace(src, src_ids.size() + 1).first->second;
        }
    }
    std::vector<bzk_mpn_withdraw> wd_in(withdraws.size());
    for (size_t k = 0; k < withdraws.size(); k++) {
        const MpnWithdraw &w = withdraws[k];
        bzk_mpn_withdraw &o = wd_in[k];
        memset(&o, 0, sizeof o);
        fr_to_canon(&o.pk_x, w.mpn_address.x); o.pk_odd = w.mpn_address.odd ? 1 : 0; o.nonce = w.nonce;
        fr_to_canon(&o.sig_rx, w.sig.r.x); fr_to_canon(&o.sig_ry, w.sig.r.y); fr_to_canon(&o.sig_s, w.sig.s);
        fr_to_canon(&o.amount_token_id, w.payment.amount.token.scalar()); fr_to_canon(&o.fee_token_id, w.payment.fee.token.scalar());
        fr_to_canon(&o.fingerprint, withdraw_fingerprint(w.payment));
        o.amount = w.payment.amount.amount; o.fee = w.payment.fee.amount;
        o.check_calldata = 1; fr_to_canon(&o.calldata, w.payment.calldata);
    }
    std::vector<bzk_mpn_tx> up_in(updates.size());
    for (size_t k = 0; k < updates.size(); k++) {
        const MpnTx &t = updates[k];
        bzk_mpn_tx &o = up_in[k];
        memset(&o, 0, sizeof o);
        o.nonce = t.nonce; o.amount = t.amount.amount; o.fee = t.fee.amount;
        o.src_pk_odd = t.src.odd ? 1 : 0; o.dst_pk_odd = t.dst.odd ? 1 : 0;
        fr_to_canon(&o.src_pk_x, t.src.x); fr_to_canon(&o.dst_pk_x, t.dst.x);
        fr_to_canon(&o.amount_token_id, t.amount.token.scalar()); fr_to_canon(&o.fee_token_id, t.fee.token.scalar());
        fr_to_canon(&o.sig_rx, t.sig.r.x); fr_to_canon(&o.sig_ry, t.sig.r.y); fr_to_canon(&o.sig_s, t.sig.s);
    }
    // ---- the batches, on one fork
    bzk_mpn_state *fork = nullptr;
    BZK_TRY(bzk_mpn_state_clone(state, &fork));
    std::vector<Work> works;
    int32_t st = BZK_OK;
    auto finish = [&](Work &w, const bzk_fr public3[3], uint32_t kind) -> Work && {
        w.config = config; w.height = height; w.kind = kind;
        Fr v[3];
        for (int i = 0; i < 3; i++) { memcpy(v[i].l, public3 + i, 32); v[i] = v[i].to_mont(); }
        w.state = v[0]; w.aux_data = v[1]; w.next_state = v[2];
        bzk_fr root;
        uint64_t sz = 0;
        bzk_mpn_state_info(fork, &root, &sz, nullptr, nullptr);
        Fr rt;
        memcpy(rt.l, &root, 32);
        w.new_root_hash = rt.to_mont(); w.new_root_size = sz;
        w.reward = rewards[kind];
        return std::move(w);
    };
    // a batch's transitions carry the transaction they were made from, as it came in
    auto add = [&](auto &bt, const auto &inputs, auto &into) {
        for (size_t i = 0; i < bt.t.size(); i++) { bt.t[i].tx = inputs[bt.from[i]]; into.push_back(std::move(bt.t[i])); }
    };
    for (uint64_t b = 0; st == BZK_OK && b < config.n_deposit_batches; b++) {
        Built<DepositTransition> bt;
        Work w;
        st = mpn_deposit_build_impl(ctx, fork, dep_in.data(), dep_in.size(), config.log4_deposit_batch, &bt);
        if (st == BZK_OK) { add(bt, deposits, w.deposits); works.push_back(finish(w, bt.public3, KIND_DEPOSIT)); }
    }
    for (uint64_t b = 0; st == BZK_OK && b < config.n_withdraw_batches; b++) {
        Built<WithdrawTransition> bt;
        Work w;
        st = mpn_withdraw_build_impl(ctx, fork, wd_in.data(), wd_in.size(), config.log4_withdraw_batch, &bt);
        if (st == BZK_OK) { add(bt, withdraws, w.withdraws); works.push_back(finish(w, bt.public3, KIND_WITHDRAW)); }
    }
    for (uint64_t b = 0; st == BZK_OK && b < config.n_update_batches; b++) {
        Built<UpdateTransition> bt;
        Work w;
        st = mpn_update_build_impl(ctx, fork, up_in.data(), up_in.size(), config.log4_update_batch, fee_token, &bt);
        if (st == BZK_OK) { add(bt, updates, w.updates); works.push_back(finish(w, bt.public3, KIND_UPDATE)); }
    }
    if (st != BZK_OK) { bzk_mpn_state_free(fork); return st; }
    Writer out;
    out.u64(works.size());
    for (size_t i = 0; i < works.size(); i++) { out.u64(i); enc_work(out, works[i]); }
    uint8_t *buf = (uint8_t *)malloc(out.b.size() ? out.b.size() : 1);
    if (!buf) { bzk_mpn_state_free(fork); return BZK_ERR_OOM; }
    memcpy(buf, out.b.data(), out.b.size());
    *works_bytes = buf; *works_len = out.b.size(); *n_works = works.size(); *fork_out = fork;
    return BZK_OK;
}

int32_t bzk_buffer_free(uint8_t *buffer) {
    free(buffer);
    return BZK_OK;
}

}  // extern "C"
