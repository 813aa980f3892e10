// bazuka_b200 — the worker protocol's wire types (host only): what a Bazuka node hands an MPN prover and takes back.
//
//   MpnWork {config, public_inputs, data, new_root, reward}       /root/reference/src/mpn/mod.rs:264-270
//   MpnConfig, MpnWorkData, ZkPublicInputs                        /root/reference/src/mpn/mod.rs:203-262
//   {Deposit,Withdraw,Update}Transition                           /root/reference/src/mpn/mod.rs:427-537
//   MpnAccount, MpnTransaction, MpnDeposit, MpnWithdraw, Money    /root/reference/src/zk/mod.rs:60-94,573-644, src/core/transaction.rs:120-189
//
// bincode 1.x default options (`bincode::serialize`): little-endian fixed-width integers, `usize` and every length prefix as
// u64, enum variant index as u32, bool / Option tag one byte, structs and fixed arrays as their fields back to back.  Field
// elements travel as their raw MONTGOMERY limbs (`ZkScalar([u64;4])`, serde derive on the tuple struct) and are kept that way
// here (bzk::Fr).  `HashMap`s are kept as vectors in arrival order, so a decoded work re-encodes to the bytes it came from.
// ed25519 `Address` / `Signature` (un-vendored crate, restated from its serde behaviour): `serialize_bytes`, u64 length + bytes.
#pragma once
#include <string>
#include <utility>
#include <vector>

#include "common.cuh"

namespace bzk {

inline Fr fr_from_u64(uint64_t v) {   // Montgomery
    Fr a = Fr::zero();
    a.l[0] = (uint32_t)v;
    a.l[1] = (uint32_t)(v >> 32);
    return a.to_mont();
}
inline void fr_to_canon(bzk_fr *out, const Fr &mont) { const Fr c = mont.from_mont(); memcpy(out, c.l, 32); }

// Widths of the circuits' rows (elements per slot): UpdateCircuit's raws; the deposit / withdraw circuits' phase-1 raws, phase-2
// raws and revealed rows.
inline uint32_t update_raw_width(uint32_t A, uint32_t T) { return 32 + 9 * T + 6 * A; }
struct DwWidths { uint32_t raw1, raw2, reveal; };
inline DwWidths deposit_widths(uint32_t A, uint32_t T) { return {5, 9 + 3 * T + 3 * A, 4}; }
inline DwWidths withdraw_widths(uint32_t A, uint32_t T) { return {12, 12 + 6 * T + 3 * A, 7}; }

namespace wire {

struct ContractId {          // TokenId / ContractId::{Null, Ziesha, Custom(scalar)}
    uint32_t tag = 0;
    Fr custom = Fr::zero();  // Montgomery, tag 2 only
    // `impl From<TokenId> for ZkScalar` (/root/reference/src/zk/mod.rs:280-288), Montgomery
    Fr scalar() const { return tag == 0 ? Fr::zero() : tag == 1 ? Fr::one() : custom; }
    static ContractId of_scalar(const Fr &s) {
        ContractId c;
        if (s.is_zero()) c.tag = 0;
        else if (s == Fr::one()) c.tag = 1;
        else { c.tag = 2; c.custom = s; }
        return c;
    }
};
struct Money { ContractId token; uint64_t amount = 0; };
struct PointW { Fr x = Fr::zero(), y = Fr::zero(); };             // jubjub::PointAffine
struct PubKey { Fr x = Fr::zero(); bool odd = false; };           // jubjub::PublicKey(PointCompressed(x, is_odd))
struct Sig { PointW r; Fr s = Fr::zero(); };                      // jubjub::Signature
struct Account {
    uint64_t tx_nonce = 0, withdraw_nonce = 0;                    // u32 on the wire
    PointW address;
    std::vector<std::pair<uint64_t, Money>> tokens;               // HashMap<u64, Money>, arrival order
};
struct MpnTx { uint64_t nonce = 0; PubKey src, dst; Money amount, fee; Sig sig; };   // nonce: u32 on the wire
struct ContractDeposit {
    std::string memo;
    ContractId contract_id;
    uint32_t circuit_id = 0;
    Fr calldata = Fr::zero();
    uint8_t src[32] = {0};
    Money amount, fee;
    uint32_t nonce = 0;
    bool has_sig = false;
    std::vector<uint8_t> sig;
};
struct ContractWithdraw {
    std::string memo;
    ContractId contract_id;
    uint32_t circuit_id = 0;
    Fr calldata = Fr::zero();
    uint8_t dst[32] = {0};
    Money amount, fee;
};
struct MpnDeposit { PubKey mpn_address; ContractDeposit payment; };
struct MpnWithdraw { PubKey mpn_address; uint32_t nonce = 0; Sig sig; ContractWithdraw payment; };
using Proof = std::vector<Fr>;   // Vec<[ZkScalar; 3]>: 3 per level, leaf level first

struct UpdateTransition {
    bool enabled = false;
    MpnTx tx;
    Account src_before;
    Fr src_before_balances_hash = Fr::zero();
    Money src_before_balance, src_before_fee_balance;
    Proof src_proof;
    uint64_t src_index = 0, src_token_index = 0;
    Proof src_balance_proof;
    uint64_t src_fee_token_index = 0;
    Proof src_fee_balance_proof;
    Account dst_before;
    Fr dst_before_balances_hash = Fr::zero();
    Money dst_before_balance;
    Proof dst_proof;
    uint64_t dst_index = 0, dst_token_index = 0;
    Proof dst_balance_proof;
};
struct DepositTransition {
    bool enabled = false;
    MpnDeposit tx;
    Account before;
    Fr before_balances_hash = Fr::zero();
    Money before_balance;
    Proof proof;
    uint64_t account_index = 0, token_index = 0;
    Proof balance_proof;
};
struct WithdrawTransition {
    bool enabled = false;
    MpnWithdraw tx;
    Account before;
    Money before_token_balance, before_fee_balance;
    Proof proof;
    uint64_t account_index = 0, token_index = 0;
    Proof token_balance_proof;
    Fr before_token_hash = Fr::zero();
    uint64_t fee_token_index = 0;
    Proof fee_balance_proof;
};
struct Config {
    uint8_t log4_tree = 0, log4_token = 0, log4_deposit_batch = 0, log4_withdraw_batch = 0, log4_update_batch = 0;
    ContractId contract_id;
    uint64_t n_update_batches = 0, n_deposit_batches = 0, n_withdraw_batches = 0;
    std::vector<uint8_t> vk[3];   // deposit, withdraw, update: the Groth16VerifyingKey image WITHOUT its u32 enum tag
};
enum : uint32_t { KIND_DEPOSIT = 0, KIND_WITHDRAW = 1, KIND_UPDATE = 2 };   // MpnWorkData variant order
struct Work {
    Config config;
    uint64_t height = 0;
    Fr state = Fr::zero(), aux_data = Fr::zero(), next_state = Fr::zero();
    uint32_t kind = KIND_UPDATE;
    std::vector<DepositTransition> deposits;
    std::vector<WithdrawTransition> withdraws;
    std::vector<UpdateTransition> updates;
    Fr new_root_hash = Fr::zero();
    uint64_t new_root_size = 0;
    uint64_t reward = 0;
    size_t n_transitions() const { return kind == KIND_DEPOSIT ? deposits.size() : kind == KIND_WITHDRAW ? withdraws.size() : updates.size(); }
    uint32_t log4_batch() const {
        return kind == KIND_DEPOSIT ? config.log4_deposit_batch : kind == KIND_WITHDRAW ? config.log4_withdraw_batch : config.log4_update_batch;
    }
};

// ---- bincode
struct Writer {
    std::vector<uint8_t> b;
    void u8(uint8_t v) { b.push_back(v); }
    void boolean(bool v) { b.push_back(v ? 1 : 0); }
    void u32(uint32_t v) { for (int i = 0; i < 4; i++) b.push_back((uint8_t)(v >> (8 * i))); }
    void u64(uint64_t v) { for (int i = 0; i < 8; i++) b.push_back((uint8_t)(v >> (8 * i))); }
    void raw(const void *p, size_t n) { const uint8_t *q = (const uint8_t *)p; b.insert(b.end(), q, q + n); }
    void fr(const Fr &v) { raw(v.l, 32); }
    void bytes(const void *p, size_t n) { u64(n); raw(p, n); }
};
struct Reader {
    const uint8_t *d;
    size_t n, o = 0;
    bool ok = true;
    Reader(const uint8_t *data, size_t len) : d(data), n(len) {}
    const uint8_t *take(size_t k) {
        if (!ok || k > n - o) { ok = false; return nullptr; }
        const uint8_t *p = d + o;
        o += k;
        return p;
    }
    uint8_t u8() { const uint8_t *p = take(1); return p ? *p : 0; }
    bool boolean() { const uint8_t v = u8(); if (v > 1) ok = false; return v == 1; }
    uint32_t u32() { const uint8_t *p = take(4); uint32_t v = 0; if (p) memcpy(&v, p, 4); return v; }
    uint64_t u64() { const uint8_t *p = take(8); uint64_t v = 0; if (p) memcpy(&v, p, 8); return v; }
    Fr fr() {   // raw Montgomery limbs, must be reduced
        Fr v = Fr::zero();
        const uint8_t *p = take(32);
        if (p) {
            memcpy(v.l, p, 32);
            if (Fr::reduce_once(v) != v) { ok = false; v = Fr::zero(); }
        }
        return v;
    }
    uint64_t len(uint64_t limit) { const uint64_t v = u64(); if (v > limit) { ok = false; return 0; } return v; }
};

void enc_work(Writer &w, const Work &work);
bool dec_work(Reader &r, Work &work);
void enc_contract_withdraw(Writer &w, const ContractWithdraw &p);
// `bincode::serialize(&Vec<MpnWithdraw>)` / `&Vec<MpnTransaction>` images; false on a truncated image, trailing bytes, a bad tag
// or an unreduced scalar
bool dec_withdraws(const uint8_t *b, size_t n, std::vector<MpnWithdraw> &out);
bool dec_txs(const uint8_t *b, size_t n, std::vector<MpnTx> &out);
bool dec_deposits(const uint8_t *b, size_t n, std::vector<MpnDeposit> &out);
// bincode of the payment with sig = None: the message its ed25519 signature covers (`ContractDeposit::verify_signature`,
// src/core/transaction.rs:192-201)
void enc_contract_deposit_unsigned(Writer &w, const ContractDeposit &p);
// `bincode::serialize(&MpnConfig)`; false on a truncated image, trailing bytes or a bad tag
bool dec_config_bytes(const uint8_t *b, size_t n, Config &c);

// sha3-256 (FIPS 202) — `Hasher::hash` of the reference (/root/reference/src/crypto/mod.rs, sha3::Sha3_256)
void sha3_256(const uint8_t *data, size_t len, uint8_t out[32]);
// `ZkScalar::new(bytes)` (/root/reference/src/zk/mod.rs:262-271): little-endian integer mod r, Montgomery
Fr fr_from_le_bytes_mod_r(const uint8_t bytes[32]);
// `MpnWork::verify`'s commitment (/root/reference/src/mpn/mod.rs:283-285): ZkScalar::new(sha3(bincode((prover, reward)))), Montgomery
Fr commitment(const uint8_t prover[32], uint64_t reward);
// `ContractWithdraw::fingerprint` (/root/reference/src/core/transaction.rs:205-210): hash-to-scalar of the payment with calldata zeroed
Fr withdraw_fingerprint(const ContractWithdraw &p);

}  // namespace wire

// `{Update,Deposit,Withdraw}Transition::null` (/root/reference/src/mpn/mod.rs:440-537): what a batch is padded with — the builders
// and a work carry only the transitions made, the circuit always has 4^B slots
wire::UpdateTransition null_update(uint32_t A, uint32_t T);
wire::DepositTransition null_deposit(uint32_t A, uint32_t T);
wire::WithdrawTransition null_withdraw(uint32_t A, uint32_t T);
// a batch padded to its 4^B slots; false when it holds more transitions than that
template <class Tr>
bool padded(const std::vector<Tr> &ts, uint32_t log4_batch, const Tr &null, std::vector<Tr> &out) {
    if (log4_batch > 8) return false;
    const size_t slots = (size_t)1 << (2 * log4_batch);
    if (ts.size() > slots) return false;
    out = ts;
    out.resize(slots, null);
    return true;
}

// What a slot's circuit rows need besides its transition, one entry per slot of the padded batch (Montgomery): the state root
// entering the slot, the decompressed key of its transaction ((0, -1) for a null slot: `PublicKey::default().decompress()`),
// and per kind the deposit's H(pk), the withdrawal's fingerprint and calldata hash (zero where the slot is not enabled).
struct SlotData { std::vector<Fr> roots; std::vector<wire::PointW> keys; std::vector<Fr> pk_hash, fingerprint, calldata; };

// The one writer of each circuit's rows (canonical scalars), from a padded batch and its SlotData; the builders' C ABI and the
// work decoder both call it.  Update: raws[4^B][update_raw_width], ext[4^B][2] = {fee token, entering root}.  Deposit / withdraw:
// raws1, raws2, the entering roots and the revealed rows ({deposit,withdraw}_widths).
int32_t write_update_rows(const std::vector<wire::UpdateTransition> &ts, const SlotData &d, uint32_t A, uint32_t T, const Fr &fee_token, bzk_fr *raws,
                          bzk_fr *ext);
int32_t write_deposit_rows(const std::vector<wire::DepositTransition> &ts, const SlotData &d, uint32_t A, uint32_t T, bzk_fr *raws1, bzk_fr *raws2,
                           bzk_fr *roots, bzk_fr *reveal);
int32_t write_withdraw_rows(const std::vector<wire::WithdrawTransition> &ts, const SlotData &d, uint32_t A, uint32_t T, bzk_fr *raws1, bzk_fr *raws2,
                            bzk_fr *roots, bzk_fr *reveal);
// a slot's revealed row (Montgomery): deposit {enabled, token, amount, H(pk)}, withdraw {enabled, token, amount, fee token, fee,
// fingerprint, calldata}; the root of their list is the batch's aux_data
void deposit_reveal(const wire::DepositTransition &t, const SlotData &d, size_t slot, Fr out[4]);
void withdraw_reveal(const wire::WithdrawTransition &t, const SlotData &d, size_t slot, Fr out[7]);

// The transition builders of csrc/mpn_host.cu: the transitions of the accepted inputs (`tx` as the builder saw it; from[i] = index
// of the input the i-th transition was made from), their SlotData over the 4^B slots, and {state, aux_data, next_state} (canonical).
template <class Tr>
struct Built {
    std::vector<Tr> t;
    std::vector<uint64_t> from;
    SlotData d;
    bzk_fr public3[3];
};
int32_t mpn_update_build_impl(bzk_ctx *ctx, bzk_mpn_state *s, const bzk_mpn_tx *txs, uint64_t n_txs, uint32_t log4_batch, const bzk_fr *fee_token_canon,
                              Built<wire::UpdateTransition> *out);
int32_t mpn_deposit_build_impl(bzk_ctx *ctx, bzk_mpn_state *s, const bzk_mpn_deposit *deps, uint64_t n_deps, uint32_t log4_batch,
                               Built<wire::DepositTransition> *out);
int32_t mpn_withdraw_build_impl(bzk_ctx *ctx, bzk_mpn_state *s, const bzk_mpn_withdraw *wds, uint64_t n_wds, uint32_t log4_batch,
                                Built<wire::WithdrawTransition> *out);
// bzk_mpn_prover_prove_work on a decoded work (csrc/mpn_prover.cu); witness_ms (optional): milliseconds until the rows and the
// witness were done, the context synchronised for it
int32_t mpn_prover_prove(bzk_ctx *ctx, bzk_mpn_prover *p, const bzk_mpn_work *work, const uint8_t prover_address[32], const bzk_fr *r, const bzk_fr *s,
                         int32_t check_satisfied, uint8_t zkproof391[391], double *witness_ms);
// BZK_OK when the key's five vector lengths are those the prover's uploaded R1CS gives (bzk_r1cs_shape), else BZK_ERR_BAD_ARG
int32_t mpn_prover_key_check(const bzk_mpn_prover *p, const bzk_groth16_params *params);
}  // namespace bzk
