// bazuka_b200 — the MPN worker: a node's `GetMpnWorkResponse` bytes in, the `PostMpnSolutionRequest` bytes out (the reference's
// external prover between `GET /bincode/mpn/work` and `POST /bincode/mpn/solution`, src/mpn/mod.rs:79-129).
//
//   bzk_mpn_worker_create          config -> the three circuits compiled once (update: blocked) -> one bzk_mpn_prover per context
//                                  and kind, each key checked against the config's verifying key and its circuit's R1CS
//   bzk_mpn_worker_prove_response  decode -> filter (foreign config) -> blinding -> one host thread per context, largest circuit
//                                  first -> self-check (bzk_groth16_verify_batch per kind) -> encode
// Host code only: the device work is the prover's (rows, witness, Groth16), on the context each thread owns.
#include <sys/random.h>

#include <algorithm>
#include <atomic>
#include <cerrno>
#include <chrono>
#include <memory>
#include <thread>

#include "mpn_wire.cuh"

using namespace bzk;

namespace {
using Clock = std::chrono::steady_clock;
double ms_since(Clock::time_point t0) { return std::chrono::duration<double, std::milli>(Clock::now() - t0).count(); }

// vk image offsets (`Groth16VerifyingKey` bincode): alpha_g1, beta_g1, beta_g2, gamma_g2, delta_g1, delta_g2, |ic|, ic
constexpr size_t kVkAlphaG1 = 0, kVkBetaG1 = 97, kVkBetaG2 = 194, kVkDeltaG1 = 580, kVkDeltaG2 = 677, kVkHead = 878;

// the key's alpha_g1, beta_g1, beta_g2, delta_g1, delta_g2 against the verifying key the node holds for its kind
int32_t key_matches_vk(const bzk_groth16_params *params, const std::vector<uint8_t> &vk) {
    if (vk.size() < kVkHead) return BZK_ERR_BAD_ARG;
    bzk_g1_affine a1, b1, d1;
    bzk_g2_affine b2, d2;
    BZK_TRY(bzk_groth16_params_info(params, nullptr, &a1, &b1, &b2, &d1, &d2));
    const uint8_t *v = vk.data();
    const bool same = !memcmp(&a1, v + kVkAlphaG1, 97) && !memcmp(&b1, v + kVkBetaG1, 97) && !memcmp(&b2, v + kVkBetaG2, 193) &&
                      !memcmp(&d1, v + kVkDeltaG1, 97) && !memcmp(&d2, v + kVkDeltaG2, 193);
    return same ? BZK_OK : BZK_ERR_BAD_ARG;
}

bool os_random(uint8_t *out, size_t n) {
    while (n) {
        const ssize_t k = getrandom(out, n, 0);
        if (k < 0) {
            if (errno == EINTR) continue;
            return false;
        }
        out += k; n -= (size_t)k;
    }
    return true;
}

// a blinding scalar (Montgomery): 64 OS bytes reduced mod r, or SHA3(seed || id || tag) mod r (the test hook)
bool blinding(const uint8_t *seed32, uint64_t id, char tag, Fr *out) {
    if (seed32) {
        uint8_t msg[41], h[32];
        memcpy(msg, seed32, 32);
        for (int i = 0; i < 8; i++) msg[32 + i] = (uint8_t)(id >> (8 * i));
        msg[40] = (uint8_t)tag;
        wire::sha3_256(msg, sizeof msg, h);
        *out = wire::fr_from_le_bytes_mod_r(h);
        return true;
    }
    uint8_t b[64];
    if (!os_random(b, sizeof b)) return false;
    // lo + hi * 2^256 mod r: fr_from_le_bytes_mod_r gives x*R, so hi's term is (hi*R)*R = to_mont of hi's image
    *out = wire::fr_from_le_bytes_mod_r(b) + wire::fr_from_le_bytes_mod_r(b + 32).to_mont();
    return true;
}

// errors that say the device or the host is in trouble, not the work
bool fatal(int32_t st) { return st == BZK_ERR_CUDA || st == BZK_ERR_OOM || st == BZK_ERR_NO_DEVICE || st == BZK_ERR_NO_PARAMS; }
}  // namespace

struct bzk_mpn_worker {
    wire::Config config;
    struct Device {
        bzk_ctx *ctx = nullptr;
        bzk_mpn_prover *prover[3] = {nullptr, nullptr, nullptr};   // MpnWorkData order: deposit, withdraw, update
    };
    std::vector<Device> devs;
    bzk_groth16_pvk *pvk[3] = {nullptr, nullptr, nullptr};
    uint64_t rows[3] = {0, 0, 0};   // constraints of each served circuit: the larger goes first
    double last_ms[4] = {0, 0, 0, 0};
};

extern "C" {

int32_t bzk_mpn_worker_free(bzk_mpn_worker *w) {
    if (!w) return BZK_OK;
    for (auto &d : w->devs)
        for (auto *p : d.prover)
            if (p) bzk_mpn_prover_free(d.ctx, p);
    for (auto *k : w->pvk)
        if (k) bzk_groth16_pvk_free(k);
    delete w;
    return BZK_OK;
}

int32_t bzk_mpn_worker_create(const uint8_t *config_bytes, size_t config_len, const bzk_mpn_worker_device *devices, uint32_t n_devices,
                              const uint8_t *poseidon_blob, size_t blob_len, const bzk_fr jubjub[3], const bzk_fr *fee_token, bzk_mpn_worker **out) {
    if (!config_bytes || !devices || !n_devices || !poseidon_blob || !jubjub || !fee_token || !out) return BZK_ERR_BAD_ARG;
    for (uint32_t i = 0; i < n_devices; i++)
        if (!devices[i].ctx) return BZK_ERR_BAD_ARG;
    std::unique_ptr<bzk_mpn_worker, int32_t (*)(bzk_mpn_worker *)> w(new (std::nothrow) bzk_mpn_worker, bzk_mpn_worker_free);
    if (!w) return BZK_ERR_OOM;
    if (!wire::dec_config_bytes(config_bytes, config_len, w->config)) return BZK_ERR_BAD_ARG;
    const wire::Config &cf = w->config;
    w->devs.resize(n_devices);
    for (uint32_t i = 0; i < n_devices; i++) w->devs[i].ctx = devices[i].ctx;
    const uint32_t log4_batch[3] = {cf.log4_deposit_batch, cf.log4_withdraw_batch, cf.log4_update_batch};
    for (uint32_t k = 0; k < 3; k++) {
        bool served = false;
        for (uint32_t i = 0; i < n_devices; i++) served |= devices[i].params[k] != nullptr;
        if (!served) continue;
        for (uint32_t i = 0; i < n_devices; i++)
            if (devices[i].params[k]) BZK_TRY(key_matches_vk(devices[i].params[k], cf.vk[k]));
        BZK_TRY(bzk_groth16_pvk_from_bytes(cf.vk[k].data(), cf.vk[k].size(), &w->pvk[k]));
        bzk_mpn_circuit *c = nullptr;
        BZK_TRY(k == wire::KIND_UPDATE
                    ? bzk_mpn_update_circuit_compile_blocked(cf.log4_tree, cf.log4_token, log4_batch[k], poseidon_blob, blob_len, jubjub, &c)
                    : bzk_mpn_dw_circuit_compile(k + 1, cf.log4_tree, cf.log4_token, log4_batch[k], poseidon_blob, blob_len, jubjub, &c));
        std::unique_ptr<bzk_mpn_circuit, int32_t (*)(bzk_mpn_circuit *)> circuit(c, bzk_mpn_circuit_free);
        uint64_t shape[12];
        BZK_TRY(bzk_mpn_circuit_shape(c, shape));
        w->rows[k] = shape[2];
        for (uint32_t i = 0; i < n_devices; i++) {
            if (!devices[i].params[k]) continue;
            BZK_TRY(bzk_mpn_prover_create(devices[i].ctx, c, devices[i].params[k], &jubjub[0], fee_token, &w->devs[i].prover[k]));
            BZK_TRY(mpn_prover_key_check(w->devs[i].prover[k], devices[i].params[k]));
        }
    }
    *out = w.release();
    return BZK_OK;
}

int32_t bzk_mpn_worker_prove_response(bzk_mpn_worker *w, const uint8_t *response, size_t len, const uint8_t prover_address[32], const uint8_t *seed32,
                                      uint8_t **solution, size_t *solution_len, int32_t *status_each, uint64_t status_cap, uint64_t *n_works) {
    if (!w || !response || !prover_address || !solution || !solution_len || (status_cap && !status_each)) return BZK_ERR_BAD_ARG;
    const auto t_call = Clock::now();
    *solution = nullptr; *solution_len = 0;
    if (len < 8) return BZK_ERR_BAD_ARG;
    uint64_t count = 0;
    memcpy(&count, response, 8);
    const uint64_t cap = std::min<uint64_t>(count, 1u << 16);   // the decoder refuses more
    std::vector<uint64_t> ids(cap + 1);
    std::vector<bzk_mpn_work *> raw(cap + 1, nullptr);
    uint64_t n = 0;
    BZK_TRY(bzk_mpn_get_work_response_decode(response, len, ids.data(), raw.data(), cap, &n));
    std::vector<std::unique_ptr<bzk_mpn_work, int32_t (*)(bzk_mpn_work *)>> works;
    for (uint64_t j = 0; j < n; j++) works.emplace_back(raw[j], bzk_mpn_work_free);

    // which works are the worker's: this config's shape for the kind and the same verifying-key bytes; blinding for those
    const wire::Config &cf = w->config;
    const uint32_t log4_batch[3] = {cf.log4_deposit_batch, cf.log4_withdraw_batch, cf.log4_update_batch};
    std::vector<int32_t> status(n, BZK_OK);
    std::vector<uint32_t> kind(n, 0);
    std::vector<bzk_fr> r(n), s(n);
    std::vector<uint8_t> zk(n * 391);
    std::vector<uint64_t> order;
    for (uint64_t j = 0; j < n; j++) {
        bzk_mpn_work_info info;
        BZK_TRY(bzk_mpn_work_get_info(works[j].get(), &info));
        const uint8_t *vk = nullptr;
        size_t vk_len = 0;
        BZK_TRY(bzk_mpn_work_vk(works[j].get(), &vk, &vk_len));
        const uint32_t k = kind[j] = info.kind;
        bool served = false;
        for (auto &d : w->devs) served |= d.prover[k] != nullptr;
        if (!served || info.log4_tree != cf.log4_tree || info.log4_token != cf.log4_token || info.log4_batch != log4_batch[k] ||
            vk_len != cf.vk[k].size() || memcmp(vk, cf.vk[k].data(), vk_len)) {
            status[j] = BZK_ERR_BAD_ARG;
            continue;
        }
        Fr rv, sv;
        if (!blinding(seed32, ids[j], 'r', &rv) || !blinding(seed32, ids[j], 's', &sv)) return BZK_ERR_BAD_ARG;
        memcpy(&r[j], rv.l, 32); memcpy(&s[j], sv.l, 32);
        order.push_back(j);
    }
    std::stable_sort(order.begin(), order.end(), [&](uint64_t a, uint64_t b) { return w->rows[kind[a]] > w->rows[kind[b]]; });

    // one thread per context; each takes the next unclaimed work of a kind it serves
    std::unique_ptr<std::atomic<bool>[]> taken(new std::atomic<bool>[n ? n : 1]);
    for (uint64_t j = 0; j < n; j++) taken[j] = false;
    std::vector<double> witness_ms(w->devs.size(), 0.0), prove_ms(w->devs.size(), 0.0);
    auto run = [&](size_t di) {
        auto &d = w->devs[di];
        for (uint64_t j : order) {
            bzk_mpn_prover *p = d.prover[kind[j]];
            if (!p || taken[j].exchange(true)) continue;
            const auto t0 = Clock::now();
            double wit = 0;
            try {
                status[j] = mpn_prover_prove(d.ctx, p, works[j].get(), prover_address, &r[j], &s[j], 1, &zk[j * 391], &wit);
            } catch (...) {
                status[j] = BZK_ERR_OOM;
            }
            witness_ms[di] += wit;
            prove_ms[di] += ms_since(t0) - wit;
        }
    };
    if (w->devs.size() == 1) {
        run(0);
    } else {
        std::vector<std::thread> threads;
        for (size_t di = 0; di < w->devs.size(); di++) threads.emplace_back(run, di);
        for (auto &t : threads) t.join();
    }
    for (uint64_t j = 0; j < n; j++)
        if (fatal(status[j])) return status[j];

    // self-check: every kept proof against its work's verifying key (the worker's, byte for byte) and public inputs
    const auto t_check = Clock::now();
    for (uint32_t k = 0; k < 3; k++) {
        std::vector<uint64_t> js;
        for (uint64_t j = 0; j < n; j++)
            if (kind[j] == k && status[j] == BZK_OK) js.push_back(j);
        if (js.empty()) continue;
        std::vector<bzk_fr> inputs(js.size() * 5);
        std::vector<uint8_t> proofs(js.size() * 387), ok(js.size(), 0);
        for (size_t q = 0; q < js.size(); q++) {
            BZK_TRY(bzk_mpn_work_public_inputs(works[js[q]].get(), prover_address, &inputs[q * 5]));
            memcpy(&proofs[q * 387], &zk[js[q] * 391 + 4], 387);
        }
        uint64_t batch_seed = 0;
        if (!os_random((uint8_t *)&batch_seed, sizeof batch_seed)) return BZK_ERR_BAD_ARG;
        const int32_t v = bzk_groth16_verify_batch(w->pvk[k], inputs.data(), 5, proofs.data(), js.size(), batch_seed, 0, ok.data());
        if (v < 0) return v;
        for (size_t q = 0; q < js.size(); q++)
            if (!ok[q]) status[js[q]] = BZK_ERR_REJECTED;
    }
    const double check_ms = ms_since(t_check);

    std::vector<uint64_t> kept_ids;
    std::vector<uint8_t> kept;
    for (uint64_t j = 0; j < n; j++) {
        if (status[j] != BZK_OK) continue;
        kept_ids.push_back(ids[j]);
        kept.insert(kept.end(), &zk[j * 391 + 4], &zk[j * 391 + 391]);
    }
    size_t sz = 0;
    BZK_TRY(bzk_mpn_post_solution_request_encode(prover_address, kept_ids.data(), kept.data(), kept_ids.size(), nullptr, 0, &sz));
    uint8_t *buf = (uint8_t *)malloc(sz ? sz : 1);
    if (!buf) return BZK_ERR_OOM;
    const int32_t st = bzk_mpn_post_solution_request_encode(prover_address, kept_ids.data(), kept.data(), kept_ids.size(), buf, sz, &sz);
    if (st != BZK_OK) { free(buf); return st; }
    *solution = buf; *solution_len = sz;
    for (uint64_t j = 0; j < n && j < status_cap; j++) status_each[j] = status[j];
    if (n_works) *n_works = n;
    double wit_sum = 0, prove_sum = 0;
    for (size_t di = 0; di < w->devs.size(); di++) { wit_sum += witness_ms[di]; prove_sum += prove_ms[di]; }
    w->last_ms[0] = ms_since(t_call); w->last_ms[1] = wit_sum; w->last_ms[2] = prove_sum; w->last_ms[3] = check_ms;
    return BZK_OK;
}

int32_t bzk_mpn_worker_last_timing(const bzk_mpn_worker *w, double ms[4]) {
    if (!w || !ms) return BZK_ERR_BAD_ARG;
    memcpy(ms, w->last_ms, sizeof w->last_ms);
    return BZK_OK;
}

}  // extern "C"
