// TEST INFRASTRUCTURE (CPU tier only) — never linked into libbzk.so.
//
// The stand-ins of mpn_shim.cpp, plus what the MPN worker (csrc/mpn_worker.cu) reaches beyond them, so that the worker runs
// on the host build of libbzk's MPN sources (tests/test_mpn_worker_cpu.py):
//   * bzk_groth16_prove_dev    -> mpn_shim.cpp's satisfiability check, then a "proof" that carries r in a.x and s in c.x, so
//                                 that the bytes show which blinding scalars a proof was made with;
//   * bzk_r1cs_upload_blocked  -> the blocked matrices expanded on the host into mpn_shim.cpp's explicit CSR;
//   * bzk_r1cs_shape           -> bellman's domain and density counts of that CSR;
//   * the prepared verifying key and bzk_groth16_verify_batch -> accept every proof, or reject all while shim_reject_all(1);
//   * shim_params_create       -> a key handle with the given vector lengths and vk points (the vectors hold no points).
#define bzk_groth16_prove_dev shim_base_prove_dev
#include "mpn_shim.cpp"
#undef bzk_groth16_prove_dev

static int g_reject_all = 0;
static uint64_t g_verify_calls = 0, g_verify_proofs = 0;

extern "C" {
int32_t bzk_groth16_prove_dev(bzk_ctx *ctx, const bzk_groth16_params *params, const bzk_r1cs *r, const void *d_inputs, const void *d_aux, const bzk_fr *rr,
                              const bzk_fr *ss, int32_t check_satisfied, bzk_g1_affine *pa, bzk_g2_affine *pb, bzk_g1_affine *pc) {
    BZK_TRY(shim_base_prove_dev(ctx, params, r, d_inputs, d_aux, rr, ss, check_satisfied, pa, pb, pc));
    pa->infinity = pc->infinity = 0;
    memcpy(pa->x, rr, 32);
    memcpy(pc->x, ss, 32);
    return BZK_OK;
}

int32_t bzk_r1cs_upload_blocked(bzk_ctx *ctx, uint64_t ni, uint64_t na, uint64_t head, uint64_t tmpl, uint64_t reps, uint64_t tail, uint64_t var_lo,
                                uint64_t stride, const uint64_t *const rowptr[3], const uint32_t *const col[3], const bzk_fr *const val[3], bzk_r1cs **out) {
    if (!ctx || !out) return BZK_ERR_BAD_ARG;
    const uint64_t rows = head + reps * tmpl + tail;
    std::vector<uint64_t> rp[3];
    std::vector<uint32_t> cl[3];
    std::vector<bzk_fr> vl[3];
    for (int s = 0; s < 3; s++) {
        rp[s].push_back(0);
        auto copy_rows = [&](uint64_t lo, uint64_t n, uint64_t shift) {
            for (uint64_t row = lo; row < lo + n; row++) {
                for (uint64_t k = rowptr[s][row]; k < rowptr[s][row + 1]; k++) {
                    const uint32_t c = col[s][k];
                    cl[s].push_back(c >= var_lo ? (uint32_t)(c + shift) : c);
                    vl[s].push_back(val[s][k]);
                }
                rp[s].push_back(cl[s].size());
            }
        };
        copy_rows(0, head, 0);
        for (uint64_t k = 0; k < reps; k++) copy_rows(head, tmpl, k * stride);
        copy_rows(head + tmpl, tail, 0);
        cl[s].push_back(0);
        vl[s].push_back(bzk_fr{});
    }
    return bzk_r1cs_upload(ctx, ni, na, rows, rp[0].data(), cl[0].data(), vl[0].data(), rp[1].data(), cl[1].data(), vl[1].data(), rp[2].data(),
                           cl[2].data(), vl[2].data(), out);
}

// {log2 m, m - 1, num_aux, num_inputs + |A aux density|, |B density|} as groth16.cu derives them
int32_t bzk_r1cs_shape(const bzk_r1cs *r, uint64_t out[5]) {
    if (!r || !out) return BZK_ERR_BAD_ARG;
    uint64_t log_m = 0;
    while ((1ull << log_m) < r->ncons + r->ni) log_m++;
    std::vector<uint8_t> a(r->ni + r->na, 0), b(r->ni + r->na, 0);
    for (size_t k = 0; k < r->col[0].size(); k++) if (!r->val[0][k].is_zero()) a[r->col[0][k]] = 1;
    for (size_t k = 0; k < r->col[1].size(); k++) if (!r->val[1][k].is_zero()) b[r->col[1][k]] = 1;
    uint64_t na = r->ni, nb = 0;
    for (uint64_t v = r->ni; v < a.size(); v++) na += a[v];
    for (uint64_t v = 0; v < b.size(); v++) nb += b[v];
    const uint64_t o[5] = {log_m, (1ull << log_m) - 1, r->na, na, nb};
    memcpy(out, o, sizeof o);
    return BZK_OK;
}

struct bzk_groth16_pvk { int unused; };
int32_t bzk_groth16_pvk_from_bytes(const uint8_t *vk, size_t len, bzk_groth16_pvk **out) {
    if (!vk || len < 878 || !out) return BZK_ERR_BAD_ARG;
    *out = new bzk_groth16_pvk{0};
    return BZK_OK;
}
int32_t bzk_groth16_pvk_free(bzk_groth16_pvk *k) {
    delete k;
    return BZK_OK;
}
int32_t bzk_groth16_verify_batch(const bzk_groth16_pvk *k, const bzk_fr *, size_t n_inputs, const uint8_t *proofs, size_t m, uint64_t, int32_t,
                                 uint8_t *ok_each) {
    if (!k || n_inputs != 5 || (m && !proofs)) return BZK_ERR_BAD_ARG;
    g_verify_calls++;
    g_verify_proofs += m;
    if (ok_each) memset(ok_each, g_reject_all ? 0 : 1, m);
    return g_reject_all ? 0 : 1;
}
void shim_reject_all(int on) { g_reject_all = on; }
uint64_t shim_verify_calls(uint64_t *proofs) {
    if (proofs) *proofs = g_verify_proofs;
    return g_verify_calls;
}

// lens = {h, l, a, b_g1, b_g2}; vk = a Groth16VerifyingKey image whose points the handle takes as its own
bzk_groth16_params *shim_params_create(const uint64_t lens[5], const uint8_t *vk) {
    auto *p = new bzk_groth16_params();
    bzk_g1_affine g1[3];
    bzk_g2_affine g2[2];
    memset(g1, 0, sizeof g1); memset(g2, 0, sizeof g2);
    memcpy(&g1[0], vk + 0, 97); memcpy(&g1[1], vk + 97, 97); memcpy(&g1[2], vk + 580, 97);
    memcpy(&g2[0], vk + 194, 193); memcpy(&g2[1], vk + 677, 193);
    p->alpha_g1 = from_wire(&g1[0]); p->beta_g1 = from_wire(&g1[1]); p->delta_g1 = from_wire(&g1[2]);
    p->beta_g2 = from_wire(&g2[0]); p->delta_g2 = from_wire(&g2[1]);
    p->h = new bzk_g1_bases(); p->h->n = lens[0];
    p->l = new bzk_g1_bases(); p->l->n = lens[1];
    p->a = new bzk_g1_bases(); p->a->n = lens[2];
    p->b1 = new bzk_g1_bases(); p->b1->n = lens[3];
    p->b2 = new bzk_g2_bases(); p->b2->n = lens[4];
    return p;
}
void shim_params_free(bzk_groth16_params *p) {
    if (!p) return;
    delete p->h; delete p->l; delete p->a; delete p->b1; delete p->b2;
    delete p;
}
}
