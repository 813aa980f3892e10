// bazuka_b200 — G1 instantiation of the Pippenger MSM (see msm_impl.cuh for the algorithm).
// Kept in its own translation unit so the G1 and G2 kernels compile in parallel.
#include "msm_impl.cuh"

namespace bzk {

int32_t msm_g1_run(bzk_ctx *ctx, const BasesRef<Fp> &d_bases, const Fr *d_scalars, size_t n, bzk_g1_affine *out) {
    return msm_run<Fp>(ctx, d_bases, d_scalars, n, out);
}
int32_t msm_g1_enqueue(bzk_ctx *ctx, cudaStream_t st, void **ws, size_t *ws_bytes, StreamPipe *pipe, const BasesRef<Fp> &d_bases,
                       const Fr *d_scalars, size_t n, void *h_win, MsmPlan *plan) {
    return msm_enqueue<Fp>(ctx, st, ws, ws_bytes, pipe, false, d_bases, d_scalars, n, (Xyzz<Fp> *)h_win, plan);
}
void msm_g1_finish(const MsmPlan *plan, const void *h_win, bzk_g1_affine *out) { msm_host_finish<Fp>(*plan, (const Xyzz<Fp> *)h_win, out); }
int32_t precompute_g1(bzk_ctx *ctx, bzk_g1_bases *b, uint32_t max_levels) {
    if (b->tab_T > 1) return BZK_OK;
    return bases_precompute<Fp>(ctx, &b->d, b->n, max_levels, &b->tab_c, &b->tab_T, &b->tab_G);
}
int32_t pack_g1(bzk_ctx *ctx, const uint8_t *d_images, size_t n, G1Affine *d_out, uint32_t *d_bad) {
    if (n == 0) return BZK_OK;
    k_pack_g1<<<div_up(n, 256), 256, 0, ctx->stream>>>(d_images, n, d_out, d_bad);
    BZK_LAUNCHED(ctx);
    return BZK_OK;
}
int32_t random_g1(bzk_ctx *ctx, uint64_t seed, size_t n, uint8_t *d_out) {
    if (n == 0) return BZK_OK;
    k_random_g1<<<div_up(n, 128), 128, 0, ctx->stream>>>(seed, n, g1_generator(), d_out);
    BZK_LAUNCHED(ctx);
    return BZK_OK;
}
int32_t random_fr(bzk_ctx *ctx, uint64_t seed, size_t n, Fr *d_out) {
    if (n == 0) return BZK_OK;
    k_random_fr<<<div_up(n, 256), 256, 0, ctx->stream>>>(seed, n, d_out);
    BZK_LAUNCHED(ctx);
    return BZK_OK;
}
int32_t host_g1_add(const bzk_g1_affine *a, const bzk_g1_affine *b, bzk_g1_affine *out) {
    G1Xyzz acc = G1Xyzz::from_affine(from_wire(a));
    acc.madd(from_wire(b));
    to_wire(out, acc.to_affine());
    return BZK_OK;
}

}  // namespace bzk
