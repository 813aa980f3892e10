// bazuka_b200 — G2 instantiation of the Pippenger MSM (see msm_impl.cuh for the algorithm).
// Kept in its own translation unit so the G1 and G2 kernels compile in parallel.
#include "msm_impl.cuh"

namespace bzk {

int32_t msm_g2_run(bzk_ctx *ctx, const BasesRef<Fp2> &d_bases, const Fr *d_scalars, size_t n, bzk_g2_affine *out) {
    return msm_run<Fp2>(ctx, d_bases, d_scalars, n, out);
}
int32_t msm_g2_enqueue(bzk_ctx *ctx, cudaStream_t st, void **ws, size_t *ws_bytes, StreamPipe *pipe, const BasesRef<Fp2> &d_bases,
                       const Fr *d_scalars, size_t n, void *h_win, MsmPlan *plan) {
    return msm_enqueue<Fp2>(ctx, st, ws, ws_bytes, pipe, false, d_bases, d_scalars, n, (Xyzz<Fp2> *)h_win, plan);
}
void msm_g2_finish(const MsmPlan *plan, const void *h_win, bzk_g2_affine *out) { msm_host_finish<Fp2>(*plan, (const Xyzz<Fp2> *)h_win, out); }
int32_t precompute_g2(bzk_ctx *ctx, bzk_g2_bases *b, uint32_t max_levels) {
    if (b->tab_T > 1) return BZK_OK;
    return bases_precompute<Fp2>(ctx, &b->d, b->n, max_levels, &b->tab_c, &b->tab_T, &b->tab_G);
}
int32_t pack_g2(bzk_ctx *ctx, const uint8_t *d_images, size_t n, G2Affine *d_out, uint32_t *d_bad) {
    if (n == 0) return BZK_OK;
    k_pack_g2<<<div_up(n, 128), 128, 0, ctx->stream>>>(d_images, n, d_out, d_bad);
    BZK_LAUNCHED(ctx);
    return BZK_OK;
}
int32_t random_g2(bzk_ctx *ctx, uint64_t seed, size_t n, uint8_t *d_out) {
    if (n == 0) return BZK_OK;
    k_random_g2<<<div_up(n, 64), 64, 0, ctx->stream>>>(seed, n, g2_generator(), d_out);
    BZK_LAUNCHED(ctx);
    return BZK_OK;
}
int32_t host_g2_add(const bzk_g2_affine *a, const bzk_g2_affine *b, bzk_g2_affine *out) {
    G2Xyzz acc = G2Xyzz::from_affine(from_wire(a));
    acc.madd(from_wire(b));
    to_wire(out, acc.to_affine());
    return BZK_OK;
}

}  // namespace bzk
