// bazuka_b200 — radix-2 NTT over BLS12-381 Fr on sm_90a.
//
// GPU replacement for bellman 0.14.0 `domain::EvaluationDomain::{fft, ifft, coset_fft, icoset_fft,
// divide_by_z_on_coset, mul_assign, sub_assign}` (un-vendored crate; reached from every
// `create_random_proof`, /root/reference/src/mpn/circuits/test.rs:135,175,215).  Same maps as
// bellman: natural order in, natural order out, omega = ROOT_OF_UNITY^(2^(32-log n)), coset
// generator 7, ifft scales by n^-1.
//
// Structure (differs from bellman's bit-reverse-then-DIT on purpose): decimation-in-frequency
// passes of K = 3 stages held in registers (8 elements / thread, twiddles read from a resident
// omega^j table, so a pass costs no extra field products), then one pass that undoes the bit
// reversal and applies whatever per-element scaling the op needs (n^-1, 7^-i).  An Fr element is
// 32 B = one DRAM sector, so the strided element accesses of every pass are sector-exact; a
// 2^24 transform moves 8 x 1 GiB + the permutation.  See DESIGN.md for the roofline.
#include "common.cuh"

namespace bzk {

// ---------------------------------------------------------------------------------------------
// table builders
// ---------------------------------------------------------------------------------------------
// out[j] = base^j for j < count; each thread seeds with a pow and walks `run` entries
__global__ void k_powers(Fr base, Fr *__restrict__ out, size_t count, uint32_t run) {
    size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    size_t j0 = t * run;
    if (j0 >= count) return;
    uint32_t e[2] = {(uint32_t)j0, (uint32_t)(j0 >> 32)};
    Fr v = base.pow(e, 2);
    for (uint32_t k = 0; k < run && j0 + k < count; k++) {
        store_vec(out + j0 + k, v);
        v = v * base;
    }
}

static Fr host_root_of_unity(uint32_t log_n) {
    // ROOT_OF_UNITY = 7^((r-1) >> 32)  (ff derive, generator 7: /root/reference/src/zk/mod.rs:204)
    uint32_t e[8];
    for (int i = 0; i < 8; i++) e[i] = FrParams::p(i);
    e[0] -= 1;
    uint32_t sh[8];
    for (int i = 0; i < 7; i++) sh[i] = e[i + 1];
    sh[7] = 0;
    Fr w = Fr::from_u32(7).pow(sh, 8);
    for (uint32_t i = log_n; i < 32; i++) w = w.sqr();
    return w;
}

// both tables are built into locals and published together: `tb.d_fwd` set means both tables are there.  A failed
// allocation or launch (out of memory on a shared card) frees what was allocated, so a later call retries from scratch
// instead of reading the inverse twiddles through a null pointer.
static int32_t ensure_tables(bzk_ctx *ctx, uint32_t log_n) {
    NttTables &tb = ctx->ntt[log_n];
    if (tb.d_fwd) return BZK_OK;
    size_t half = log_n ? ((size_t)1 << (log_n - 1)) : 1;
    Fr w = host_root_of_unity(log_n);
    Fr wi = w.inv();
    Fr *fwd = nullptr, *inv = nullptr;
    cudaError_t e = cudaMalloc(&fwd, half * sizeof(Fr));
    if (e == cudaSuccess) {
        e = cudaMalloc(&inv, half * sizeof(Fr));
        if (e == cudaSuccess) {
            const uint32_t run = 32;
            uint32_t blocks = div_up(div_up(half, run), 128);
            k_powers<<<blocks, 128, 0, ctx->stream>>>(w, fwd, half, run);
            k_powers<<<blocks, 128, 0, ctx->stream>>>(wi, inv, half, run);
            ctx->launches += 2;
            e = cudaGetLastError();  // a failed launch stays the last error even if the one after it succeeds
            if (e != cudaSuccess) cudaFree(inv);
        }
        if (e != cudaSuccess) cudaFree(fwd);
    }
    if (e != cudaSuccess) {
        cudaGetLastError();  // reported here: the retry's launch check must not find it again
        return set_cuda_err(ctx, e, "ntt twiddle tables", __FILE__, __LINE__);
    }
    tb.d_fwd = fwd;
    tb.d_inv = inv;
    tb.log_n = log_n;
    return BZK_OK;
}

// coset generator powers, two-level: g^i = lo[i & 16383] * hi[i >> 14]; tables for g = 7 and 7^-1
constexpr uint32_t kGpowBits = 14;
constexpr size_t kGpowN = (size_t)1 << kGpowBits;
static int32_t ensure_gpow(bzk_ctx *ctx) {
    if (ctx->d_gpow) return BZK_OK;
    BZK_CUDA(ctx, cudaMalloc(&ctx->d_gpow, 4 * kGpowN * sizeof(Fr)));
    Fr g = Fr::from_u32(7), gi = g.inv();
    uint32_t e[1] = {(uint32_t)kGpowN};
    Fr gh = g.pow(e, 1), gih = gi.pow(e, 1);
    const Fr bases[4] = {g, gh, gi, gih};
    for (int k = 0; k < 4; k++) {
        k_powers<<<div_up(div_up(kGpowN, 32), 128), 128, 0, ctx->stream>>>(bases[k], ctx->d_gpow + k * kGpowN, kGpowN, 32);
        BZK_LAUNCHED(ctx);
    }
    return BZK_OK;
}

// ---------------------------------------------------------------------------------------------
// DIF pass: stages s .. s+K-1 on 2^K register-resident elements per thread
// ---------------------------------------------------------------------------------------------
template <int K>
__global__ void __launch_bounds__(256) k_ntt_dif(Fr *__restrict__ a, const Fr *__restrict__ tw, uint32_t log_n, uint32_t s) {
    const size_t n = (size_t)1 << log_n;
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (n >> K)) return;
    const uint32_t log_h = log_n - s - K;  // h_last = 2^log_h : smallest butterfly distance of the pass
    const size_t h_last = (size_t)1 << log_h;
    const size_t low = t & (h_last - 1);
    const size_t p0 = ((t >> log_h) << (log_h + K)) + low;
    Fr x[1 << K];
#pragma unroll
    for (int m = 0; m < (1 << K); m++) x[m] = load_vec(a + p0 + (size_t)m * h_last);
#pragma unroll
    for (int q = 0; q < K; q++) {
        constexpr int dummy = 0;
        (void)dummy;
        const int d = 1 << (K - 1 - q);
        // table index = low * n/(2 d h_last) + (m mod d) * n/(2d)
        const uint32_t sh_low = log_n - 1 - (K - 1 - q) - log_h;  // log2(n/(2 d h_last)) = s + q
        const uint32_t sh_m = log_n - 1 - (K - 1 - q);
#pragma unroll
        for (int m = 0; m < (1 << K); m++) {
            if (m & d) continue;
            const size_t idx = (low << sh_low) + ((size_t)(m & (d - 1)) << sh_m);
            Fr u = x[m], v = x[m + d];
            x[m] = u + v;
            Fr df = u - v;
            x[m + d] = (idx == 0) ? df : df * load_vec(tw + idx);
        }
    }
#pragma unroll
    for (int m = 0; m < (1 << K); m++) store_vec(a + p0 + (size_t)m * h_last, x[m]);
}

// ---------------------------------------------------------------------------------------------
// DIT pass: stages s .. s+K-1 (butterfly distances 2^s .. 2^(s+K-1)) on 2^K register-resident elements per thread.
// Takes its input in BIT-REVERSED order and leaves natural order after the last pass — what follows a DIF transform
// whose reversal pass was skipped (the quotient pipeline: ifft -> coset_fft needs no permutation in between).
// PRESCALE (first pass only): element at position p is first multiplied by c * g^rev(p) — the n^-1 of the ifft that
// came before and the coset's distribute_powers(7) on the coefficient that sits at p.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ Fr gpow_at(const Fr *lo, const Fr *hi, size_t i);
template <int K, bool PRESCALE>
__global__ void __launch_bounds__(256) k_ntt_dit(Fr *__restrict__ a, const Fr *__restrict__ tw, uint32_t log_n, uint32_t s, Fr c,
                                                 const Fr *__restrict__ glo, const Fr *__restrict__ ghi) {
    const size_t n = (size_t)1 << log_n;
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (n >> K)) return;
    const size_t h0 = (size_t)1 << s;
    const size_t low = t & (h0 - 1);
    const size_t p0 = ((t >> s) << (s + K)) + low;
    Fr x[1 << K];
#pragma unroll
    for (int m = 0; m < (1 << K); m++) {
        const size_t p = p0 + (size_t)m * h0;
        x[m] = load_vec(a + p);
        if (PRESCALE) {
            const size_t coeff = (size_t)(__brevll((unsigned long long)p) >> (64 - log_n));
            x[m] = x[m] * (c * gpow_at(glo, ghi, coeff));
        }
    }
#pragma unroll
    for (int q = 0; q < K; q++) {
        const int d = 1 << q;
        const uint32_t sh = log_n - 1 - s - q;  // log2(n / (2 h)), h = h0 * d
#pragma unroll
        for (int m = 0; m < (1 << K); m++) {
            if (m & d) continue;
            const size_t idx = (low + (size_t)(m & (d - 1)) * h0) << sh;
            const Fr u = x[m];
            const Fr v = (idx == 0) ? x[m + d] : x[m + d] * load_vec(tw + idx);
            x[m] = u + v;
            x[m + d] = u - v;
        }
    }
#pragma unroll
    for (int m = 0; m < (1 << K); m++) store_vec(a + p0 + (size_t)m * h0, x[m]);
}

// ---------------------------------------------------------------------------------------------
// bit-reversal permutation fused with the op's output scaling:
//   mode 0: none     mode 1: * c (n^-1)     mode 2: * c * g^-i (icoset)   (i = natural output index)
// pairs (i, rev i) are swapped by the thread owning the smaller index.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ Fr gpow_at(const Fr *lo, const Fr *hi, size_t i) {
    Fr l = load_vec(lo + (i & (kGpowN - 1)));
    size_t h = i >> kGpowBits;
    if (h == 0) return l;
    return l * load_vec(hi + h);
}

__global__ void __launch_bounds__(256) k_bitrev_scale(Fr *__restrict__ a, uint32_t log_n, int mode, Fr c,
                                                      const Fr *__restrict__ glo, const Fr *__restrict__ ghi) {
    const size_t n = (size_t)1 << log_n;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const size_t j = log_n ? (size_t)(__brevll((unsigned long long)i) >> (64 - log_n)) : 0;
    if (i > j) return;
    Fr vi = load_vec(a + i);  // lands at j
    Fr vj = load_vec(a + j);  // lands at i
    if (mode >= 1) {
        Fr si = c, sj = c;
        if (mode == 2) {
            si = c * gpow_at(glo, ghi, i);
            sj = c * gpow_at(glo, ghi, j);
        }
        vi = vi * sj;
        vj = vj * si;
    }
    store_vec(a + j, vi);
    if (i != j) store_vec(a + i, vj);
}

// a[i] *= c * g^i   (distribute_powers; c folds any constant factor)
__global__ void __launch_bounds__(256) k_scale_powers(Fr *__restrict__ a, size_t n, Fr c, int use_c,
                                                      const Fr *__restrict__ glo, const Fr *__restrict__ ghi) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Fr v = load_vec(a + i) * gpow_at(glo, ghi, i);
    if (use_c) v = v * c;
    store_vec(a + i, v);
}

__global__ void __launch_bounds__(256) k_scale_const(Fr *__restrict__ a, size_t n, Fr c) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    store_vec(a + i, load_vec(a + i) * c);
}

// a[i] = (a[i]*b[i] - c[i]) * zinv     (mul_assign, sub_assign, divide_by_z_on_coset in one pass)
__global__ void __launch_bounds__(256) k_h_pointwise(Fr *__restrict__ a, const Fr *__restrict__ b, const Fr *__restrict__ c,
                                                     size_t n, Fr zinv) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Fr v = load_vec(a + i) * load_vec(b + i) - load_vec(c + i);
    store_vec(a + i, v * zinv);
}

static int32_t run_dif(bzk_ctx *ctx, Fr *d, uint32_t log_n, const Fr *tw) {
    uint32_t s = 0;
    while (s < log_n) {
        uint32_t K = log_n - s >= 3 ? 3 : log_n - s;
        size_t threads = ((size_t)1 << log_n) >> K;
        uint32_t blocks = div_up(threads, 256);
        if (K == 3) k_ntt_dif<3><<<blocks, 256, 0, ctx->stream>>>(d, tw, log_n, s);
        else if (K == 2) k_ntt_dif<2><<<blocks, 256, 0, ctx->stream>>>(d, tw, log_n, s);
        else k_ntt_dif<1><<<blocks, 256, 0, ctx->stream>>>(d, tw, log_n, s);
        BZK_LAUNCHED(ctx);
        s += K;
    }
    return BZK_OK;
}

// bit-reversed in, natural out; the first pass multiplies position p by c * g^rev(p)
static int32_t run_dit_prescaled(bzk_ctx *ctx, Fr *d, uint32_t log_n, const Fr *tw, const Fr &c, const Fr *glo, const Fr *ghi) {
    uint32_t s = 0;
    bool first = true;
    if (log_n == 0) {  // a single element: only the scaling (g^0 = 1)
        k_scale_const<<<1, 256, 0, ctx->stream>>>(d, 1, c);
        BZK_LAUNCHED(ctx);
        return BZK_OK;
    }
    while (s < log_n) {
        const uint32_t K = log_n - s >= 3 ? 3 : log_n - s;
        const size_t threads = ((size_t)1 << log_n) >> K;
        const uint32_t blocks = div_up(threads, 256);
#define BZK_DIT(KK)                                                                                              \
    if (first) k_ntt_dit<KK, true><<<blocks, 256, 0, ctx->stream>>>(d, tw, log_n, s, c, glo, ghi);                \
    else k_ntt_dit<KK, false><<<blocks, 256, 0, ctx->stream>>>(d, tw, log_n, s, c, glo, ghi);
        if (K == 3) { BZK_DIT(3) } else if (K == 2) { BZK_DIT(2) } else { BZK_DIT(1) }
#undef BZK_DIT
        BZK_LAUNCHED(ctx);
        first = false;
        s += K;
    }
    return BZK_OK;
}

int32_t ntt_launch(bzk_ctx *ctx, Fr *d, uint32_t log_n, int32_t op) {
    if (log_n > 28 || op < 0 || op > 3 || !d) return BZK_ERR_BAD_ARG;
    const size_t n = (size_t)1 << log_n;
    BZK_TRY(ensure_tables(ctx, log_n));
    BZK_TRY(ensure_gpow(ctx));
    const NttTables &tb = ctx->ntt[log_n];
    const Fr *glo = ctx->d_gpow, *ghi = ctx->d_gpow + kGpowN;
    const Fr *gilo = ctx->d_gpow + 2 * kGpowN, *gihi = ctx->d_gpow + 3 * kGpowN;
    const uint32_t eb = div_up(n, 256);
    if (op == BZK_NTT_COSET_FFT) {
        k_scale_powers<<<eb, 256, 0, ctx->stream>>>(d, n, Fr::one(), 0, glo, ghi);
        BZK_LAUNCHED(ctx);
    }
    const bool inverse = (op == BZK_NTT_IFFT || op == BZK_NTT_ICOSET_FFT);
    BZK_TRY(run_dif(ctx, d, log_n, inverse ? tb.d_inv : tb.d_fwd));
    Fr c = Fr::one();
    int mode = 0;
    if (inverse) {
        uint32_t e[1] = {log_n};
        c = Fr::from_u32(2).inv().pow(e, 1);  // n^-1 = (2^-1)^log_n
        mode = (op == BZK_NTT_ICOSET_FFT) ? 2 : 1;
    }
    k_bitrev_scale<<<eb, 256, 0, ctx->stream>>>(d, log_n, mode, c, gilo, gihi);
    BZK_LAUNCHED(ctx);
    return BZK_OK;
}

static Fr host_zinv(uint32_t log_n) {
    // (7^n - 1)^-1
    Fr g = Fr::from_u32(7);
    for (uint32_t i = 0; i < log_n; i++) g = g.sqr();
    return (g - Fr::one()).inv();
}

int32_t divide_by_z_launch(bzk_ctx *ctx, Fr *d, uint32_t log_n) {
    if (log_n > 28 || !d) return BZK_ERR_BAD_ARG;
    const size_t n = (size_t)1 << log_n;
    k_scale_const<<<div_up(n, 256), 256, 0, ctx->stream>>>(d, n, host_zinv(log_n));
    BZK_LAUNCHED(ctx);
    return BZK_OK;
}

// one evaluation vector to the coset: ifft then coset_fft, the first half of the quotient pipeline below.  The two
// transforms run WITHOUT the two permutation passes and the two scaling passes in between: the DIF transform leaves the
// coefficients bit-reversed, the DIT transform takes them that way, and its first pass applies n^-1 * 7^i to coefficient
// i on the way in (values identical to the four separate maps)
int32_t groth16_to_coset_launch(bzk_ctx *ctx, Fr *v, uint32_t log_n) {
    if (log_n > 28 || !v) return BZK_ERR_BAD_ARG;
    BZK_TRY(ensure_tables(ctx, log_n));
    BZK_TRY(ensure_gpow(ctx));
    const NttTables &tb = ctx->ntt[log_n];
    uint32_t e[1] = {log_n};
    const Fr ninv = Fr::from_u32(2).inv().pow(e, 1);
    BZK_TRY(run_dif(ctx, v, log_n, tb.d_inv));
    return run_dit_prescaled(ctx, v, log_n, tb.d_fwd, ninv, ctx->d_gpow, ctx->d_gpow + kGpowN);
}

// the second half: a <- coefficients of (a*b - c) / Z from the three vectors on the coset
int32_t groth16_h_combine_launch(bzk_ctx *ctx, Fr *a, Fr *b, Fr *c, uint32_t log_n) {
    if (log_n > 28 || !a || !b || !c) return BZK_ERR_BAD_ARG;
    const size_t n = (size_t)1 << log_n;
    k_h_pointwise<<<div_up(n, 256), 256, 0, ctx->stream>>>(a, b, c, n, host_zinv(log_n));
    BZK_LAUNCHED(ctx);
    return ntt_launch(ctx, a, log_n, BZK_NTT_ICOSET_FFT);
}

// the whole quotient pipeline: a <- coefficients of (a*b - c) / Z from the three evaluation vectors
int32_t groth16_h_launch(bzk_ctx *ctx, Fr *a, Fr *b, Fr *c, uint32_t log_n) {
    if (log_n > 28 || !a || !b || !c) return BZK_ERR_BAD_ARG;
    for (Fr *v : {a, b, c}) BZK_TRY(groth16_to_coset_launch(ctx, v, log_n));
    return groth16_h_combine_launch(ctx, a, b, c, log_n);
}

}  // namespace bzk
