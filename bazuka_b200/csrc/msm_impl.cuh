// bazuka_b200 — Pippenger multi-scalar multiplication over BLS12-381 G1 / G2 on sm_90a.
//
// GPU replacement for bellman 0.14.0 `multiexp::multiexp` (un-vendored crate), the eight sums
// h, l, a_inputs, a_aux, b_g1_inputs, b_g1_aux, b_g2_inputs, b_g2_aux of `create_proof`
// (reference call sites /root/reference/src/mpn/circuits/test.rs:135,175,215 and every gadget test).
// The result is the same group element bellman computes; the algorithm is re-designed for the GPU:
//
//   1. digits     signed-digit (Booth) recoding of every scalar with window c: W = ceil(256/c)
//                 digits in [-2^(c-1), 2^(c-1)], halving the bucket count.  Scalars arrive as
//                 Montgomery images and are converted in-register.  Histogram by (window, |digit|)
//                 with global REDs.                        [bellman: unsigned windows, c = ceil(ln n)]
//   2. scan       exclusive prefix sum of the W * 2^(c-1) counters -> bucket offsets.
//   3. scatter    counting sort: entry = base index | sign bit, grouped by (window, bucket).
//   4. accumulate the sorted entry list is cut into equal chunks, one per thread, INDEPENDENT of
//                 bucket boundaries, so the work per thread is identical whatever the scalar
//                 distribution (witness vectors are full of 0/1 and small values; bellman special-
//                 cases them, here they are just long runs).  A thread walks its chunk, gathers the
//                 96-byte packed affine base with 6 LDG.128, mixed-adds into an XYZZ accumulator
//                 and flushes at bucket boundaries: runs wholly inside the chunk go straight to the
//                 bucket array, the (at most two) runs cut by a chunk edge go to a side list.
//   5. fixup      side-list runs of the same bucket are folded and stored.
//   6. reduce     per window sum_b (b+1) * B_b: slices of buckets -> running-sum trick per thread
//                 (+ [slice offset] * slice-sum), then a shared-memory tree per window.
//   7. combine    the W window sums (W * 192 B) go to the host, which does the Horner chain of
//                 c*(W-1) doublings and the affine conversion: 255 dependent doublings are a serial
//                 chain no GPU thread runs faster than a CPU core, and it is < 2 % of the job.
//
// Algorithmic traffic: 128 B per term (32 B scalar + 96 B base) for G1, 224 B for G2; the kernel is
// integer-ALU bound (≈ W * 10 Fp products per term), see DESIGN.md for both rooflines.
#pragma once
#include "common.cuh"
#include "msm_affine.cuh"
#include <algorithm>
#include <cstdlib>
#ifndef BZK_ACC_MIN_BLOCKS_G1
#define BZK_ACC_MIN_BLOCKS_G1 4
#endif

namespace bzk {

// ---------------------------------------------------------------------------------------------
// plan
// ---------------------------------------------------------------------------------------------

// cost of a plan in "mixed additions": n*W bucket insertions + kReduceCost per bucket for the reduction
// (two full additions per bucket in the running sums, the latency-bound tree and the extra digit /
// scatter work of more windows).  kReduceCost and kNarrowTopCost were calibrated at 2^20 on the previous
// target GPU and are carried over unchanged: they have not been re-tuned on the H100.
// A narrow TOP window is expensive: scalars are < 2^255, so window W-1 holds only 255 - c*(W-1) meaningful bits; when
// that is a handful (c = 19: 8 bits, c = 18 or 21: 3), a sixteenth of all entries lands in a few hundred buckets — the
// histogram's REDs and the scatter's ATOMs serialise on those addresses and the runs go through the long-run path
// — about 1.5 additions per term.
constexpr double kReduceCost = 6.0, kNarrowTopCost = 1.5;
static double plan_cost(size_t n, uint32_t c, uint32_t T) {
    const uint32_t W = (256 + c - 1) / c;
    const uint32_t Te = T < W ? T : W, G = (W + Te - 1) / Te;
    const int top_bits = 255 - (int)(c * (W - 1));
    const double narrow = (W > 1 && top_bits < 10 && n >= 4096) ? kNarrowTopCost * (double)n : 0.0;
    return (double)n * W + kReduceCost * G * (double)(1u << (c - 1)) + narrow;
}
// window plan for n terms over a base table of T levels built for window c_tab (0 = free choice)
static MsmPlan make_plan(size_t n, uint32_t c_tab = 0, uint32_t T = 1, uint32_t G_tab = 0) {
    uint32_t best_c = c_tab;
    if (!c_tab) {
        double best = 1e300;
        for (uint32_t c = 2; c <= 18; c++) {
            double cost = plan_cost(n, c, 1);
            if (cost < best) { best = cost; best_c = c; }
        }
        T = 1;
    }
    MsmPlan p;
    p.c = best_c;
    // W*c >= 256 guarantees the recoding carry never leaves the top window (scalars < 2^255)
    p.W = (256 + p.c - 1) / p.c;
    p.T = T < p.W ? T : p.W;
    p.G = c_tab ? G_tab : p.W;
    p.NB = 1u << (p.c - 1);
    p.TB = p.G * p.NB;
    return p;
}
// window size and level count of the table to build for an n-point resident vector; ctx_c != 0 forces the window
// (bzk_ctx_set_msm_table_window), else the BZK_TABLE_C environment value does, else the cost model picks it
static void choose_table(size_t n, uint32_t max_levels, uint32_t ctx_c, uint32_t *c_out, uint32_t *T_out, uint32_t *G_out) {
    double best = 1e300;
    uint32_t bc = 16, bT = 1;
    static const uint32_t env_c = std::getenv("BZK_TABLE_C") ? (uint32_t)atoi(std::getenv("BZK_TABLE_C")) : 0;  // tuning aid
    const uint32_t force_c = ctx_c ? ctx_c : env_c;
    for (uint32_t c = 8; c <= 23; c++) {
        if (force_c && c != force_c) continue;
        const uint32_t W = (256 + c - 1) / c;
        const uint32_t T = max_levels < W ? max_levels : W;
        if ((double)n * T >= 1073741824.0) continue;  // table index must fit 30 bits
        double cost = plan_cost(n, c, T);
        if (cost < best) { best = cost; bc = c; bT = T; }
    }
    const uint32_t W = (256 + bc - 1) / bc;
    *c_out = bc;
    *G_out = (W + bT - 1) / bT;
    *T_out = (W + *G_out - 1) / *G_out;  // levels really needed for that many groups
}

// signed digit w of canonical scalar k (8 LE 32-bit limbs): value in [-2^(c-1), 2^(c-1)]
__host__ __device__ __forceinline__ int32_t signed_digit(const uint32_t k[8], uint32_t c, uint32_t w, uint32_t &carry) {
    const uint32_t pos = w * c;
    uint32_t raw = 0;
    if (pos < 256) {
        const uint32_t limb = pos >> 5, sh = pos & 31;
        uint64_t two = k[limb];
        if (limb + 1 < 8) two |= (uint64_t)k[limb + 1] << 32;
        raw = (uint32_t)(two >> sh) & ((1u << c) - 1);
    }
    raw += carry;
    if (raw > (1u << (c - 1))) {
        carry = 1;
        return (int32_t)raw - (int32_t)(1u << c);
    }
    carry = 0;
    return (int32_t)raw;
}

// ---------------------------------------------------------------------------------------------
// 1. digits + histogram          3. scatter
// ---------------------------------------------------------------------------------------------
template <bool SCATTER>
__global__ void __launch_bounds__(256) k_digits(const Fr *__restrict__ scalars, size_t n, uint32_t c, uint32_t W, uint32_t NB, uint32_t G,
                                                uint32_t n_tab, uint32_t off, uint32_t *__restrict__ counts_or_cursor, uint32_t *__restrict__ sorted) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Fr k = load_vec(scalars + i).from_mont();
    uint32_t carry = 0;
    for (uint32_t w = 0; w < W; w++) {
        int32_t d = signed_digit(k.l, c, w, carry);
        if (d == 0) continue;
        uint32_t neg = d < 0;
        uint32_t b = (uint32_t)(neg ? -d : d) - 1;
        // window w = t*G + g: bucket group g, point [2^(c*G*t)] P_i from level t of the table
        const uint32_t t = w / G, g = w - t * G;
        uint32_t slot = g * NB + b;
        if (SCATTER) {
            uint32_t pos = atomicAdd(&counts_or_cursor[slot], 1u);
            sorted[pos] = (t * n_tab + off + (uint32_t)i) | (neg << 31);
        } else {
            atomicAdd(&counts_or_cursor[slot], 1u);
        }
    }
}

// ---------------------------------------------------------------------------------------------
// 2. exclusive scan of uint32 counters (three small kernels)
// ---------------------------------------------------------------------------------------------
constexpr int kScanBlock = 256, kScanItems = 4, kScanTile = kScanBlock * kScanItems;

static __global__ void __launch_bounds__(kScanBlock) k_scan_tile_sums(const uint32_t *__restrict__ in, uint32_t count, uint32_t *__restrict__ tile_sums) {
    __shared__ uint32_t sh[kScanBlock / 32];
    uint32_t base = blockIdx.x * kScanTile + threadIdx.x * kScanItems;
    uint32_t s = 0;
#pragma unroll
    for (int k = 0; k < kScanItems; k++)
        if (base + k < count) s += in[base + k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t t = 0;
        for (int k = 0; k < kScanBlock / 32; k++) t += sh[k];
        tile_sums[blockIdx.x] = t;
    }
}
// single block: exclusive scan of tile sums in place; writes grand total to tile_sums[ntiles]
static __global__ void __launch_bounds__(1024) k_scan_tiles(uint32_t *__restrict__ tile_sums, uint32_t ntiles) {
    __shared__ uint32_t sh[1024];
    __shared__ uint32_t carry;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (uint32_t base = 0; base < ntiles; base += 1024) {
        uint32_t idx = base + threadIdx.x;
        uint32_t v = idx < ntiles ? tile_sums[idx] : 0;
        sh[threadIdx.x] = v;
        __syncthreads();
        for (uint32_t o = 1; o < 1024; o <<= 1) {
            uint32_t t = threadIdx.x >= o ? sh[threadIdx.x - o] : 0;
            __syncthreads();
            sh[threadIdx.x] += t;
            __syncthreads();
        }
        uint32_t incl = sh[threadIdx.x];
        if (idx < ntiles) tile_sums[idx] = carry + incl - v;
        __syncthreads();
        if (threadIdx.x == 1023) carry += incl;
        __syncthreads();
    }
    if (threadIdx.x == 0) tile_sums[ntiles] = carry;
}
// offsets[i] = exclusive prefix; offsets[count] = total; cursor = copy of offsets
static __global__ void __launch_bounds__(kScanBlock) k_scan_apply(const uint32_t *__restrict__ in, uint32_t count, const uint32_t *__restrict__ tile_sums,
                                                           uint32_t ntiles, uint32_t *__restrict__ offsets, uint32_t *__restrict__ cursor) {
    __shared__ uint32_t sh[kScanBlock];
    uint32_t base = blockIdx.x * kScanTile + threadIdx.x * kScanItems;
    uint32_t v[kScanItems], s = 0;
#pragma unroll
    for (int k = 0; k < kScanItems; k++) { v[k] = (base + k < count) ? in[base + k] : 0; s += v[k]; }
    sh[threadIdx.x] = s;
    __syncthreads();
    for (uint32_t o = 1; o < kScanBlock; o <<= 1) {
        uint32_t t = threadIdx.x >= o ? sh[threadIdx.x - o] : 0;
        __syncthreads();
        sh[threadIdx.x] += t;
        __syncthreads();
    }
    uint32_t run = tile_sums[blockIdx.x] + sh[threadIdx.x] - s;
#pragma unroll
    for (int k = 0; k < kScanItems; k++) {
        if (base + k < count) { offsets[base + k] = run; cursor[base + k] = run; }
        run += v[k];
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) offsets[count] = tile_sums[ntiles];
}

// ---------------------------------------------------------------------------------------------
// 4. accumulate (chunked, bucket-boundary agnostic)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t effective_chunk(uint32_t M, uint32_t threads, uint32_t min_chunk) {
    uint32_t c = (M + threads - 1) / threads;
    return c < min_chunk ? min_chunk : c;
}

// occupancy target of the accumulate kernel: G1 fits 4 CTAs of 128 threads per SM when capped at 128
// registers (4 warps per sub-partition keep the integer-multiply pipe fed through the carry chains)
template <class F> struct AccBlocks { static constexpr int value = 1; };
template <> struct AccBlocks<Fp> { static constexpr int value = BZK_ACC_MIN_BLOCKS_G1; };

template <class F>
__global__ void __launch_bounds__(128, AccBlocks<F>::value) k_accumulate(const Affine<F> *__restrict__ bases, const Affine<F> *__restrict__ scr, const uint32_t *__restrict__ sorted,
                                                    const uint32_t *__restrict__ offsets, uint32_t TB, uint32_t min_chunk,
                                                    Xyzz<F> *__restrict__ buckets, Xyzz<F> *__restrict__ part_pts,
                                                    int32_t *__restrict__ part_bucket) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t M = offsets[TB];
    // the launch is sized for "every digit non-zero"; spread the entries that really exist over all
    // launched threads (witness vectors are full of zeros: M is often half of n*W)
    const uint32_t chunk = effective_chunk(M, gridDim.x * blockDim.x, min_chunk);
    const uint64_t start64 = (uint64_t)t * chunk;
    part_bucket[2 * t] = -1;
    part_bucket[2 * t + 1] = -1;
    if (start64 >= M) return;
    const uint32_t start = (uint32_t)start64;
    const uint32_t end = (uint32_t)(start64 + chunk < M ? start64 + chunk : M);
    // largest b with offsets[b] <= start
    uint32_t lo = 0, hi = TB;  // invariant: offsets[lo] <= start < offsets[hi] (offsets[TB] = M > start)
    while (hi - lo > 1) {
        uint32_t mid = (lo + hi) >> 1;
        if (offsets[mid] <= start) lo = mid; else hi = mid;
    }
    uint32_t b = lo;
    uint32_t bend = offsets[b + 1];
    while (bend <= start) { b++; bend = offsets[b + 1]; }  // skip empty buckets sharing the offset
    uint32_t run_start = start;
    bool run_from_bucket_start = (offsets[b] == start);
    Xyzz<F> acc = Xyzz<F>::inf();
    for (uint32_t pos = start; pos < end; pos++) {
        if (pos == bend) {
            // bucket b ended exactly here: flush
            if (run_from_bucket_start) {
                store_vec(buckets + b, acc);
            } else {
                const uint32_t slot = 2 * t + (run_start == start ? 0 : 1);
                store_vec(part_pts + slot, acc);
                part_bucket[slot] = (int32_t)b;
            }
            acc = Xyzz<F>::inf();
            do { b++; bend = offsets[b + 1]; } while (bend <= pos);
            run_start = pos;
            run_from_bucket_start = true;
        }
        const uint32_t e = sorted[pos];
        // scr != nullptr: the list went through affine rounds and bit 30 selects the pool of intermediate sums
        Affine<F> p;
        if (scr) {
            p = load_ref(bases, scr, e);
        } else {
            p = load_vec(bases + (e & 0x7fffffffu));
            if (e >> 31) p.y = p.y.neg();
        }
        acc.madd(p);
    }
    // final run: complete only if it started at the bucket start and the bucket ends at `end`
    if (run_from_bucket_start && bend == end) {
        store_vec(buckets + b, acc);
    } else {
        const uint32_t slot = 2 * t + (run_start == start ? 0 : 1);
        store_vec(part_pts + slot, acc);
        part_bucket[slot] = (int32_t)b;
    }
}

// 5. fold the side list.  The first slot of each bucket's run of partials owns the run: short runs
// (the common case: a bucket cut by one or two chunk edges) are summed by that thread; long runs
// — a bucket that swallows thousands of chunks, e.g. digit 1 of window 0 when a third of a Groth16
// witness is boolean — are queued for k_fixup_long, where a whole CTA sums the run with a
// shared-memory tree instead of one thread walking it serially.
constexpr uint32_t kLongRun = 6;        // partials; longer runs go to the CTA-wide path
constexpr uint32_t kLongQueueCap = 4096;
struct LongRun { uint32_t first, last; int32_t bucket; uint32_t pad; };

template <class F>
__global__ void __launch_bounds__(128) k_fixup(const Xyzz<F> *__restrict__ part_pts, const int32_t *__restrict__ part_bucket,
                                               uint32_t nslots_max, const uint32_t *__restrict__ offsets, uint32_t TB, uint32_t acc_threads, uint32_t min_chunk,
                                               Xyzz<F> *__restrict__ buckets,
                                               LongRun *__restrict__ queue, uint32_t *__restrict__ queue_len) {
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    // only the chunks that actually hold entries have slots (the launch is sized for the worst case
    // "every digit non-zero"; witness vectors are far sparser)
    const uint32_t M = offsets[TB];
    const uint32_t chunk = effective_chunk(M, acc_threads, min_chunk);
    uint32_t nslots = 2 * ((M + chunk - 1) / chunk);
    if (nslots > nslots_max) nslots = nslots_max;
    if (e >= nslots) return;
    const int32_t b = part_bucket[e];
    if (b < 0) return;
    for (uint32_t q = e; q-- > 0;) {
        int32_t pb = part_bucket[q];
        if (pb < 0) continue;
        if (pb == b) return;  // not the head of the run
        break;
    }
    // measure the run (slot indices only)
    uint32_t last = e, count = 1;
    for (uint32_t q = e + 1; q < nslots; q++) {
        int32_t nb = part_bucket[q];
        if (nb < 0) continue;
        if (nb != b) break;
        last = q;
        count++;
    }
    if (count > kLongRun) {
        uint32_t at = atomicAdd(queue_len, 1u);
        if (at < kLongQueueCap) {
            queue[at] = LongRun{e, last, b, 0};
            return;
        }
        // queue full (cannot happen with <= kLongQueueCap long runs; fall through to the serial sum)
    }
    Xyzz<F> acc = load_vec(part_pts + e);
    for (uint32_t q = e + 1; q <= last; q++)
        if (part_bucket[q] == b) acc.add(load_vec(part_pts + q));
    store_vec(buckets + b, acc);
}

// one CTA per queued long run (grid-stride over the queue)
template <class F>
__global__ void __launch_bounds__(256) k_fixup_long(const Xyzz<F> *__restrict__ part_pts, const int32_t *__restrict__ part_bucket,
                                                    Xyzz<F> *__restrict__ buckets, const LongRun *__restrict__ queue,
                                                    const uint32_t *__restrict__ queue_len) {
    extern __shared__ uint4 smem_raw[];
    Xyzz<F> *sh = (Xyzz<F> *)smem_raw;
    uint32_t nq = *queue_len;
    if (nq > kLongQueueCap) nq = kLongQueueCap;
    for (uint32_t r = blockIdx.x; r < nq; r += gridDim.x) {
        const LongRun run = queue[r];
        Xyzz<F> acc = Xyzz<F>::inf();
        for (uint32_t q = run.first + threadIdx.x; q <= run.last; q += blockDim.x)
            if (part_bucket[q] == run.bucket) acc.add(load_vec(part_pts + q));
        sh[threadIdx.x] = acc;
        __syncthreads();
        for (uint32_t o = blockDim.x / 2; o > 0; o >>= 1) {
            if (threadIdx.x < o) {
                Xyzz<F> a = sh[threadIdx.x];
                a.add(sh[threadIdx.x + o]);
                sh[threadIdx.x] = a;
            }
            __syncthreads();
        }
        if (threadIdx.x == 0) store_vec(buckets + run.bucket, sh[0]);
        __syncthreads();
    }
}

// the chunks after the first of a streamed sum accumulate into a cleared pass array (so k_accumulate / k_fixup run
// unchanged); this adds each bucket the chunk touched into the sum's buckets.  One thread per bucket, no atomics.
template <class F>
__global__ void __launch_bounds__(128) k_bucket_fold(Xyzz<F> *__restrict__ buckets, const Xyzz<F> *__restrict__ pass, uint32_t TB) {
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= TB) return;
    const Xyzz<F> v = load_vec(pass + b);
    if (v.is_inf()) return;
    Xyzz<F> t = load_vec(buckets + b);
    t.add(v);
    store_vec(buckets + b, t);
}

// ---------------------------------------------------------------------------------------------
// 6. bucket reduction: per window  sum_b (b+1) * B_b
// ---------------------------------------------------------------------------------------------
// A group's sum is  sum_b (b+1) B_b.  The buckets are cut into slices of `slice` consecutive buckets; slice s
// (buckets lo = s*slice ...) contributes  acc_s + lo * run_s  with  run_s = sum B,  acc_s = sum (k+1) B_{lo+k}.
// The dependent chain per thread is just the 2*slice running-sum additions: the [lo] multiple is NOT formed per
// slice (a ~30-addition double-and-add that used to cost as much as the running sums) but through the bits of s,
//     sum_s lo_s run_s = slice * sum_j 2^j T_j ,   T_j = sum over the slices whose index has bit j set of run_s ,
// i.e. 1 + nbits independent tree sums per group (k_slice_combine, k_partial_sum) and a ~2 nbits-operation Horner
// fold on the host.
template <class F>
__global__ void __launch_bounds__(128) k_bucket_slices(const Xyzz<F> *__restrict__ buckets, uint32_t NB, uint32_t slice, uint32_t nslices_total,
                                                       Xyzz<F> *__restrict__ acc_out, Xyzz<F> *__restrict__ run_out) {
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= nslices_total) return;
    const uint32_t per_win = (NB + slice - 1) / slice;  // the last slice of a group may be short
    const uint32_t w = g / per_win, sidx = g % per_win;
    const uint32_t lo = sidx * slice;
    const uint32_t len = (lo + slice <= NB) ? slice : NB - lo;
    const Xyzz<F> *B = buckets + (size_t)w * NB;
    Xyzz<F> run = Xyzz<F>::inf(), acc = Xyzz<F>::inf();
    for (uint32_t k = len; k-- > 0;) {
        run.add(load_vec(B + lo + k));
        acc.add(run);
    }
    store_vec(acc_out + g, acc);
    store_vec(run_out + g, run);
}

// grid (parts, 1 + nbits, G): CTA (p, j, g) tree-sums 256 consecutive slices of group g — acc_s for j = 0, run_s of
// the slices with bit j-1 set for j >= 1 — into partial[(g*(1+nbits) + j) * parts + p]
// (a dependent addition costs ~9 us whatever the occupancy, so the shape is: kCombineSerial serial additions per
// thread, then a 6-level shared-memory tree over 64 threads; the ~600 two-warp CTAs of a 2^19-bucket group are all
// resident at once)
constexpr uint32_t kCombineThreads = 64, kCombineSerial = 8, kCombineSpan = kCombineThreads * kCombineSerial;
template <class F>
__global__ void __launch_bounds__(kCombineThreads) k_slice_combine(const Xyzz<F> *__restrict__ acc_in, const Xyzz<F> *__restrict__ run_in, uint32_t per_win,
                                                                  Xyzz<F> *__restrict__ partial) {
    extern __shared__ uint4 smem_raw[];
    Xyzz<F> *sh = (Xyzz<F> *)smem_raw;
    const uint32_t j = blockIdx.y, g = blockIdx.z;
    Xyzz<F> v = Xyzz<F>::inf();
    for (uint32_t k = 0; k < kCombineSerial; k++) {
        const uint32_t s = blockIdx.x * kCombineSpan + k * kCombineThreads + threadIdx.x;
        if (s >= per_win) break;
        if (j == 0) v.add(load_vec(acc_in + (size_t)g * per_win + s));
        else if ((s >> (j - 1)) & 1) v.add(load_vec(run_in + (size_t)g * per_win + s));
    }
    sh[threadIdx.x] = v;
    __syncthreads();
    for (uint32_t o = kCombineThreads / 2; o > 0; o >>= 1) {
        if (threadIdx.x < o) {
            Xyzz<F> a = sh[threadIdx.x];
            a.add(sh[threadIdx.x + o]);
            sh[threadIdx.x] = a;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) store_vec(partial + ((size_t)(g * gridDim.y + j)) * gridDim.x + blockIdx.x, sh[0]);
}
// one CTA per (j, g): sum of its `parts` partials
template <class F>
__global__ void __launch_bounds__(128) k_partial_sum(const Xyzz<F> *__restrict__ partial, uint32_t parts, Xyzz<F> *__restrict__ win_out) {
    extern __shared__ uint4 smem_raw[];
    Xyzz<F> *sh = (Xyzz<F> *)smem_raw;
    const size_t row = blockIdx.x;
    Xyzz<F> acc = Xyzz<F>::inf();
    for (uint32_t k = threadIdx.x; k < parts; k += blockDim.x) acc.add(load_vec(partial + row * parts + k));
    sh[threadIdx.x] = acc;
    __syncthreads();
    for (uint32_t o = blockDim.x / 2; o > 0; o >>= 1) {
        if (threadIdx.x < o) {
            Xyzz<F> a = sh[threadIdx.x];
            a.add(sh[threadIdx.x + o]);
            sh[threadIdx.x] = a;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) store_vec(win_out + row, sh[0]);
}

// ---------------------------------------------------------------------------------------------
// wire image <-> packed, synthetic inputs
// ---------------------------------------------------------------------------------------------
static __global__ void __launch_bounds__(256) k_pack_g1(const uint8_t *__restrict__ images, size_t n, G1Affine *__restrict__ out, uint32_t *bad) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    G1Affine p = load_g1_image(images + i * 104);
    if (bad && !p.is_inf() && !on_curve(p)) atomicAdd(bad, 1u);
    store_vec(out + i, p);
}
static __global__ void __launch_bounds__(128) k_pack_g2(const uint8_t *__restrict__ images, size_t n, G2Affine *__restrict__ out, uint32_t *bad) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    G2Affine p = load_g2_image(images + i * 200);
    if (bad && !p.is_inf() && !on_curve(p)) atomicAdd(bad, 1u);
    store_vec(out + i, p);
}

static __global__ void __launch_bounds__(128) k_random_g1(uint64_t seed, size_t n, G1Affine gen, uint8_t *__restrict__ out) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Fr k = splitmix_fr_canonical(seed, i);
    store_g1_image(out + i * 104, scalar_mul(gen, k.l).to_affine());
}
static __global__ void __launch_bounds__(64) k_random_g2(uint64_t seed, size_t n, G2Affine gen, uint8_t *__restrict__ out) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Fr k = splitmix_fr_canonical(seed, i);
    store_g2_image(out + i * 200, scalar_mul(gen, k.l).to_affine());
}
static __global__ void __launch_bounds__(256) k_random_fr(uint64_t seed, size_t n, Fr *__restrict__ out) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    store_vec(out + i, splitmix_fr_canonical(seed, i).to_mont());
}

// the wire image type of an Affine<F> (converted with from_wire / to_wire, common.cuh)
template <class F> struct Wire;
template <> struct Wire<Fp> { typedef bzk_g1_affine image; };
template <> struct Wire<Fp2> { typedef bzk_g2_affine image; };

// ---------------------------------------------------------------------------------------------
// fixed-base table: level t of point i = [2^(bits*t)] P_i, affine.  One thread per base walks the doubling
// chain in XYZZ, keeps the T-1 level points in local memory and converts them with ONE inversion
// (Montgomery's trick over q_t = ZZ_t * ZZZ_t).  Run once per resident vector (a proving-key column).
// ---------------------------------------------------------------------------------------------
constexpr uint32_t kMaxLevels = 16;
template <class F>
__global__ void __launch_bounds__(128) k_precompute(Affine<F> *__restrict__ tab, size_t n, uint32_t T, uint32_t bits) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const Affine<F> P = load_vec(tab + i);
    Xyzz<F> L[kMaxLevels - 1];
    F pre[kMaxLevels - 1];
    Xyzz<F> acc = Xyzz<F>::from_affine(P);
    F run = F::one();
    for (uint32_t t = 1; t < T; t++) {
        for (uint32_t k = 0; k < bits; k++) acc = acc.dbl();
        L[t - 1] = acc;
        pre[t - 1] = run;
        if (!acc.is_inf()) run = run * (acc.ZZ * acc.ZZZ);
    }
    F inv = run.inv();
    for (uint32_t t = T - 1; t >= 1; t--) {
        const Xyzz<F> &Q = L[t - 1];
        Affine<F> out = Affine<F>::inf();
        if (!Q.is_inf()) {
            const F qi = inv * pre[t - 1];  // 1 / (ZZ * ZZZ)
            inv = inv * (Q.ZZ * Q.ZZZ);
            out.x = Q.X * Q.ZZZ * qi;
            out.y = Q.Y * Q.ZZ * qi;
        }
        store_vec(tab + (size_t)t * n + i, out);
    }
}

// grow a resident vector into a table of up to max_levels levels (the bases stay level 0)
template <class F>
static int32_t bases_precompute(bzk_ctx *ctx, Affine<F> **d, size_t n, uint32_t max_levels, uint32_t *c_out, uint32_t *T_out, uint32_t *G_out) {
    if (max_levels > kMaxLevels) max_levels = kMaxLevels;
    uint32_t c = 0, T = 1, G = 0;
    if (n == 0 || max_levels <= 1) { *c_out = 0; *T_out = 1; *G_out = 0; return BZK_OK; }
    choose_table(n, max_levels, ctx->table_c, &c, &T, &G);
    if (T <= 1) { *c_out = 0; *T_out = 1; *G_out = 0; return BZK_OK; }
    Affine<F> *tab = nullptr;
    cudaError_t e = cudaMalloc(&tab, (size_t)T * n * sizeof(Affine<F>));
    if (e != cudaSuccess) return set_cuda_err(ctx, e, "cudaMalloc(base table)", __FILE__, __LINE__);
    BZK_CUDA(ctx, cudaMemcpyAsync(tab, *d, n * sizeof(Affine<F>), cudaMemcpyDeviceToDevice, ctx->stream));
    k_precompute<F><<<div_up(n, 128), 128, 0, ctx->stream>>>(tab, n, T, c * G);
    BZK_LAUNCHED(ctx);
    BZK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    cudaFree(*d);
    *d = tab;
    *c_out = c; *T_out = T; *G_out = G;
    return BZK_OK;
}

// ---------------------------------------------------------------------------------------------
// host driver
// ---------------------------------------------------------------------------------------------
// Points per chunk buffer of a streamed sum unless bzk_ctx_set_msm_stream_chunk says otherwise: 384 MB per buffer for G1 and
// for G2, two buffers per sum.  A chunk is long enough that its digit / scan / reduction overheads stay small next to its
// accumulation, and its copy (~8 ms at 50 GB/s) hides behind the accumulation of the one before.
template <class F>
static size_t stream_chunk_points(const bzk_ctx *ctx) {
    if (ctx->stream_chunk) return (size_t)ctx->stream_chunk;
    return sizeof(F) == sizeof(Fp) ? ((size_t)1 << 22) : ((size_t)1 << 21);
}

// the copy stream, events and at least `bytes` of chunk buffers of one pipe (grown only)
static int32_t ensure_pipe(bzk_ctx *ctx, StreamPipe *p, cudaStream_t st, size_t bytes) {
    if (!p->copy) BZK_CUDA(ctx, cudaStreamCreateWithFlags(&p->copy, cudaStreamNonBlocking));
    for (int b = 0; b < 2; b++) {
        if (!p->ready[b]) BZK_CUDA(ctx, cudaEventCreateWithFlags(&p->ready[b], cudaEventDisableTiming));
        if (!p->freed[b]) BZK_CUDA(ctx, cudaEventCreateWithFlags(&p->freed[b], cudaEventDisableTiming));
    }
    if (p->bytes >= bytes) return BZK_OK;
    if (p->buf) {
        // the buffers' last users: copies on the pipe's stream, kernels on the sum's stream
        BZK_CUDA(ctx, cudaStreamSynchronize(p->copy));
        BZK_CUDA(ctx, cudaStreamSynchronize(st));
        BZK_CUDA(ctx, cudaFree(p->buf));
        p->buf = nullptr;
        p->bytes = 0;
    }
    BZK_CUDA(ctx, cudaMalloc(&p->buf, bytes));
    p->bytes = bytes;
    return BZK_OK;
}

template <class F>
// Enqueue one MSM on stream `st` with its own workspace arena; the W window sums are copied into
// `h_win` (host, ideally pinned; >= 64 entries) by the last operation on the stream.  Nothing here
// synchronises: several MSMs can be in flight on different streams (the Groth16 driver runs its
// five sums concurrently), and msm_host_finish folds the window sums once the stream is done.
// `d_long_len` (optional) receives the device address of the long-run queue length k_fixup counts.
//
// A host-resident vector (bases.host) is streamed through `pipe`: the sum runs in passes over chunks of its terms.  Each
// chunk's points are copied on the pipe's stream into one of two device buffers while the previous chunk is accumulated;
// the chunk's digits, scan and scatter index into that buffer.  The first chunk's accumulate / fixup fill the bucket array;
// each later chunk's fill a cleared pass array that k_bucket_fold then adds into it.  One bucket reduction ends the sum,
// as for a resident vector.  The first copies wait for nothing on `st`, so they overlap whatever `st` runs before the sum.
// Streamed sums use no batched-affine rounds and record no stage marks.  `stream_out` (optional): chunks, chunk points,
// bytes copied host->device, 1 if streamed.
static int32_t msm_enqueue(bzk_ctx *ctx, cudaStream_t st, void **ws, size_t *ws_bytes, StreamPipe *pipe, bool timed, const BasesRef<F> &bases,
                           const Fr *d_scalars, size_t n, Xyzz<F> *h_win, MsmPlan *plan_out, uint32_t **d_long_len = nullptr,
                           uint64_t *stream_out = nullptr) {
    if (stream_out) memset(stream_out, 0, 4 * sizeof(uint64_t));
    if (n == 0) { plan_out->W = 0; return BZK_OK; }
    if (n >= ((size_t)1 << 31) || bases.off + n > bases.n_tab) return BZK_ERR_BAD_ARG;
    const bool streamed = bases.host;
    if (streamed && (bases.T != 1 || !pipe)) return BZK_ERR_BAD_ARG;
    const MsmPlan pl = make_plan(n, bases.c, bases.T, bases.G);
    if ((double)bases.n_tab * pl.T >= 2147483648.0) return BZK_ERR_BAD_ARG;
    const Affine<F> *d_bases = bases.tab;
    *plan_out = pl;
    if ((double)n * pl.W >= 4294967295.0) return BZK_ERR_BAD_ARG;
    // terms per pass: all of them, or one chunk of a streamed sum
    size_t cn = n;
    if (streamed) cn = std::min(n, stream_chunk_points<F>(ctx));
    const size_t passes = (n + cn - 1) / cn;
    const uint64_t max_entries = (uint64_t)cn * pl.W;

    // thread geometry of the accumulate kernel
    const uint32_t acc_threads_target = (uint32_t)ctx->sm_count * 128 * (sizeof(F) == sizeof(Fp) ? BZK_ACC_MIN_BLOCKS_G1 : 2);
    uint32_t chunk = (uint32_t)((max_entries + acc_threads_target - 1) / acc_threads_target);
    if (chunk < 16) chunk = 16;
    const uint32_t acc_threads = (uint32_t)((max_entries + chunk - 1) / chunk);
    const uint32_t acc_blocks = div_up(acc_threads, 128);
    const uint32_t nslots = 2 * acc_blocks * 128;

    // batched-affine rounds before the XYZZ accumulation (msm_affine.cuh): worth it when buckets hold several entries
    // and the point references fit 30 bits; R rounds leave 2^-R of the additions to the XYZZ kernel
    // k_round_fwd is load-latency bound and each round ends in a single-thread inversion chain, so for G1 the rounds
    // made the whole sum slower; the default for G1 is 0 rounds; the knobs stay for G2 and for tuning.
    static const int env_g1 = std::getenv("BZK_AFFINE_ROUNDS") ? atoi(std::getenv("BZK_AFFINE_ROUNDS")) : 0;
    static const int env_g2 = std::getenv("BZK_AFFINE_ROUNDS_G2") ? atoi(std::getenv("BZK_AFFINE_ROUNDS_G2")) : 0;
    const int ctx_rounds = ctx->affine_rounds[sizeof(F) == sizeof(Fp) ? 0 : 1];
    const int env_rounds = ctx_rounds >= 0 ? ctx_rounds : (sizeof(F) == sizeof(Fp) ? env_g1 : env_g2);
    uint32_t R = 0;
    if (!streamed && env_rounds > 0 && (double)bases.n_tab * pl.T < 1073741824.0 && max_entries >= 8ull * pl.TB) {
        R = (uint32_t)env_rounds;
        while (R && (max_entries >> R) < 2ull * pl.TB) R--;   // stop when buckets are down to a couple of entries
    }
    if (R > 6) R = 6;
    uint64_t cap[8];
    cap[0] = max_entries;
    uint64_t scr_points = 0;
    for (uint32_t r = 0; r < R; r++) { cap[r + 1] = (cap[r] + pl.TB) / 2 + 1; scr_points += cap[r + 1]; }
    if (scr_points >= (1ull << 30)) { R = 0; scr_points = 0; }
    const uint32_t rnd_blocks = (uint32_t)ctx->sm_count * (sizeof(F) == sizeof(Fp) ? 4 : 2);
    const uint32_t rnd_threads = rnd_blocks * kRoundThreads;
    uint32_t mid_threads = 32;
    while (mid_threads < rnd_blocks) mid_threads <<= 1;

    // slice length trades the serial running-sum (2*slice adds) against the [offset]*sum
    // double-and-add (~log2(NB/slice) doublings): short slices keep every SM busy
    // Slice length: the reduction is bound by the integer-multiply pipe, and its total work is
    // TB * (2 + smul/slice) additions (smul = the ~19-op [slice offset] double-and-add), so LONGER
    // slices mean less work; one warp per SM sub-partition already saturates that pipe, so the
    // kernel runs ONE 128-thread CTA per SM (measured at 2^20: 1 CTA/SM 1.43 ms, 3 CTAs/SM 1.91 ms).
    static const int red_blocks_per_sm = std::getenv("BZK_RED_BLOCKS") ? atoi(std::getenv("BZK_RED_BLOCKS")) : 1;
    const uint32_t red_capacity = (uint32_t)ctx->sm_count * (uint32_t)(red_blocks_per_sm > 0 ? red_blocks_per_sm : 1) * 128;
    uint32_t slice = (uint32_t)(((uint64_t)pl.TB + red_capacity - 1) / red_capacity);
    if (slice < 4) slice = pl.NB >= 4 ? 4 : pl.NB;
    if (slice > pl.NB) slice = pl.NB;
    const uint32_t per_win = (pl.NB + slice - 1) / slice;
    const uint32_t nslices = per_win * pl.G;
    const uint32_t ntiles = div_up(pl.TB, kScanTile);
    uint32_t nbits = 0;  // bits of the largest slice index
    while (nbits < 32 && ((per_win - 1) >> nbits)) nbits++;
    const uint32_t rows = pl.G * (1 + nbits);      // tree sums per MSM: A and T_0..T_{nbits-1} of every group
    const uint32_t parts = div_up(per_win, kCombineSpan);
    if (rows > kMaxWinPoints) return BZK_ERR_BAD_ARG;
    MsmPlan full = pl;
    full.slice = slice;
    full.nbits = nbits;
    *plan_out = full;

    // workspace
    size_t need = 0;
    {
        Carver cv(nullptr);
        cv.take<uint32_t>(pl.TB + 1); cv.take<uint32_t>(pl.TB + 1); cv.take<uint32_t>(pl.TB + 1);
        cv.take<uint32_t>(ntiles + 1);
        cv.take<uint32_t>(max_entries);
        if (R) {
            cv.take<uint32_t>(cap[1]); cv.take<uint32_t>(cap[1]);
            cv.take<uint32_t>(pl.TB + 2); cv.take<uint32_t>(pl.TB + 2);
            cv.take<Affine<F>>(scr_points);
            cv.take<F>(cap[1]);
            cv.take<F>(rnd_threads); cv.take<F>(rnd_threads);
            cv.take<F>(rnd_blocks); cv.take<F>(rnd_blocks); cv.take<F>(rnd_blocks); cv.take<F>(4);
        }
        cv.take<Xyzz<F>>(pl.TB);
        cv.take<Xyzz<F>>(passes > 1 ? pl.TB : 0);
        cv.take<Xyzz<F>>(nslots); cv.take<int32_t>(nslots);
        cv.take<LongRun>(kLongQueueCap); cv.take<uint32_t>(4);
        cv.take<Xyzz<F>>(nslices); cv.take<Xyzz<F>>(nslices);
        cv.take<Xyzz<F>>((size_t)rows * parts);
        cv.take<Xyzz<F>>(rows);
        need = cv.used();
    }
    BZK_TRY(ensure_ws(ctx, ws, ws_bytes, need));
    Carver cv(*ws);
    uint32_t *counts = cv.take<uint32_t>(pl.TB + 1);
    uint32_t *offsets = cv.take<uint32_t>(pl.TB + 1);
    uint32_t *cursor = cv.take<uint32_t>(pl.TB + 1);
    uint32_t *tile_sums = cv.take<uint32_t>(ntiles + 1);
    uint32_t *sorted = cv.take<uint32_t>(max_entries);
    uint32_t *rlist[2] = {nullptr, nullptr}, *roff[2] = {nullptr, nullptr};
    Affine<F> *scr = nullptr;
    F *rpre = nullptr, *thr_pre = nullptr, *thr_suf = nullptr, *blk_tot = nullptr, *blk_pre = nullptr, *blk_suf = nullptr, *inv_total = nullptr;
    if (R) {
        rlist[0] = cv.take<uint32_t>(cap[1]); rlist[1] = cv.take<uint32_t>(cap[1]);
        roff[0] = cv.take<uint32_t>(pl.TB + 2); roff[1] = cv.take<uint32_t>(pl.TB + 2);
        scr = cv.take<Affine<F>>(scr_points);
        rpre = cv.take<F>(cap[1]);
        thr_pre = cv.take<F>(rnd_threads); thr_suf = cv.take<F>(rnd_threads);
        blk_tot = cv.take<F>(rnd_blocks); blk_pre = cv.take<F>(rnd_blocks); blk_suf = cv.take<F>(rnd_blocks); inv_total = cv.take<F>(4);
    }
    Xyzz<F> *buckets = cv.take<Xyzz<F>>(pl.TB);
    Xyzz<F> *pass_buckets = cv.take<Xyzz<F>>(passes > 1 ? pl.TB : 0);  // a streamed sum's later chunks (k_bucket_fold)
    Xyzz<F> *part_pts = cv.take<Xyzz<F>>(nslots);
    int32_t *part_bucket = cv.take<int32_t>(nslots);
    LongRun *long_queue = cv.take<LongRun>(kLongQueueCap);
    uint32_t *long_len = cv.take<uint32_t>(4);
    if (d_long_len) *d_long_len = long_len;
    Xyzz<F> *slice_acc = cv.take<Xyzz<F>>(nslices), *slice_run = cv.take<Xyzz<F>>(nslices);
    Xyzz<F> *partial = cv.take<Xyzz<F>>((size_t)rows * parts);
    Xyzz<F> *win_out = cv.take<Xyzz<F>>(rows);

    Affine<F> *chunk_buf[2] = {nullptr, nullptr};
    if (streamed) {
        const size_t half = (cn * sizeof(Affine<F>) + 255) & ~(size_t)255;
        BZK_TRY(ensure_pipe(ctx, pipe, st, 2 * half));
        chunk_buf[0] = (Affine<F> *)pipe->buf;
        chunk_buf[1] = (Affine<F> *)((char *)pipe->buf + half);
        if (stream_out) {
            stream_out[0] = passes; stream_out[1] = cn; stream_out[2] = (uint64_t)n * sizeof(Affine<F>); stream_out[3] = 1;
        }
    }

    // stage marks: 0 clear+digits/histogram, 1 scan, 2 scatter, 3 accumulate, 4 fixup,
    //              5 bucket slices, 6 window sums (+ D2H of W points)
    const bool saved_timing = ctx->timing;
    ctx->timing = saved_timing && timed && !streamed;
    timing_begin(ctx);
    BZK_CUDA(ctx, cudaMemsetAsync(buckets, 0, (size_t)pl.TB * sizeof(Xyzz<F>), st));  // all-zero = identity
    const size_t fsmem = 256 * sizeof(Xyzz<F>);
    BZK_CUDA(ctx, cudaFuncSetAttribute(k_fixup_long<F>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fsmem));
    for (size_t pass = 0; pass < passes; pass++) {
        const size_t p0 = pass * cn, pn = std::min(cn, n - p0);
        const Fr *p_scalars = d_scalars + p0;
        // a streamed chunk's entries index its buffer (offset 0); T == 1, so n_tab only has to match the launch's bound checks
        const uint32_t p_tab = streamed ? (uint32_t)pn : (uint32_t)bases.n_tab, p_off = streamed ? 0u : (uint32_t)bases.off;
        const int cb = (int)(pass & 1);
        if (streamed) {
            d_bases = chunk_buf[cb];
            BZK_CUDA(ctx, cudaStreamWaitEvent(pipe->copy, pipe->freed[cb], 0));
            BZK_CUDA(ctx, cudaMemcpyAsync(chunk_buf[cb], bases.tab + bases.off + p0, pn * sizeof(Affine<F>), cudaMemcpyHostToDevice, pipe->copy));
            BZK_CUDA(ctx, cudaEventRecord(pipe->ready[cb], pipe->copy));
        }
        BZK_CUDA(ctx, cudaMemsetAsync(counts, 0, (pl.TB + 1) * sizeof(uint32_t), st));
        k_digits<false><<<div_up(pn, 256), 256, 0, st>>>(p_scalars, pn, pl.c, pl.W, pl.NB, pl.G, p_tab, p_off, counts, nullptr);
        BZK_LAUNCHED(ctx);
        timing_mark(ctx);
        k_scan_tile_sums<<<ntiles, kScanBlock, 0, st>>>(counts, pl.TB, tile_sums);
        BZK_LAUNCHED(ctx);
        k_scan_tiles<<<1, 1024, 0, st>>>(tile_sums, ntiles);
        BZK_LAUNCHED(ctx);
        k_scan_apply<<<ntiles, kScanBlock, 0, st>>>(counts, pl.TB, tile_sums, ntiles, offsets, cursor);
        BZK_LAUNCHED(ctx);
        timing_mark(ctx);
        k_digits<true><<<div_up(pn, 256), 256, 0, st>>>(p_scalars, pn, pl.c, pl.W, pl.NB, pl.G, p_tab, p_off, cursor, sorted);
        BZK_LAUNCHED(ctx);
        timing_mark(ctx);
        const uint32_t *acc_list = sorted, *acc_off = offsets;
        if (R) {
            const size_t fsm = 2 * kRoundThreads * sizeof(F), msm_ = 2 * (size_t)mid_threads * sizeof(F);
            BZK_CUDA(ctx, cudaFuncSetAttribute(k_round_mid<F>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)msm_));
            uint32_t scr_base = 0;
            for (uint32_t r = 0; r < R; r++) {
                uint32_t *off1 = roff[r & 1], *list1 = rlist[r & 1];
                k_round_counts<<<div_up(pl.TB + 1, 256), 256, 0, st>>>(acc_off, pl.TB, counts);
                BZK_LAUNCHED(ctx);
                k_scan_tile_sums<<<ntiles, kScanBlock, 0, st>>>(counts, pl.TB, tile_sums);
                BZK_LAUNCHED(ctx);
                k_scan_tiles<<<1, 1024, 0, st>>>(tile_sums, ntiles);
                BZK_LAUNCHED(ctx);
                k_scan_apply<<<ntiles, kScanBlock, 0, st>>>(counts, pl.TB, tile_sums, ntiles, off1, cursor);
                BZK_LAUNCHED(ctx);
                k_round_fwd<F><<<rnd_blocks, kRoundThreads, fsm, st>>>(d_bases, scr, acc_list, acc_off, off1, pl.TB, rpre, thr_pre, thr_suf, blk_tot);
                BZK_LAUNCHED(ctx);
                k_round_mid<F><<<1, mid_threads, msm_, st>>>(blk_tot, rnd_blocks, blk_pre, blk_suf, inv_total);
                BZK_LAUNCHED(ctx);
                k_round_bwd<F><<<rnd_blocks, kRoundThreads, 0, st>>>(d_bases, scr, scr_base, acc_list, acc_off, off1, pl.TB, rpre, thr_pre, thr_suf, blk_pre,
                                                                     blk_suf, inv_total, list1);
                BZK_LAUNCHED(ctx);
                scr_base += (uint32_t)cap[r + 1];
                acc_list = list1;
                acc_off = off1;
            }
        }
        if (streamed) BZK_CUDA(ctx, cudaStreamWaitEvent(st, pipe->ready[cb], 0));
        // the first pass fills the buckets; later ones fill the cleared pass array, folded in below
        Xyzz<F> *target = pass ? pass_buckets : buckets;
        if (pass) BZK_CUDA(ctx, cudaMemsetAsync(pass_buckets, 0, (size_t)pl.TB * sizeof(Xyzz<F>), st));
        k_accumulate<F><<<acc_blocks, 128, 0, st>>>(d_bases, R ? scr : nullptr, acc_list, acc_off, pl.TB, 16u, target, part_pts, part_bucket);
        BZK_LAUNCHED(ctx);
        timing_mark(ctx);
        BZK_CUDA(ctx, cudaMemsetAsync(long_len, 0, 16, st));
        k_fixup<F><<<div_up(nslots, 128), 128, 0, st>>>(part_pts, part_bucket, nslots, acc_off, pl.TB, acc_blocks * 128, 16u, target, long_queue, long_len);
        BZK_LAUNCHED(ctx);
        k_fixup_long<F><<<ctx->sm_count, 256, fsmem, st>>>(part_pts, part_bucket, target, long_queue, long_len);
        BZK_LAUNCHED(ctx);
        if (streamed) BZK_CUDA(ctx, cudaEventRecord(pipe->freed[cb], st));  // the chunk buffer is free for chunk pass + 2
        if (pass) {
            k_bucket_fold<F><<<div_up(pl.TB, 128), 128, 0, st>>>(buckets, pass_buckets, pl.TB);
            BZK_LAUNCHED(ctx);
        }
    }
    timing_mark(ctx);
    k_bucket_slices<F><<<div_up(nslices, 128), 128, 0, st>>>(buckets, pl.NB, slice, nslices, slice_acc, slice_run);
    BZK_LAUNCHED(ctx);
    timing_mark(ctx);
    {
        const size_t smem = kCombineThreads * sizeof(Xyzz<F>);
        BZK_CUDA(ctx, cudaFuncSetAttribute(k_slice_combine<F>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        k_slice_combine<F><<<dim3(parts, 1 + nbits, pl.G), kCombineThreads, smem, st>>>(slice_acc, slice_run, per_win, partial);
        BZK_LAUNCHED(ctx);
        uint32_t ps_threads = 128;
        while (ps_threads > 32 && ps_threads / 2 >= parts) ps_threads /= 2;
        const size_t smem2 = ps_threads * sizeof(Xyzz<F>);
        BZK_CUDA(ctx, cudaFuncSetAttribute(k_partial_sum<F>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem2));
        k_partial_sum<F><<<rows, ps_threads, smem2, st>>>(partial, parts, win_out);
        BZK_LAUNCHED(ctx);
    }

    // 7. the (1 + nbits) sums of every group go to the host for the Horner folds (msm_host_finish)
    BZK_CUDA(ctx, cudaMemcpyAsync(h_win, win_out, rows * sizeof(Xyzz<F>), cudaMemcpyDeviceToHost, st));
    timing_mark(ctx);
    ctx->timing = saved_timing;
    return BZK_OK;
}

template <class F>
static void msm_host_finish(const MsmPlan &pl, const Xyzz<F> *h_win, typename Wire<F>::image *out) {
    if (pl.W == 0) { to_wire(out, Affine<F>::inf()); return; }
    // group sum = A + slice * sum_j 2^j T_j  (see k_bucket_slices)
    auto group_sum = [&](uint32_t g) {
        const Xyzz<F> *row = h_win + (size_t)g * (1 + pl.nbits);
        Xyzz<F> S = Xyzz<F>::inf();
        for (int j = (int)pl.nbits - 1; j >= 0; j--) {
            S = S.dbl();
            S.add(row[1 + j]);
        }
        Xyzz<F> m = Xyzz<F>::inf();
        for (int i = 31; i >= 0; i--) {
            m = m.dbl();
            if ((pl.slice >> i) & 1) m.add(S);
        }
        m.add(row[0]);
        return m;
    };
    // group g carries weight 2^(c*g) (the level factor 2^(c*G*t) is already in the table points)
    Xyzz<F> acc = group_sum(pl.G - 1);
    for (int w = (int)pl.G - 2; w >= 0; w--) {
        for (uint32_t k = 0; k < pl.c; k++) acc = acc.dbl();
        acc.add(group_sum((uint32_t)w));
    }
    to_wire(out, acc.to_affine());
}

template <class F>
static int32_t msm_run(bzk_ctx *ctx, const BasesRef<F> &d_bases, const Fr *d_scalars, size_t n, typename Wire<F>::image *out) {
    if (!out) return BZK_ERR_BAD_ARG;
    static_assert(kMaxWinPoints * sizeof(Xyzz<F>) <= 160 * 1024, "h_win on the stack");
    Xyzz<F> h_win[kMaxWinPoints];
    MsmPlan pl;
    uint32_t *d_long_len = nullptr;
    BZK_TRY(msm_enqueue<F>(ctx, ctx->stream, &ctx->ws, &ctx->ws_bytes, &ctx->pipe[0], true, d_bases, d_scalars, n, h_win, &pl, &d_long_len,
                           ctx->last_stream));
    // the plan this call ran (bzk_ctx_last_msm_plan); the queue length costs a copy, so only with timing on
    uint32_t long_len = 0;
    if (ctx->timing && d_long_len) BZK_CUDA(ctx, cudaMemcpyAsync(&long_len, d_long_len, sizeof long_len, cudaMemcpyDeviceToHost, ctx->stream));
    BZK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    timing_collect(ctx);
    const uint32_t rec[8] = {pl.c, pl.W, pl.T, pl.G, pl.NB, pl.slice, pl.nbits, long_len};
    memcpy(ctx->last_plan, rec, sizeof rec);
    msm_host_finish<F>(pl, h_win, out);
    return BZK_OK;
}

}  // namespace bzk
