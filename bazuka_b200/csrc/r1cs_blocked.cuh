// bazuka_b200 — a blocked R1CS: the index arithmetic of a constraint system whose middle is one block of rows repeated
// `reps` times (device + host; the kernels and the upload around it are in groth16.cu).
//
// Stored rows, per side, in row order:  head (explicit) | template (tmpl_rows) | tail (explicit).
// Logical rows:                         head | reps copies of the template | tail.
// Head and tail columns are absolute z indices.  A template column c >= var_lo is slot-relative: in copy k (0-based) it
// names c + k * var_stride; a template column c < var_lo (ONE, the inputs, variables shared by every copy) names c in
// every copy.  An MPN update batch is this with head = prologue + slot 0, template = slot 1, reps = n - 1, var_stride =
// the variables one slot allocates, tail = epilogue: the device holds one slot instead of n.
//
// The transposed product (out[j] = sum_row M[row][j] lag[row], what the trusted setup needs) is split so that every
// output has one writer per pass and no atomics are needed:
//   slot columns j >= var_lo   from the template transposed over relative columns [0, span): copy k contributes when
//                              0 <= j - var_lo - k * var_stride < span, i.e. for at most ceil(span / var_stride) copies
//   shared template columns    sum_t val * S[t], S[t] = sum_k lag[head_rows + k * tmpl_rows + t] (computed once per t)
//   head and tail columns      a small transposed list over the logical rows
// The host builders (density lists, transposed pieces) are plain C++ so that the CPU tier compiles this header with g++.
#pragma once
#include <algorithm>
#include <vector>
#include "ec.cuh"

namespace bzk {

struct BlockedShape {
    uint64_t head_rows = 0, tmpl_rows = 0, reps = 0, tail_rows = 0, var_lo = 0, var_stride = 0;
    BZK_HD uint64_t stored_rows() const { return head_rows + tmpl_rows + tail_rows; }
    BZK_HD uint64_t rows() const { return head_rows + tmpl_rows * reps + tail_rows; }
    // the logical row of template row t in copy k
    BZK_HD uint64_t tmpl_row(uint64_t k, uint64_t t) const { return head_rows + k * tmpl_rows + t; }
    // the first logical row of the tail
    BZK_HD uint64_t tail_base() const { return head_rows + tmpl_rows * reps; }
};

// logical row r -> its stored row, and the column shift of its copy (0 outside the template)
BZK_HD uint64_t blocked_row(const BlockedShape &b, uint64_t r, uint64_t *shift) {
    *shift = 0;
    if (r < b.head_rows) return r;
    const uint64_t q = r - b.head_rows, body = b.tmpl_rows * b.reps;
    if (q < body) {
        const uint64_t k = q / b.tmpl_rows;
        *shift = k * b.var_stride;
        return b.head_rows + (q - k * b.tmpl_rows);
    }
    return b.head_rows + b.tmpl_rows + (q - body);
}

// the z index a stored column names in a row with the given shift (head / tail rows have shift 0)
BZK_HD uint64_t blocked_col(const BlockedShape &b, uint32_t c, uint64_t shift) { return c >= b.var_lo ? c + shift : c; }

BZK_HD Fr fr_ld(const Fr *p) {
#if defined(__CUDA_ARCH__)
    Fr r;
    const uint4 *s = (const uint4 *)p;
    uint4 *d = (uint4 *)&r;
    d[0] = __ldg(s);
    d[1] = __ldg(s + 1);
    return r;
#else
    return *p;
#endif
}

// <M_row, z> of logical row r
BZK_HD Fr blocked_row_dot(const BlockedShape &b, const uint64_t *rowptr, const uint32_t *col, const Fr *val, uint64_t r, const Fr *z) {
    uint64_t shift;
    const uint64_t s = blocked_row(b, r, &shift);
    Fr acc = Fr::zero();
    const uint64_t k1 = rowptr[s + 1];
    for (uint64_t k = rowptr[s]; k < k1; k++) acc = acc + fr_ld(val + k) * fr_ld(z + blocked_col(b, col[k], shift));
    return acc;
}

// S[t] = sum over the copies of lag at template row t
BZK_HD Fr blocked_tmpl_rowsum(const BlockedShape &b, const Fr *lag, uint64_t t) {
    Fr acc = Fr::zero();
    for (uint64_t k = 0; k < b.reps; k++) acc = acc + fr_ld(lag + b.tmpl_row(k, t));
    return acc;
}

// the slot part of the transposed product at column j: the template transposed over relative columns d = c - var_lo in
// [0, span) (s_ptr[span + 1], s_row = template row, s_val)
BZK_HD Fr blocked_slot_column(const BlockedShape &b, uint64_t span, const uint64_t *s_ptr, const uint32_t *s_row, const Fr *s_val,
                              const Fr *lag, uint64_t j) {
    Fr acc = Fr::zero();
    if (j < b.var_lo || span == 0 || b.reps == 0) return acc;
    const uint64_t d = j - b.var_lo;
    const uint64_t k_lo = d >= span ? (d - span) / b.var_stride + 1 : 0;
    const uint64_t k_hi = d / b.var_stride < b.reps - 1 ? d / b.var_stride : b.reps - 1;
    for (uint64_t k = k_lo; k <= k_hi; k++) {
        const uint64_t rel = d - k * b.var_stride;
        for (uint64_t e = s_ptr[rel]; e < s_ptr[rel + 1]; e++) acc = acc + fr_ld(s_val + e) * fr_ld(lag + b.tmpl_row(k, s_row[e]));
    }
    return acc;
}

// one column of a transposed list: sum_e val[e] * w[row[e]] over the entries [ptr[u], ptr[u + 1])
BZK_HD Fr col_list_dot(const uint64_t *ptr, const uint32_t *row, const Fr *val, const Fr *w, uint64_t u) {
    Fr acc = Fr::zero();
    for (uint64_t e = ptr[u]; e < ptr[u + 1]; e++) acc = acc + fr_ld(val + e) * fr_ld(w + row[e]);
    return acc;
}

// ---- host side: validation, density, transposed pieces ------------------------------------------------------------

// A transposed list: the distinct columns `col`, each with its entries [ptr[u], ptr[u + 1]) of (row, val).
struct HostColList {
    std::vector<uint32_t> col;
    std::vector<uint64_t> ptr{0};
    std::vector<uint32_t> row;
    std::vector<Fr> val;
};
inline HostColList col_list(std::vector<std::pair<uint64_t, uint32_t>> &keys, const std::vector<Fr> &vals) {
    // keys[i] = (column, row) of vals[i]; sorted by column, rows ascending within a column
    std::vector<size_t> order(keys.size());
    for (size_t i = 0; i < order.size(); i++) order[i] = i;
    std::stable_sort(order.begin(), order.end(), [&](size_t x, size_t y) { return keys[x] < keys[y]; });
    HostColList L;
    for (size_t i : order) {
        if (L.col.empty() || L.col.back() != keys[i].first) {
            if (!L.col.empty()) L.ptr.push_back(L.row.size());
            L.col.push_back((uint32_t)keys[i].first);
        }
        L.row.push_back(keys[i].second);
        L.val.push_back(vals[i]);
    }
    if (!L.col.empty()) L.ptr.push_back(L.row.size());
    return L;
}

// one side's transposed pieces
struct HostBlockedT {
    uint64_t span = 0;  // template slot columns lie in [var_lo, var_lo + span)
    std::vector<uint64_t> s_ptr{0};
    std::vector<uint32_t> s_row;
    std::vector<Fr> s_val;
    HostColList shared, fixed;  // template columns < var_lo (rows = template rows); head and tail (rows = logical rows)
};
inline HostBlockedT blocked_transpose(const BlockedShape &b, const uint64_t *rp, const uint32_t *col, const Fr *val) {
    HostBlockedT T;
    const uint64_t t0 = b.head_rows, t1 = b.head_rows + b.tmpl_rows;
    for (uint64_t e = rp[t0]; e < rp[t1]; e++)
        if (col[e] >= b.var_lo) T.span = std::max<uint64_t>(T.span, col[e] - b.var_lo + 1);
    std::vector<uint64_t> cnt(T.span + 1, 0);
    std::vector<std::pair<uint64_t, uint32_t>> sk, fk;
    std::vector<Fr> sv, fv;
    for (uint64_t r = 0; r < b.stored_rows(); r++) {
        const bool tmpl = r >= t0 && r < t1;
        const uint64_t logical = r < t0 ? r : b.tail_base() + (r - t1);
        for (uint64_t e = rp[r]; e < rp[r + 1]; e++) {
            if (!tmpl) { fk.emplace_back(col[e], (uint32_t)logical); fv.push_back(val[e]); }
            else if (col[e] < b.var_lo) { sk.emplace_back(col[e], (uint32_t)(r - t0)); sv.push_back(val[e]); }
            else cnt[col[e] - b.var_lo + 1]++;
        }
    }
    if (b.reps == 0) { sk.clear(); sv.clear(); std::fill(cnt.begin(), cnt.end(), 0); }  // no copy reads the template
    T.s_ptr.assign(T.span + 1, 0);
    for (uint64_t d = 0; d < T.span; d++) T.s_ptr[d + 1] = T.s_ptr[d] + cnt[d + 1];
    T.s_row.resize(T.s_ptr[T.span]);
    T.s_val.resize(T.s_ptr[T.span]);
    std::vector<uint64_t> cur(T.s_ptr.begin(), T.s_ptr.end() - 1);
    if (b.reps)
        for (uint64_t r = t0; r < t1; r++)
            for (uint64_t e = rp[r]; e < rp[r + 1]; e++)
                if (col[e] >= b.var_lo) {
                    const uint64_t at = cur[col[e] - b.var_lo]++;
                    T.s_row[at] = (uint32_t)(r - t0);
                    T.s_val[at] = val[e];
                }
    T.shared = col_list(sk, sv);
    T.fixed = col_list(fk, fv);
    return T;
}

// Marks present[v] for every variable v some logical row names with a non-zero coefficient (bellman's density tracker;
// zero coefficients are skipped as `eval` does).  Template slot columns are marked once per copy.
inline void blocked_presence(const BlockedShape &b, const uint64_t *rp, const uint32_t *col, const Fr *val, std::vector<uint8_t> &present) {
    const uint64_t t0 = b.head_rows, t1 = b.head_rows + b.tmpl_rows;
    std::vector<uint32_t> rel;  // distinct slot columns of the template
    std::vector<uint8_t> seen;
    for (uint64_t r = 0; r < b.stored_rows(); r++) {
        const bool tmpl = r >= t0 && r < t1;
        if (tmpl && b.reps == 0) continue;
        for (uint64_t e = rp[r]; e < rp[r + 1]; e++) {
            if (val[e].is_zero()) continue;
            if (!tmpl || col[e] < b.var_lo) { present[col[e]] = 1; continue; }
            const uint64_t d = col[e] - b.var_lo;
            if (d >= seen.size()) seen.resize(d + 1, 0);
            if (!seen[d]) { seen[d] = 1; rel.push_back((uint32_t)d); }
        }
    }
    for (uint64_t k = 0; k < b.reps; k++)
        for (uint32_t d : rel) present[b.var_lo + d + k * b.var_stride] = 1;
}

// bellman's density lists from the presence of each variable in A and in B: a = every input ++ the aux present in A,
// b = the inputs and aux present in B
inline void density_lists(uint64_t num_inputs, const std::vector<uint8_t> &a_d, const std::vector<uint8_t> &b_d, std::vector<uint32_t> &a_idx,
                          std::vector<uint32_t> &b_idx) {
    const uint64_t nv = a_d.size();
    for (uint64_t v = 0; v < num_inputs; v++) a_idx.push_back((uint32_t)v);
    for (uint64_t v = num_inputs; v < nv; v++) if (a_d[v]) a_idx.push_back((uint32_t)v);
    for (uint64_t v = 0; v < nv; v++) if (b_d[v]) b_idx.push_back((uint32_t)v);
}

// Every stored coefficient must be its canonical Montgomery image (< r).  Presence is decided on the limbs, so an image
// >= r whose value is zero (r itself) would put its variable in a density list with an identity column, which bellman's
// Fr cannot hold and the key file reader refuses.  v: four little-endian 64-bit limbs, compared from the top one down.
inline bool fr_image_canonical(const uint64_t v[4]) {
    constexpr uint64_t r[4] = {0xffffffff00000001ull, 0x53bda402fffe5bfeull, 0x3339d80809a1d805ull, 0x73eda753299d7d48ull};
    for (int i = 3; i >= 0; i--)
        if (v[i] != r[i]) return v[i] < r[i];
    return false;
}

// Refuses (false) what the blocked form cannot name: a non-monotone rowptr, a missing array, an expanded column at or
// beyond nv (every copy of a slot column, up to the last), a template that repeats with a zero stride, a coefficient
// image >= r.
inline bool blocked_valid(const BlockedShape &b, uint64_t nv, const uint64_t *rp, const uint32_t *col, const void *val) {
    if (!rp || rp[0] != 0) return false;
    const uint64_t n = b.stored_rows(), t0 = b.head_rows, t1 = b.head_rows + b.tmpl_rows;
    for (uint64_t r = 0; r < n; r++) if (rp[r + 1] < rp[r]) return false;
    if (rp[n] && (!col || !val)) return false;
    if (b.reps && b.var_stride == 0) return false;
    for (uint64_t e = 0; e < rp[n]; e++)
        if (!fr_image_canonical((const uint64_t *)val + 4 * e)) return false;
    const uint64_t last = b.reps ? b.reps - 1 : 0;
    for (uint64_t r = 0; r < n; r++) {
        const bool tmpl = r >= t0 && r < t1;
        for (uint64_t e = rp[r]; e < rp[r + 1]; e++) {
            const uint64_t c = col[e];
            if (c >= nv) return false;
            if (tmpl && b.reps && c >= b.var_lo && (nv - c - 1) / b.var_stride < last) return false;  // c + last * stride >= nv
        }
    }
    return true;
}

}  // namespace bzk
