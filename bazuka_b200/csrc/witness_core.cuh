// bazuka_b200 — the witness-program interpreter's per-slot loop, shared by the device kernel (witness.cu) and
// the host test shim (tests/hostshim: the "not gpu" tier runs real slot programs through this exact code).
// The memory policy is a template parameter: Mem::load(slot) / store(slot, v) address the slot's variable
// array, Mem::out(j, v) additionally emits block variable j into z, Mem::prefetch(slot) is a hint.
#pragma once
#include <algorithm>
#include <vector>

#include "ff.cuh"
#include "jubjub.cuh"

namespace bzk {

enum : int32_t { W_RAW = 0, W_MUL, W_BIT, W_ISZERO, W_INVZ, W_SELECT, W_JJ, W_NOP };

struct WitProgDev {
    const int32_t *ops;      // [n_ops][6]: opcode, lc0, lc1, lc2, lc3, imm
    const int32_t *lc_ptr;   // [n_lc + 1]
    const int32_t *lc_slot;  // [n_terms]
    const int32_t *lc_coef;  // [n_terms], 0 = coefficient one
    const Fr *coefs;         // Montgomery
    uint32_t n_ops, n_raw, n_ext;
};

BZK_HD int wit_operands(int32_t code) {
    return code == W_JJ ? 4 : code == W_SELECT ? 3 : code == W_MUL ? 2 : (code == W_RAW || code == W_NOP) ? 0 : 1;
}

template <class Mem>
BZK_HD_POW Fr wit_eval_lc(const WitProgDev &P, int32_t l, const Mem &mem) {  // not inlined on the device: ten call sites
    Fr acc = Fr::zero();
    const int32_t lo = P.lc_ptr[l], hi = P.lc_ptr[l + 1];
    for (int32_t k = lo; k < hi; k++) {
        const int32_t ci = P.lc_coef[k];
        Fr v = mem.load(P.lc_slot[k]);
        if (ci != 0) v = v * P.coefs[ci];
        acc = acc + v;
    }
    return acc;
}

template <class Mem>
BZK_HD void wit_prefetch_lc(const WitProgDev &P, int32_t l, const Mem &mem) {
    const int32_t lo = P.lc_ptr[l], hi = P.lc_ptr[l + 1];
    for (int32_t k = lo; k < hi; k++) mem.prefetch(P.lc_slot[k]);
}

// op j of the program (any order that respects the data flow): code / a0..a3 / imm = its row of P.ops
template <class Mem>
BZK_HD void wit_exec_op(const WitProgDev &P, const Fr &jj_d, const Fr *raws, uint32_t j, int32_t code, int32_t a0, int32_t a1, int32_t a2, int32_t a3,
                        int32_t imm, Mem &mem) {
    const uint32_t block0 = 1 + P.n_ext;
    Fr out = Fr::zero();
    switch (code) {
    case W_RAW: out = raws[imm].to_mont(); break;
    case W_MUL: {
        Fr a = wit_eval_lc(P, a0, mem);
        out = (a1 == a0) ? a.sqr() : a * wit_eval_lc(P, a1, mem);
        break;
    }
    case W_BIT: {
        Fr c = wit_eval_lc(P, a0, mem).from_mont();
        uint32_t w = 0;
#pragma unroll
        for (int i = 0; i < Fr::N; i++) w = (i == (imm >> 5)) ? c.l[i] : w;
        out = ((w >> (imm & 31)) & 1u) ? Fr::one() : Fr::zero();
        break;
    }
    case W_ISZERO: out = wit_eval_lc(P, a0, mem).is_zero() ? Fr::one() : Fr::zero(); break;
    case W_INVZ: {
        Fr a = wit_eval_lc(P, a0, mem);
        out = a.inv_gcd();  // 0 -> 0
        break;
    }
    case W_SELECT: {
        Fr s = wit_eval_lc(P, a0, mem), a = wit_eval_lc(P, a1, mem), b = wit_eval_lc(P, a2, mem);
        out = s.is_zero() ? a : b;
        break;
    }
    case W_JJ: {
        // twisted Edwards, a = -1 (/root/reference/src/crypto/jubjub/curve.rs:123-160; the gadget's hint
        // /root/reference/src/zk/groth16/gadgets/eddsa/mod.rs:75-101 yields (0,0) for off-curve inputs)
        Fr x1 = wit_eval_lc(P, a0, mem), y1 = wit_eval_lc(P, a1, mem);
        Fr x2 = wit_eval_lc(P, a2, mem), y2 = wit_eval_lc(P, a3, mem);
        Fr ox = Fr::zero(), oy = Fr::zero();
        if (jj_on_curve(x1, y1, jj_d) && jj_on_curve(x2, y2, jj_d)) {
            Fr x1x2 = x1 * x2, y1y2 = y1 * y2;
            Fr k = jj_d * x1x2 * y1y2;
            Fr dp = Fr::one() + k, dm = Fr::one() - k;
            Fr inv = (dp * dm).inv_gcd();
            ox = (x1 * y2 + y1 * x2) * dm * inv;
            oy = (y1y2 + x1x2) * dp * inv;
        }
        out = ox;
        mem.store(block0 + j + 1, oy);
        mem.out(j + 1, oy);
        break;
    }
    default: return;  // W_NOP: written by the preceding JJ
    }
    mem.store(block0 + j, out);
    mem.out(j, out);
}

// one slot in program order: raws / ext are the slot's rows (canonical); slots: 0 = ONE, 1..n_ext externals, then block variables
template <class Mem>
BZK_HD void wit_run_slot(const WitProgDev &P, const Fr &jj_d, const Fr *raws, const Fr *ext, Mem &mem) {
    mem.store(0, Fr::one());
    for (uint32_t k = 0; k < P.n_ext; k++) mem.store(1 + k, ext[k].to_mont());
    for (uint32_t j = 0; j < P.n_ops; j++) {
        const int32_t *op = P.ops + (size_t)j * 6;
        const int32_t code = op[0], a0 = op[1], a1 = op[2], a2 = op[3], a3 = op[4], imm = op[5];
        {
            // pull every operand towards L1 before the dependent evaluation starts (device: CCTL.E.PF1)
            const int nlc = wit_operands(code);
            if (nlc > 0) wit_prefetch_lc(P, a0, mem);
            if (nlc > 1 && a1 != a0) wit_prefetch_lc(P, a1, mem);
            if (nlc > 2) wit_prefetch_lc(P, a2, mem);
            if (nlc > 3) wit_prefetch_lc(P, a3, mem);
        }
        wit_exec_op(P, jj_d, raws, j, code, a0, a1, a2, a3, imm, mem);
    }
}

// Level schedule of a program (host): level of an op = 1 + the deepest of its operands (ONE, externals and raw inputs are at
// depth 0), so the ops of one level are mutually independent.  sops[k][8] = {opcode, lc0..lc3, imm, op index, 0} ordered by
// (level, opcode), NOPs dropped (a JJ writes both of its variables); level_ptr[L] .. level_ptr[L+1] delimit level L+1.
inline uint32_t wit_build_schedule(const int32_t *ops, uint64_t n_ops, const int32_t *lc_ptr, const int32_t *lc_slot, uint32_t n_ext,
                                   std::vector<int32_t> &sops, std::vector<int32_t> &level_ptr) {
    const uint64_t block0 = 1 + (uint64_t)n_ext;
    std::vector<uint32_t> depth(block0 + n_ops, 0);
    uint32_t n_levels = 0;
    uint64_t n_exec = 0;
    for (uint64_t j = 0; j < n_ops; j++) {
        const int32_t *op = ops + j * 6;
        if (op[0] == W_NOP) continue;  // its variable took the JJ's depth below
        uint32_t d = 0;
        const int nlc = wit_operands(op[0]);
        for (int a = 0; a < nlc; a++)
            for (int32_t k = lc_ptr[op[1 + a]]; k < lc_ptr[op[1 + a] + 1]; k++) d = std::max(d, depth[lc_slot[k]]);
        depth[block0 + j] = d + 1;
        if (op[0] == W_JJ) depth[block0 + j + 1] = d + 1;
        n_levels = std::max(n_levels, d + 1);
        n_exec++;
    }
    level_ptr.assign(n_levels + 2, 0);
    sops.assign(n_exec * 8 + 8, 0);
    // counting sort on (level, opcode); levels are 1-based
    std::vector<uint64_t> cnt((size_t)(n_levels + 1) * 8 + 1, 0);
    for (uint64_t j = 0; j < n_ops; j++)
        if (ops[j * 6] != W_NOP) cnt[(size_t)depth[block0 + j] * 8 + ops[j * 6] + 1]++;
    for (size_t i = 1; i < cnt.size(); i++) cnt[i] += cnt[i - 1];
    for (uint32_t L = 1; L <= n_levels + 1; L++) level_ptr[L - 1] = (int32_t)cnt[(size_t)L * 8];
    for (uint64_t j = 0; j < n_ops; j++) {
        const int32_t *op = ops + j * 6;
        if (op[0] == W_NOP) continue;
        int32_t *o = sops.data() + cnt[(size_t)depth[block0 + j] * 8 + op[0]]++ * 8;
        o[0] = op[0]; o[1] = op[1]; o[2] = op[2]; o[3] = op[3]; o[4] = op[4]; o[5] = op[5]; o[6] = (int32_t)j;
    }
    return n_levels;
}

}  // namespace bzk
