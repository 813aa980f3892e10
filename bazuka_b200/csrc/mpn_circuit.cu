// bazuka_b200 — the MPN update circuit as native code: R1CS and witness program emitted by C++.
//
// Structure-only synthesis (bellman's `KeypairAssembly` role) of `UpdateCircuit`
// (/root/reference/src/mpn/circuits/update_circuit.rs:49-494) over the reference's gadgets
// (/root/reference/src/zk/groth16/gadgets/{common,poseidon,merkle,eddsa}/) and bellman's
// `AllocatedNum / AllocatedBit / Boolean / to_bits_le_strict`, emitting
//   * the R1CS of a whole batch as three CSR matrices (what bzk_r1cs_upload takes), and
//   * the slot's and the epilogue's WITNESS PROGRAMS (what bzk_witness_program_upload takes): every allocation
//     records the rule that defines its value, exactly as the Python definition in bazuka_b200/mpn does.
// Values are never computed here — witnesses come from the interpreter (witness_core.cuh) — so the only field
// arithmetic is on coefficients.  The emission order is the gadget source order; tests compare every array with
// the Python definition's output (tests/test_mpn_cpu.py::test_native_circuit_compiler_equals_python).
#include "common.cuh"
#include <algorithm>
#include <array>
#include <map>
#include <memory>
#include <vector>

using namespace bzk;

namespace cc {

using Var = uint64_t;                                // 2*i = Input(i), 2*j+1 = Aux(j)
constexpr Var ONE = 0;
constexpr Var FAKE_STATE = 2ull * 1000000000000ull + 1;  // stand-in for the state variable entering a slot

inline Fr fr_u64(uint64_t v) { Fr a = Fr::zero(); a.l[0] = (uint32_t)v; a.l[1] = (uint32_t)(v >> 32); return a.to_mont(); }
inline Fr fr_canon(const bzk_fr *c) { Fr a; memcpy(a.l, c, 32); return a.to_mont(); }

// linear combination with Python-dict semantics: insertion-ordered, zero coefficients stay until emission
struct LC {
    std::vector<std::pair<Var, Fr>> t;
    LC() {}
    LC(Var v, const Fr &c) { t.emplace_back(v, c); }
    int find(Var v) const {
        for (size_t i = 0; i < t.size(); i++)
            if (t[i].first == v) return (int)i;
        return -1;
    }
    LC add_term(const Fr &c, Var v) const {
        LC o = *this;
        int i = o.find(v);
        if (i < 0) o.t.emplace_back(v, c);
        else o.t[i].second = o.t[i].second + c;
        return o;
    }
    LC operator+(const LC &b) const {
        LC o = *this;
        for (auto &kv : b.t) { int i = o.find(kv.first); if (i < 0) o.t.push_back(kv); else o.t[i].second = o.t[i].second + kv.second; }
        return o;
    }
    LC operator-(const LC &b) const {
        LC o = *this;
        for (auto &kv : b.t) { int i = o.find(kv.first); if (i < 0) o.t.emplace_back(kv.first, kv.second.neg()); else o.t[i].second = o.t[i].second - kv.second; }
        return o;
    }
    LC scaled(const Fr &k) const { LC o = *this; for (auto &kv : o.t) kv.second = kv.second * k; return o; }
};

enum Kind : int32_t { K_RAW = 0, K_MUL, K_BIT, K_ISZERO, K_INVZ, K_SELECT, K_JJ, K_NOP };
struct Recipe { Kind kind = K_RAW; LC a, b, c, d; int32_t imm = 0; };

struct Csr { std::vector<uint64_t> rowptr{0}; std::vector<Var> col; std::vector<Fr> val; };

struct CS {
    uint64_t n_inputs = 1, n_aux = 0, n_rows = 0;
    Csr m[3];
    bool record = false;
    std::vector<Recipe> recipes;
    Var alloc(const Recipe *r = nullptr) {
        if (record) recipes.push_back(r ? *r : Recipe());
        return 2 * (n_aux++) + 1;
    }
    Var alloc_input() { return 2 * (n_inputs++); }
    void enforce(const LC &a, const LC &b, const LC &c) {
        const LC *s[3] = {&a, &b, &c};
        for (int k = 0; k < 3; k++) {
            for (auto &kv : s[k]->t)
                if (!kv.second.is_zero()) { m[k].col.push_back(kv.first); m[k].val.push_back(kv.second); }
            m[k].rowptr.push_back(m[k].col.size());
        }
        n_rows++;
    }
};

struct Ctx {  // constants shared by the gadgets
    Fr one = Fr::one(), neg1 = Fr::one().neg(), jj_d, jj_a = Fr::one().neg(), base8_x, base8_y;
    struct Pos { uint32_t rf, rp; std::vector<Fr> rc; std::vector<Fr> mds; };
    std::map<uint32_t, Pos> pos;
};

struct Recipes {
    static Recipe mul(const LC &a, const LC &b) { Recipe r; r.kind = K_MUL; r.a = a; r.b = b; return r; }
    static Recipe bit(const LC &a, int i) { Recipe r; r.kind = K_BIT; r.a = a; r.imm = i; return r; }
    static Recipe iszero(const LC &a) { Recipe r; r.kind = K_ISZERO; r.a = a; return r; }
    static Recipe invz(const LC &a) { Recipe r; r.kind = K_INVZ; r.a = a; return r; }
    static Recipe select(const LC &s, const LC &a, const LC &b) { Recipe r; r.kind = K_SELECT; r.a = s; r.b = a; r.c = b; return r; }
    static Recipe jj(const LC &x1, const LC &y1, const LC &x2, const LC &y2) { Recipe r; r.kind = K_JJ; r.a = x1; r.b = y1; r.c = x2; r.d = y2; return r; }
    static Recipe nop() { Recipe r; r.kind = K_NOP; return r; }
};

// ------------------------------------------------------------------ bellman::gadgets::boolean
struct Bit { Var var; };
inline Var alloc_bit(CS &cs, const Recipe *r = nullptr) {
    Var v = cs.alloc(r);
    cs.enforce(LC(ONE, Fr::one()).add_term(Fr::one().neg(), v), LC(v, Fr::one()), LC());  // (1 - a) * a = 0
    return v;
}
inline Var alloc_bit_conditionally(CS &cs, Var must_be_false, const Recipe *r) {
    Var v = cs.alloc(r);
    cs.enforce(LC(ONE, Fr::one()).add_term(Fr::one().neg(), must_be_false).add_term(Fr::one().neg(), v), LC(v, Fr::one()), LC());
    return v;
}
inline Var bit_and(CS &cs, Var a, Var b) {
    LC la(a, Fr::one()), lb(b, Fr::one());
    Recipe r = Recipes::mul(la, lb);
    Var o = cs.alloc(&r);
    cs.enforce(la, lb, LC(o, Fr::one()));
    return o;
}
inline Var bit_and_not(CS &cs, Var a, Var b) {
    LC la(a, Fr::one()), lb = LC(ONE, Fr::one()).add_term(Fr::one().neg(), b);
    Recipe r = Recipes::mul(la, lb);
    Var o = cs.alloc(&r);
    cs.enforce(la, lb, LC(o, Fr::one()));
    return o;
}
inline Var bit_nor(CS &cs, Var a, Var b) {
    LC la = LC(ONE, Fr::one()).add_term(Fr::one().neg(), a), lb = LC(ONE, Fr::one()).add_term(Fr::one().neg(), b);
    Recipe r = Recipes::mul(la, lb);
    Var o = cs.alloc(&r);
    cs.enforce(la, lb, LC(o, Fr::one()));
    return o;
}
struct Boolean {
    enum { IS, NOT, CONST } kind = CONST;
    Var var = 0;
    bool c = false;
    static Boolean is(Var v) { Boolean b; b.kind = IS; b.var = v; return b; }
    static Boolean constant(bool v) { Boolean b; b.kind = CONST; b.c = v; return b; }
    Boolean not_() const {
        Boolean b = *this;
        if (kind == CONST) b.c = !c; else b.kind = kind == IS ? NOT : IS;
        return b;
    }
    static Boolean and_(CS &cs, const Boolean &a, const Boolean &b) {
        if (a.kind == CONST || b.kind == CONST) {
            const Boolean &k = a.kind == CONST ? a : b, &x = a.kind == CONST ? b : a;
            return k.c ? x : constant(false);
        }
        if (a.kind == IS && b.kind == IS) return is(bit_and(cs, a.var, b.var));
        if (a.kind == IS && b.kind == NOT) return is(bit_and_not(cs, a.var, b.var));
        if (a.kind == NOT && b.kind == IS) return is(bit_and_not(cs, b.var, a.var));
        return is(bit_nor(cs, a.var, b.var));
    }
};

// ------------------------------------------------------------------ gadgets/common: Number, UnsignedInteger, mux
struct Number {
    LC lc;
    static Number zero() { return Number(); }
    static Number one() { Number n; n.lc = LC(ONE, Fr::one()); return n; }
    static Number constant(const Fr &v) { Number n; n.lc = LC(ONE, v); return n; }
    static Number of(Var v) { Number n; n.lc = LC(v, Fr::one()); return n; }
    static Number of(Var v, const Fr &coeff) { Number n; n.lc = LC(v, coeff); return n; }
    Number add_constant(const Fr &c) const { Number n; n.lc = lc.add_term(c, ONE); return n; }
    Number add_num(const Fr &c, Var v) const { Number n; n.lc = lc.add_term(c, v); return n; }
    Number operator+(const Number &o) const { Number n; n.lc = lc + o.lc; return n; }
    Number operator-(const Number &o) const { Number n; n.lc = lc - o.lc; return n; }
    Number add_scaled(const Fr &c, const Number &o) const { Number n; n.lc = lc + o.lc.scaled(c); return n; }
    Var mul(CS &cs, const Number &o) const {
        Recipe r = Recipes::mul(lc, o.lc);
        Var out = cs.alloc(&r);
        cs.enforce(lc, o.lc, LC(out, Fr::one()));
        return out;
    }
    Var compress(CS &cs) const { return mul(cs, one()); }
    Boolean is_zero(CS &cs) const {  // number.rs:75-111
        Recipe rz = Recipes::iszero(lc), ri = Recipes::invz(lc);
        Var z = alloc_bit(cs, &rz), inv = cs.alloc(&ri);
        cs.enforce(LC() - lc, LC(inv, Fr::one()), LC(z, Fr::one()).add_term(Fr::one().neg(), ONE));
        cs.enforce(LC(z, Fr::one()), lc, LC());
        return Boolean::is(z);
    }
    Boolean is_equal(CS &cs, const Number &o) const { return (*this - o).is_zero(cs); }
    void assert_equal(CS &cs, const Number &o) const { cs.enforce(lc, LC(ONE, Fr::one()), o.lc); }
    void assert_equal_if_enabled(CS &cs, const Boolean &en, const Number &o) const {  // number.rs:132-178
        if (en.kind == Boolean::IS) {
            Recipe r = Recipes::mul(LC(en.var, Fr::one()), lc);
            Var eis = cs.alloc(&r);
            cs.enforce(LC(en.var, Fr::one()), lc, LC(eis, Fr::one()));
            cs.enforce(LC(en.var, Fr::one()), o.lc, LC(eis, Fr::one()));
        } else if (en.kind == Boolean::CONST) {
            if (en.c) assert_equal(cs, o);
        }
    }
};

struct UInt {
    std::vector<Var> bits;
    Number num;
    static UInt constrain(CS &cs, const Number &num, uint32_t nbits) {  // uint.rs
        UInt u;
        u.num = num;
        LC all;
        Fr coeff = Fr::one();
        for (uint32_t i = 0; i < nbits; i++) {
            Recipe r = Recipes::bit(num.lc, (int)i);
            Var b = alloc_bit(cs, &r);
            all = all.add_term(coeff, b);
            u.bits.push_back(b);
            coeff = coeff + coeff;
        }
        cs.enforce(all, LC(ONE, Fr::one()), num.lc);
        return u;
    }
    static UInt alloc(CS &cs, uint32_t nbits) { return constrain(cs, Number::of(cs.alloc()), nbits); }
    Boolean lt(CS &cs, const UInt &o) const {
        const uint32_t n = (uint32_t)bits.size();
        Fr p = Fr::one();
        for (uint32_t i = 0; i < n + 1; i++) p = p + p;  // 2^(n+1)
        UInt sb = constrain(cs, (num - o.num).add_constant(p), n + 2);
        return Boolean::is(sb.bits[n]);
    }
    Boolean gt(CS &cs, const UInt &o) const { return o.lt(cs, *this); }
    Boolean lte(CS &cs, const UInt &o) const { return gt(cs, o).not_(); }
};

inline Number extract_bool(const Boolean &b) {
    if (b.kind == Boolean::IS) return Number::of(b.var);
    if (b.kind == Boolean::NOT) return Number::one() - Number::of(b.var);
    return b.c ? Number::one() : Number::zero();
}
inline void assert_true(CS &cs, const Boolean &b) { extract_bool(b).assert_equal(cs, Number::one()); }
inline Boolean boolean_or(CS &cs, const Boolean &a, const Boolean &b) { return Boolean::and_(cs, a.not_(), b.not_()).not_(); }

// select ? b : a — mux.rs:7-47
inline Var mux(CS &cs, const Boolean &sel, const Number &a, const Number &b) {
    if (sel.kind == Boolean::IS) {
        Recipe r = Recipes::select(LC(sel.var, Fr::one()), a.lc, b.lc);
        Var ret = cs.alloc(&r);
        cs.enforce(a.lc - b.lc, LC(sel.var, Fr::one()), a.lc.add_term(Fr::one().neg(), ret));
        return ret;
    }
    // NOT(bit): not_s ? a : b
    Recipe r = Recipes::select(LC(sel.var, Fr::one()), b.lc, a.lc);
    Var ret = cs.alloc(&r);
    cs.enforce(b.lc - a.lc, LC(sel.var, Fr::one()), b.lc.add_term(Fr::one().neg(), ret));
    return ret;
}

// ------------------------------------------------------------------ gadgets/poseidon
inline Var sbox(CS &cs, const Number &a) {
    Var a2 = a.mul(cs, a);
    Var a4 = Number::of(a2).mul(cs, Number::of(a2));
    return a.mul(cs, Number::of(a4));
}
inline Number poseidon(CS &cs, const Ctx &cx, const std::vector<Number> &vals) {
    std::vector<Number> e;
    e.push_back(Number::zero());
    for (auto &v : vals) e.push_back(v);
    const uint32_t t = (uint32_t)e.size();
    const Ctx::Pos &P = cx.pos.at(t);
    size_t off = 0;
    for (uint32_t rnd = 0; rnd < P.rf + P.rp; rnd++) {
        for (uint32_t i = 0; i < t; i++) e[i] = e[i].add_constant(P.rc[off + i]);
        off += t;
        if (rnd < P.rf / 2 || rnd >= P.rf / 2 + P.rp) {
            for (uint32_t i = 0; i < t; i++) e[i] = Number::of(sbox(cs, e[i]));
        } else {
            Number first = Number::of(sbox(cs, e[0]));
            std::vector<Number> n;
            n.push_back(first);
            for (uint32_t i = 1; i < t; i++) n.push_back(Number::of(e[i].compress(cs)));
            e = n;
        }
        std::vector<Number> o;
        for (uint32_t j = 0; j < t; j++) {
            Number acc = Number::zero();
            for (uint32_t k = 0; k < t; k++) acc = acc.add_scaled(P.mds[j * t + k], e[k]);
            o.push_back(acc);
        }
        e = o;
    }
    return e[1];
}

// ------------------------------------------------------------------ gadgets/merkle (4-ary)
using Proof = std::vector<std::array<Var, 3>>;
inline Number merge_hash4(CS &cs, const Ctx &cx, Var s0, Var s1, const Number &v, const std::array<Var, 3> &p) {
    Boolean b0 = Boolean::is(s0), b1 = Boolean::is(s1);
    Boolean and_ = Boolean::and_(cs, b0, b1), or_ = boolean_or(cs, b0, b1);
    Number p0 = Number::of(p[0]), p1 = Number::of(p[1]), p2 = Number::of(p[2]);
    Var v0 = mux(cs, or_, v, p0);
    Var v1p = mux(cs, b0, p0, v);
    Var v1 = mux(cs, b1, Number::of(v1p), p1);
    Var v2p = mux(cs, b0, v, p2);
    Var v2 = mux(cs, b1, p1, Number::of(v2p));
    Var v3 = mux(cs, and_, p2, v);
    return poseidon(cs, cx, {Number::of(v0), Number::of(v1), Number::of(v2), Number::of(v3)});
}
inline Number calc_root4(CS &cs, const Ctx &cx, const UInt &index, const Number &val, const Proof &proof) {
    Number cur = val;
    for (size_t l = 0; l < proof.size(); l++) cur = merge_hash4(cs, cx, index.bits[2 * l], index.bits[2 * l + 1], cur, proof[l]);
    return cur;
}
inline void check_proof4(CS &cs, const Ctx &cx, const Boolean &en, const UInt &index, const Number &val, const Proof &proof, const Number &root) {
    Number nr = calc_root4(cs, cx, index, val, proof);
    root.assert_equal_if_enabled(cs, en, nr);
}
inline Proof alloc_proof(CS &cs, uint32_t depth) {
    Proof p(depth);
    for (auto &lvl : p)
        for (auto &v : lvl) v = cs.alloc();
    return p;
}

// ------------------------------------------------------------------ bellman AllocatedNum::to_bits_le_strict
inline std::vector<Boolean> to_bits_le_strict(CS &cs, Var self) {
    uint32_t rm1[8];
    for (int i = 0; i < 8; i++) rm1[i] = FrParams::p(i);
    rm1[0] -= 1;
    std::vector<Var> result, current_run;
    bool have_last = false, found_one = false;
    Var last_run = 0;
    LC me(self, Fr::one());
    for (int pos = 0; pos < 256; pos++) {
        const int bit_index = 255 - pos;
        const bool b = (rm1[bit_index >> 5] >> (bit_index & 31)) & 1;
        found_one |= b;
        if (!found_one) continue;
        Recipe r = Recipes::bit(me, bit_index);
        if (b) {
            Var bit = alloc_bit(cs, &r);
            current_run.push_back(bit);
            result.push_back(bit);
        } else {
            if (!current_run.empty()) {
                if (have_last) current_run.push_back(last_run);
                Var cur = current_run[0];
                for (size_t i = 1; i < current_run.size(); i++) cur = bit_and(cs, cur, current_run[i]);
                last_run = cur;
                have_last = true;
                current_run.clear();
            }
            Var bit = alloc_bit_conditionally(cs, last_run, &r);
            result.push_back(bit);
        }
    }
    LC lc;
    Fr coeff = Fr::one();
    for (size_t i = result.size(); i-- > 0;) { lc = lc.add_term(coeff, result[i]); coeff = coeff + coeff; }
    lc = lc.add_term(Fr::one().neg(), self);
    cs.enforce(LC(), LC(), lc);
    std::vector<Boolean> out;
    for (size_t i = result.size(); i-- > 0;) out.push_back(Boolean::is(result[i]));
    return out;
}

// ------------------------------------------------------------------ gadgets/eddsa
struct Point {
    Var x, y;
    static Point alloc(CS &cs) { Point p; p.x = cs.alloc(); p.y = cs.alloc(); return p; }
    static Point alloc_sum(CS &cs, const LC &x1, const LC &y1, const LC &x2, const LC &y2) {
        Recipe r = Recipes::jj(x1, y1, x2, y2), n = Recipes::nop();
        Point p;
        p.x = cs.alloc(&r);
        p.y = cs.alloc(&n);
        return p;
    }
    Boolean is_null(CS &cs) const {
        Boolean xz = Number::of(x).is_zero(cs), yz = Number::of(y).is_zero(cs);
        return Boolean::and_(cs, xz, yz);
    }
    Boolean is_equal(CS &cs, const Point &o) const {
        Boolean xe = Number::of(x).is_equal(cs, Number::of(o.x)), ye = Number::of(y).is_equal(cs, Number::of(o.y));
        return Boolean::and_(cs, xe, ye);
    }
    void assert_on_curve(CS &cs, const Ctx &cx, const Boolean &en) const {
        Var x2 = Number::of(x).mul(cs, Number::of(x)), y2 = Number::of(y).mul(cs, Number::of(y));
        Var x2y2 = Number::of(x2).mul(cs, Number::of(y2));
        Number lhs = Number::of(y2) - Number::of(x2), rhs = Number::of(x2y2, cx.jj_d) + Number::one();
        lhs.assert_equal_if_enabled(cs, en, rhs);
    }
    Point add_const(CS &cs, const Ctx &cx, const Fr &bx, const Fr &by) const {
        Point s = alloc_sum(cs, LC(x, Fr::one()), LC(y, Fr::one()), LC(ONE, bx), LC(ONE, by));
        const Fr k = cx.jj_d * bx * by;
        Var common = Number::of(x).mul(cs, Number::of(y));
        cs.enforce(LC(ONE, Fr::one()).add_term(k, common), LC(s.x, Fr::one()), LC(x, by).add_term(bx, y));
        cs.enforce(LC(ONE, Fr::one()).add_term(k.neg(), common), LC(s.y, Fr::one()), LC(y, by).add_term((cx.jj_a * bx).neg(), x));
        return s;
    }
    Point add(CS &cs, const Ctx &cx, const Point &o) const {
        Point s = alloc_sum(cs, LC(x, Fr::one()), LC(y, Fr::one()), LC(o.x, Fr::one()), LC(o.y, Fr::one()));
        auto M = [&](Var a, Var b) { return Number::of(a).mul(cs, Number::of(b)); };
        Var common = M(M(M(x, o.x), y), o.y);
        Var x1 = M(x, o.y), x2 = M(y, o.x);
        cs.enforce(LC(ONE, Fr::one()).add_term(cx.jj_d, common), LC(s.x, Fr::one()), LC(x1, Fr::one()).add_term(Fr::one(), x2));
        Var y1 = M(y, o.y), y2 = M(x, o.x);
        cs.enforce(LC(ONE, Fr::one()).add_term(cx.jj_d.neg(), common), LC(s.y, Fr::one()), LC(y1, Fr::one()).add_term(cx.jj_a.neg(), y2));
        return s;
    }
    Point mul(CS &cs, const Ctx &cx, Var b) const {
        std::vector<Boolean> bits = to_bits_le_strict(cs, b);
        std::vector<Boolean> be(bits.rbegin(), bits.rend());
        Point res;
        res.x = mux(cs, be[0], Number::zero(), Number::of(x));
        res.y = mux(cs, be[0], Number::constant(Fr::one()), Number::of(y));
        for (size_t i = 1; i < be.size(); i++) {
            res = res.add(cs, cx, res);
            Point rpb = res.add(cs, cx, *this);
            Point n;
            n.x = mux(cs, be[i], Number::of(res.x), Number::of(rpb.x));
            n.y = mux(cs, be[i], Number::of(res.y), Number::of(rpb.y));
            res = n;
        }
        return res;
    }
};
inline Point base_mul(CS &cs, const Ctx &cx, const Fr &bx, const Fr &by, Var b) {
    std::vector<Boolean> bits = to_bits_le_strict(cs, b);
    std::vector<Boolean> be(bits.rbegin(), bits.rend());
    Point res;
    res.x = mux(cs, be[0], Number::zero(), Number::constant(bx));
    res.y = mux(cs, be[0], Number::constant(Fr::one()), Number::constant(by));
    for (size_t i = 1; i < be.size(); i++) {
        res = res.add(cs, cx, res);
        Point rpb = res.add_const(cs, cx, bx, by);
        Point n;
        n.x = mux(cs, be[i], Number::of(res.x), Number::of(rpb.x));
        n.y = mux(cs, be[i], Number::of(res.y), Number::of(rpb.y));
        res = n;
    }
    return res;
}
inline void verify_eddsa(CS &cs, const Ctx &cx, const Boolean &en, const Point &pk, const Number &msg, const Point &sig_r, Var sig_s) {
    Var h = poseidon(cs, cx, {Number::of(sig_r.x), Number::of(sig_r.y), Number::of(pk.x), Number::of(pk.y), msg}).compress(cs);
    Point sb = base_mul(cs, cx, cx.base8_x, cx.base8_y, sig_s);
    Point rpha = pk.mul(cs, cx, h);
    rpha = rpha.add(cs, cx, sig_r);
    Point q = rpha.add(cs, cx, rpha);
    q = q.add(cs, cx, q);
    q = q.add(cs, cx, q);
    Number::of(q.x).assert_equal_if_enabled(cs, en, Number::of(sb.x));
    Number::of(q.y).assert_equal_if_enabled(cs, en, Number::of(sb.y));
}

// ------------------------------------------------------------------ UpdateCircuit
struct Prologue { Var state, fee_token, aux, claimed; };
inline Var alloc_inputized(CS &cs) {
    Var w = cs.alloc(), inp = cs.alloc_input();
    cs.enforce(LC(inp, Fr::one()), LC(ONE, Fr::one()), LC(w, Fr::one()));
    return w;
}
inline Prologue prologue(CS &cs) {
    Prologue p;
    alloc_inputized(cs);                  // commitment
    alloc_inputized(cs);                  // height
    p.state = alloc_inputized(cs);
    p.fee_token = cs.alloc();
    p.aux = alloc_inputized(cs);
    p.claimed = alloc_inputized(cs);
    return p;
}
struct BlockOut { Var state, final_fee; };
inline BlockOut tx_block(CS &cs, const Ctx &cx, uint32_t A, uint32_t T, Var state_wit, Var fee_tok) {
    auto num = [](Var v) { return Number::of(v); };
    Boolean enabled = Boolean::is(alloc_bit(cs));
    UInt tx_src_token_index = UInt::alloc(cs, 2 * T), tx_src_fee_token_index = UInt::alloc(cs, 2 * T), tx_dst_token_index = UInt::alloc(cs, 2 * T);
    Var src_tx_nonce = cs.alloc(), src_withdraw_nonce = cs.alloc();
    Point src_addr = Point::alloc(cs);
    src_addr.assert_on_curve(cs, cx, enabled);
    Var src_before_balances_hash = cs.alloc(), dst_before_balances_hash = cs.alloc();
    Var src_token_id = cs.alloc();
    UInt src_balance = UInt::alloc(cs, 64);
    Number src_token_balance_hash = poseidon(cs, cx, {num(src_token_id), src_balance.num});
    Var src_fee_token_id = cs.alloc();
    UInt src_fee_balance = UInt::alloc(cs, 64);
    Number src_fee_token_balance_hash = poseidon(cs, cx, {num(src_fee_token_id), src_fee_balance.num});
    Proof src_balance_proof = alloc_proof(cs, T);
    check_proof4(cs, cx, enabled, tx_src_token_index, src_token_balance_hash, src_balance_proof, num(src_before_balances_hash));
    UInt tx_amount = UInt::alloc(cs, 64), tx_fee = UInt::alloc(cs, 64);
    Number new_token_balance_hash = poseidon(cs, cx, {num(src_token_id), src_balance.num - tx_amount.num});
    Number balance_middle_root = calc_root4(cs, cx, tx_src_token_index, new_token_balance_hash, src_balance_proof);
    Proof src_fee_balance_proof = alloc_proof(cs, T);
    check_proof4(cs, cx, enabled, tx_src_fee_token_index, src_fee_token_balance_hash, src_fee_balance_proof, balance_middle_root);
    Number new_fee_token_balance_hash = poseidon(cs, cx, {num(src_fee_token_id), src_fee_balance.num - tx_fee.num});
    Number src_balance_final_root = calc_root4(cs, cx, tx_src_fee_token_index, new_fee_token_balance_hash, src_fee_balance_proof);
    Var tx_nonce = cs.alloc();
    UInt tx_src_index = UInt::alloc(cs, 2 * A);
    Var tx_amount_token_id = cs.alloc(), tx_fee_token_id = cs.alloc();
    num(fee_tok).assert_equal_if_enabled(cs, enabled, num(tx_fee_token_id));
    num(src_token_id).assert_equal(cs, num(tx_amount_token_id));
    num(src_fee_token_id).assert_equal(cs, num(tx_fee_token_id));
    Number src_hash = poseidon(cs, cx, {num(src_tx_nonce), num(src_withdraw_nonce), num(src_addr.x), num(src_addr.y), num(src_before_balances_hash)});
    Var dst_token_id = cs.alloc(), dst_balance = cs.alloc();
    Number dst_token_balance_hash = poseidon(cs, cx, {num(dst_token_id), num(dst_balance)});
    Number new_dst_token_balance_hash = poseidon(cs, cx, {num(tx_amount_token_id), num(dst_balance) + tx_amount.num});
    Proof dst_balance_proof = alloc_proof(cs, T);
    check_proof4(cs, cx, enabled, tx_dst_token_index, dst_token_balance_hash, dst_balance_proof, num(dst_before_balances_hash));
    Number dst_balance_final_root = calc_root4(cs, cx, tx_dst_token_index, new_dst_token_balance_hash, dst_balance_proof);
    Proof src_proof = alloc_proof(cs, A);
    check_proof4(cs, cx, enabled, tx_src_index, src_hash, src_proof, num(state_wit));
    Number new_src_tx_nonce = num(src_tx_nonce) + Number::constant(Fr::one());
    Number new_src_hash = poseidon(cs, cx, {new_src_tx_nonce, num(src_withdraw_nonce), num(src_addr.x), num(src_addr.y), src_balance_final_root});
    Number middle_root = calc_root4(cs, cx, tx_src_index, new_src_hash, src_proof);
    Point tx_dst_addr = Point::alloc(cs);
    tx_dst_addr.assert_on_curve(cs, cx, enabled);
    UInt tx_dst_index = UInt::alloc(cs, 2 * A);
    Var dst_tx_nonce = cs.alloc(), dst_withdraw_nonce = cs.alloc();
    Point dst_addr = Point::alloc(cs);
    Number dst_hash = poseidon(cs, cx, {num(dst_tx_nonce), num(dst_withdraw_nonce), num(dst_addr.x), num(dst_addr.y), num(dst_before_balances_hash)});
    Proof dst_proof = alloc_proof(cs, A);
    Boolean is_dst_null = dst_addr.is_null(cs);
    Boolean is_eq = dst_addr.is_equal(cs, tx_dst_addr);
    assert_true(cs, boolean_or(cs, is_dst_null, is_eq));
    check_proof4(cs, cx, enabled, tx_dst_index, dst_hash, dst_proof, middle_root);
    Number new_dst_hash = poseidon(cs, cx, {num(dst_tx_nonce), num(dst_withdraw_nonce), num(tx_dst_addr.x), num(tx_dst_addr.y), dst_balance_final_root});
    Number next_state = calc_root4(cs, cx, tx_dst_index, new_dst_hash, dst_proof);
    BlockOut out;
    out.state = mux(cs, enabled, num(state_wit), next_state);
    UInt plus = UInt::constrain(cs, tx_amount.num + tx_fee.num, 64);
    assert_true(cs, plus.lte(cs, src_balance));
    num(tx_nonce).assert_equal_if_enabled(cs, enabled, num(src_tx_nonce) + Number::constant(Fr::one()));
    out.final_fee = mux(cs, enabled, Number::zero(), tx_fee.num);
    Number tx_hash = poseidon(cs, cx, {num(tx_nonce), num(tx_dst_addr.x), num(tx_dst_addr.y), num(tx_amount_token_id), tx_amount.num, num(tx_fee_token_id), tx_fee.num});
    Point tx_sig_r = Point::alloc(cs);
    tx_sig_r.assert_on_curve(cs, cx, enabled);
    Var tx_sig_s = cs.alloc();
    verify_eddsa(cs, cx, enabled, src_addr, tx_hash, tx_sig_r, tx_sig_s);
    return out;
}
inline void epilogue(CS &cs, const Ctx &cx, Var state_wit, const Prologue &p, const Number &fee_sum) {
    Number h = poseidon(cs, cx, {Number::of(p.fee_token), fee_sum});
    cs.enforce(LC(p.aux, Fr::one()), LC(ONE, Fr::one()), h.lc);
    cs.enforce(LC(state_wit, Fr::one()), LC(ONE, Fr::one()), LC(p.claimed, Fr::one()));
}

// ------------------------------------------------------------------ Deposit / Withdraw circuits
// (/root/reference/src/mpn/circuits/deposit_circuit.rs:47-293, withdraw_circuit.rs:49-413; `reveal` of the batch:
//  /root/reference/src/zk/groth16/gadgets/reveal/mod.rs:13-64)
struct PublicInputs { Var state, aux, claimed; };
inline PublicInputs public_inputs(CS &cs) {
    PublicInputs p;
    alloc_inputized(cs);  // commitment
    alloc_inputized(cs);  // height
    p.state = alloc_inputized(cs);
    p.aux = alloc_inputized(cs);
    p.claimed = alloc_inputized(cs);
    return p;
}
inline Number reveal_list_of_structs(CS &cs, const Ctx &cx, const std::vector<std::vector<Number>> &rows) {
    std::vector<Number> leaves;
    for (auto &r : rows) leaves.push_back(poseidon(cs, cx, r));
    while (leaves.size() != 1) {
        std::vector<Number> up;
        for (size_t i = 0; i < leaves.size(); i += 4) up.push_back(poseidon(cs, cx, {leaves[i], leaves[i + 1], leaves[i + 2], leaves[i + 3]}));
        leaves = up;
    }
    return leaves[0];
}
struct DepositWits { Boolean enabled; Var token_id; UInt amount; Point pub_key; };
inline DepositWits deposit_phase1(CS &cs, const Ctx &cx, std::vector<Number> *row) {
    DepositWits w;
    Var en = alloc_bit(cs);
    w.enabled = Boolean::is(en);
    w.token_id = cs.alloc();
    w.amount = UInt::alloc(cs, 64);
    w.pub_key = Point::alloc(cs);
    Number pk_hash = poseidon(cs, cx, {Number::of(w.pub_key.x), Number::of(w.pub_key.y)});
    Var calldata = mux(cs, w.enabled, Number::zero(), pk_hash);
    *row = {Number::of(en), Number::of(w.token_id), w.amount.num, Number::of(calldata)};
    return w;
}
inline Var deposit_phase2(CS &cs, const Ctx &cx, uint32_t A, uint32_t T, const DepositWits &w, Var state_wit) {
    auto num = [](Var v) { return Number::of(v); };
    UInt tx_index = UInt::alloc(cs, 2 * A), tx_token_index = UInt::alloc(cs, 2 * T);
    w.pub_key.assert_on_curve(cs, cx, w.enabled);
    Var src_tx_nonce = cs.alloc(), src_withdraw_nonce = cs.alloc();
    Point src_addr = Point::alloc(cs);
    Var src_balances_hash = cs.alloc(), src_token_id = cs.alloc(), src_balance = cs.alloc();
    Number src_token_balance_hash = poseidon(cs, cx, {num(src_token_id), num(src_balance)});
    Proof bproof = alloc_proof(cs, T);
    check_proof4(cs, cx, w.enabled, tx_token_index, src_token_balance_hash, bproof, num(src_balances_hash));
    Number src_hash = poseidon(cs, cx, {num(src_tx_nonce), num(src_withdraw_nonce), num(src_addr.x), num(src_addr.y), num(src_balances_hash)});
    Proof proof = alloc_proof(cs, A);
    Boolean is_null_tok = num(src_token_id).is_zero(cs);
    Boolean is_eq_tok = num(src_token_id).is_equal(cs, num(w.token_id));
    assert_true(cs, boolean_or(cs, is_null_tok, is_eq_tok));
    Boolean is_null_addr = src_addr.is_null(cs);
    Boolean is_eq_addr = src_addr.is_equal(cs, w.pub_key);
    assert_true(cs, boolean_or(cs, is_null_addr, is_eq_addr));
    check_proof4(cs, cx, w.enabled, tx_index, src_hash, proof, num(state_wit));
    Number new_bal_hash = poseidon(cs, cx, {num(w.token_id), num(src_balance) + w.amount.num});
    Number new_balances_hash = calc_root4(cs, cx, tx_token_index, new_bal_hash, bproof);
    Number new_hash = poseidon(cs, cx, {num(src_tx_nonce), num(src_withdraw_nonce), num(w.pub_key.x), num(w.pub_key.y), new_balances_hash});
    Number next_state = calc_root4(cs, cx, tx_index, new_hash, proof);
    return mux(cs, w.enabled, num(state_wit), next_state);
}
struct WithdrawWits { Boolean enabled; Var amount_token_id; UInt amount; Var fee_token_id; UInt fee; Var fingerprint; Point pub_key; Var nonce; Point sig_r; Var sig_s; };
inline WithdrawWits withdraw_phase1(CS &cs, const Ctx &cx, std::vector<Number> *row) {
    WithdrawWits w;
    Var en = alloc_bit(cs);
    w.enabled = Boolean::is(en);
    w.amount_token_id = cs.alloc();
    w.amount = UInt::alloc(cs, 64);
    w.fee_token_id = cs.alloc();
    w.fee = UInt::alloc(cs, 64);
    w.fingerprint = cs.alloc();
    w.pub_key = Point::alloc(cs);
    w.nonce = cs.alloc();
    w.sig_r = Point::alloc(cs);
    w.sig_s = cs.alloc();
    auto num = [](Var v) { return Number::of(v); };
    Number cd_hash = poseidon(cs, cx, {num(w.pub_key.x), num(w.pub_key.y), num(w.nonce), num(w.sig_r.x), num(w.sig_r.y), num(w.sig_s)});
    Var calldata = mux(cs, w.enabled, Number::zero(), cd_hash);
    *row = {num(en), num(w.amount_token_id), w.amount.num, num(w.fee_token_id), w.fee.num, num(w.fingerprint), num(calldata)};
    return w;
}
inline Var withdraw_phase2(CS &cs, const Ctx &cx, uint32_t A, uint32_t T, const WithdrawWits &w, Var state_wit) {
    auto num = [](Var v) { return Number::of(v); };
    UInt tx_index = UInt::alloc(cs, 2 * A), tx_token_index = UInt::alloc(cs, 2 * T), tx_fee_token_index = UInt::alloc(cs, 2 * T);
    w.pub_key.assert_on_curve(cs, cx, w.enabled);
    Number tx_hash = poseidon(cs, cx, {num(w.fingerprint), num(w.nonce)});
    w.sig_r.assert_on_curve(cs, cx, w.enabled);
    verify_eddsa(cs, cx, w.enabled, w.pub_key, tx_hash, w.sig_r, w.sig_s);
    Var src_tx_nonce = cs.alloc(), src_withdraw_nonce = cs.alloc();
    Point src_addr = Point::alloc(cs);
    src_addr.assert_on_curve(cs, cx, w.enabled);
    Var before_token_hash = cs.alloc(), src_token_id = cs.alloc();
    num(src_token_id).assert_equal(cs, num(w.amount_token_id));
    Var src_balance = cs.alloc();
    Number src_token_balance_hash = poseidon(cs, cx, {num(src_token_id), num(src_balance)});
    Proof tproof = alloc_proof(cs, T);
    check_proof4(cs, cx, w.enabled, tx_token_index, src_token_balance_hash, tproof, num(before_token_hash));
    Number new_token_balance_hash = poseidon(cs, cx, {num(src_token_id), num(src_balance) - w.amount.num});
    Number balance_middle_root = calc_root4(cs, cx, tx_token_index, new_token_balance_hash, tproof);
    Var src_fee_token_id = cs.alloc();
    num(src_fee_token_id).assert_equal(cs, num(w.fee_token_id));
    Var src_fee_balance = cs.alloc();
    Number src_fee_token_balance_hash = poseidon(cs, cx, {num(src_fee_token_id), num(src_fee_balance)});
    Proof fproof = alloc_proof(cs, T);
    check_proof4(cs, cx, w.enabled, tx_fee_token_index, src_fee_token_balance_hash, fproof, balance_middle_root);
    Number new_fee_token_balance_hash = poseidon(cs, cx, {num(src_fee_token_id), num(src_fee_balance) - w.fee.num});
    Number src_hash = poseidon(cs, cx, {num(src_tx_nonce), num(src_withdraw_nonce), num(src_addr.x), num(src_addr.y), num(before_token_hash)});
    Proof proof = alloc_proof(cs, A);
    check_proof4(cs, cx, w.enabled, tx_index, src_hash, proof, num(state_wit));
    num(w.nonce).assert_equal_if_enabled(cs, w.enabled, num(src_withdraw_nonce) + Number::constant(Fr::one()));
    Number balance_final_root = calc_root4(cs, cx, tx_fee_token_index, new_fee_token_balance_hash, fproof);
    Number new_hash = poseidon(cs, cx, {num(src_tx_nonce), num(src_withdraw_nonce) + Number::constant(Fr::one()), num(w.pub_key.x), num(w.pub_key.y), balance_final_root});
    Number next_state = calc_root4(cs, cx, tx_index, new_hash, proof);
    return mux(cs, w.enabled, num(state_wit), next_state);
}

// ------------------------------------------------------------------ witness program compilation (witness_program.py compile_block)
struct Program {
    std::vector<int32_t> ops, lc_ptr{0}, lc_slot, lc_coef;
    std::vector<Fr> coefs;
    uint32_t n_raw = 0, n_ext = 0;
};
struct FrLess { bool operator()(const Fr &a, const Fr &b) const { return std::lexicographical_compare(a.l, a.l + 8, b.l, b.l + 8); } };

// rec[rec_first + j] is the rule of Aux(first_aux + j), j < count
inline bool compile_block(const std::vector<Recipe> &rec, size_t rec_first, uint64_t first_aux, size_t count, const std::vector<Var> &externals,
                          Program *P) {
    std::map<Var, int32_t> ext_slot;
    for (size_t k = 0; k < externals.size(); k++) ext_slot[externals[k]] = 1 + (int32_t)k;
    const int32_t block0 = 1 + (int32_t)externals.size();
    P->n_ext = (uint32_t)externals.size();
    std::map<Fr, int32_t, FrLess> coef_index;
    P->coefs.push_back(Fr::one());
    coef_index[Fr::one()] = 0;
    using Key = std::vector<std::pair<int32_t, std::array<uint32_t, 8>>>;
    std::map<Key, int32_t> pool;
    bool ok = true;
    auto lc_id = [&](const LC &lc, size_t upto) -> int32_t {
        std::vector<std::pair<int32_t, Fr>> terms;
        for (auto &kv : lc.t) {
            if (kv.second.is_zero()) continue;
            int32_t slot;
            if (kv.first == ONE) slot = 0;
            else if (ext_slot.count(kv.first)) slot = ext_slot[kv.first];
            else {
                const uint64_t a = kv.first >> 1;
                if (!(kv.first & 1) || a < first_aux || a >= first_aux + count) { ok = false; return 0; }
                slot = block0 + (int32_t)(a - first_aux);
            }
            if (slot >= block0 + (int32_t)upto) { ok = false; return 0; }
            terms.emplace_back(slot, kv.second);
        }
        std::sort(terms.begin(), terms.end(), [](const auto &a, const auto &b) { return a.first < b.first; });
        Key key;
        for (auto &tm : terms) { std::array<uint32_t, 8> c; memcpy(c.data(), tm.second.l, 32); key.emplace_back(tm.first, c); }
        auto it = pool.find(key);
        if (it != pool.end()) return it->second;
        const int32_t id = (int32_t)P->lc_ptr.size() - 1;
        pool[key] = id;
        for (auto &tm : terms) {
            P->lc_slot.push_back(tm.first);
            auto ci = coef_index.find(tm.second);
            if (ci == coef_index.end()) { ci = coef_index.emplace(tm.second, (int32_t)P->coefs.size()).first; P->coefs.push_back(tm.second); }
            P->lc_coef.push_back(ci->second);
        }
        P->lc_ptr.push_back((int32_t)P->lc_slot.size());
        return id;
    };
    for (size_t j = 0; j < count; j++) {
        const Recipe &r = rec[rec_first + j];
        int32_t op[6] = {r.kind, 0, 0, 0, 0, 0};
        switch (r.kind) {
        case K_RAW: op[5] = (int32_t)P->n_raw++; break;
        case K_MUL: op[1] = lc_id(r.a, j); op[2] = lc_id(r.b, j); break;
        case K_BIT: op[1] = lc_id(r.a, j); op[5] = r.imm; break;
        case K_ISZERO: case K_INVZ: op[1] = lc_id(r.a, j); break;
        case K_SELECT: op[1] = lc_id(r.a, j); op[2] = lc_id(r.b, j); op[3] = lc_id(r.c, j); break;
        case K_JJ: op[1] = lc_id(r.a, j); op[2] = lc_id(r.b, j); op[3] = lc_id(r.c, j); op[4] = lc_id(r.d, j); break;
        case K_NOP: break;
        }
        for (int k = 0; k < 6; k++) P->ops.push_back(op[k]);
    }
    return ok;
}

// constants of the gadgets: the Poseidon table (the blob bzk_poseidon_load_params takes) and JubJub's d, 8*BASE
inline bool load_constants(const uint8_t *blob, size_t len, const bzk_fr jubjub[3], Ctx *cx) {
    cx->jj_d = fr_canon(jubjub + 0); cx->base8_x = fr_canon(jubjub + 1); cx->base8_y = fr_canon(jubjub + 2);
    uint32_t n;
    memcpy(&n, blob + 8, 4);
    size_t off = 12;
    for (uint32_t i = 0; i < n; i++) {
        uint32_t hdr[4];
        if (off + 16 > len) return false;
        memcpy(hdr, blob + off, 16);
        off += 16;
        const uint32_t t = hdr[0], nrc = hdr[3];
        if (off + 32ull * (nrc + t * t) > len) return false;
        Ctx::Pos P;
        P.rf = hdr[1]; P.rp = hdr[2];
        for (uint32_t k = 0; k < nrc; k++) P.rc.push_back(fr_canon((const bzk_fr *)(blob + off + 32ull * k)));
        off += 32ull * nrc;
        for (uint32_t k = 0; k < t * t; k++) P.mds.push_back(fr_canon((const bzk_fr *)(blob + off + 32ull * k)));
        off += 32ull * t * t;
        cx->pos[t] = std::move(P);
    }
    return true;
}

}  // namespace cc

struct bzk_mpn_circuit {
    uint32_t A = 0, T = 0, B = 0;
    cc::CS cs;                    // the whole batch (structure only)
    cc::Program slot, epi, reveal;  // reveal: two-phase circuits only (externals = every slot's revealed row, slot-major)
    uint64_t p_aux = 0, slot_vars = 0, state_out = 0, final_fee = 0;
    std::vector<uint32_t> col[3];  // z indices
    // deposit / withdraw (two-phase circuits): slot = phase-1 program, epi = phase-2 program
    uint32_t kind = 0;
    uint64_t reveal_vars = 0;
    std::vector<int32_t> row_local;  // where each entry of the revealed row sits in the phase-1 block
    std::vector<int32_t> ext_src;    // per phase-2 external: -1 = the entering state, else the phase-1 RAW index it copies
    // update circuit: {head_rows, tmpl_rows, reps, tail_rows, var_lo, var_stride} (bzk_mpn_circuit_blocks); a blocked
    // compile stores head | template | tail only, and nnz[] counts the entries of the expanded matrices
    bool blocked = false;
    uint64_t blocks[6] = {0, 0, 0, 0, 0, 0};
    uint64_t nnz[3] = {0, 0, 0};
};

// The update circuit.  blocked: slots >= 2 advance the variable and row counts without storing their rows, so the
// matrices hold head | template (slot 1) | tail, the form bzk_r1cs_upload_blocked takes.
static int32_t update_circuit_compile(uint32_t log4_tree, uint32_t log4_token, uint32_t log4_batch, const uint8_t *poseidon_blob, size_t blob_len,
                                      const bzk_fr jubjub[3], bool blocked, bzk_mpn_circuit **out) {
    if (!poseidon_blob || !jubjub || !out || blob_len < 12 || memcmp(poseidon_blob, "BZKPOSv1", 8) || log4_tree == 0 || log4_tree > 31 ||
        log4_token == 0 || log4_token > 8 || log4_batch > 6)
        return BZK_ERR_BAD_ARG;
    std::unique_ptr<bzk_mpn_circuit> c(new (std::nothrow) bzk_mpn_circuit);
    if (!c) return BZK_ERR_OOM;
    c->A = log4_tree; c->T = log4_token; c->B = log4_batch;
    c->blocked = blocked;
    cc::Ctx cx;
    if (!cc::load_constants(poseidon_blob, blob_len, jubjub, &cx)) return BZK_ERR_BAD_ARG;
    const uint64_t n = 1ull << (2 * log4_batch);
    // ---- the slot program: prologue + ONE slot on a recording system, the entering state as a stand-in variable
    {
        cc::CS rs;
        rs.record = true;
        cc::Prologue p = cc::prologue(rs);
        c->p_aux = rs.n_aux;
        cc::BlockOut o = cc::tx_block(rs, cx, log4_tree, log4_token, cc::FAKE_STATE, p.fee_token);
        c->slot_vars = rs.n_aux - c->p_aux;
        c->state_out = (o.state >> 1) - c->p_aux;
        c->final_fee = (o.final_fee >> 1) - c->p_aux;
        if (!cc::compile_block(rs.recipes, c->p_aux, c->p_aux, c->slot_vars, {p.fee_token, cc::FAKE_STATE}, &c->slot)) return BZK_ERR_BAD_ARG;
    }
    // ---- the whole batch: R1CS; the epilogue's allocations are recorded for its program
    cc::CS &cs = c->cs;
    cc::Prologue p = cc::prologue(cs);
    cc::Var state = p.state;
    cc::Number fee_sum = cc::Number::zero();
    std::vector<cc::Var> fee_vars;
    // Slots 0 and 1 are synthesised; every later slot is slot 1's chunk of the matrices with the block-local variable
    // ids (its own block AND the entering state, which is the previous slot's output) advanced by one block — the slots
    // of `synthesize`'s loop differ in nothing else (update_circuit.rs:81-469).
    const uint64_t first_block = cs.n_aux;
    size_t chunk_lo[3] = {0, 0, 0}, chunk_hi[3] = {0, 0, 0}, rows_lo = 0, rows_hi = 0;
    uint64_t a_tx = 0;
    cc::BlockOut o1{};
    for (uint64_t k = 0; k < n; k++) {
        cc::BlockOut o;
        if (k < 2) {
            const size_t rows_before = cs.m[0].rowptr.size();
            size_t before[3];
            for (int s = 0; s < 3; s++) before[s] = cs.m[s].col.size();
            const uint64_t aux_before = cs.n_aux;
            o = cc::tx_block(cs, cx, log4_tree, log4_token, state, p.fee_token);
            if (k == 0) rows_lo = rows_hi = cs.m[0].rowptr.size();  // the template is empty unless slot 1 exists
            if (k == 0 && n > 1 && !blocked)  // every slot emits the same amount: size the arrays once instead of doubling through GBs
                for (int s = 0; s < 3; s++) {
                    const size_t per = cs.m[s].col.size() - before[s], rows_per = cs.m[s].rowptr.size() - rows_before;
                    cs.m[s].col.reserve(cs.m[s].col.size() + per * (n - 1) + 4096);
                    cs.m[s].val.reserve(cs.m[s].val.size() + per * (n - 1) + 4096);
                    cs.m[s].rowptr.reserve(cs.m[s].rowptr.size() + rows_per * (n - 1) + 4096);
                }
            if (k == 1) {
                a_tx = cs.n_aux - aux_before;
                o1 = o;
                rows_lo = rows_before; rows_hi = cs.m[0].rowptr.size();
                for (int s = 0; s < 3; s++) { chunk_lo[s] = before[s]; chunk_hi[s] = cs.m[s].col.size(); }
            }
        } else {
            const uint64_t shift = 2 * (k - 1) * a_tx;  // Var encoding: aux j = 2j + 1
            for (int s = 0; s < 3 && !blocked; s++) {
                cc::Csr &m = cs.m[s];
                const size_t base = m.col.size() - chunk_lo[s];
                for (size_t i = chunk_lo[s]; i < chunk_hi[s]; i++) {
                    const cc::Var v = m.col[i];
                    m.col.push_back(((v & 1) && (v >> 1) >= first_block) ? v + shift : v);
                }
                m.val.insert(m.val.end(), m.val.begin() + chunk_lo[s], m.val.begin() + chunk_hi[s]);
                for (size_t r = rows_lo; r < rows_hi; r++) m.rowptr.push_back(m.rowptr[r] + base);
            }
            cs.n_aux += a_tx;
            cs.n_rows += rows_hi - rows_lo;
            o.state = o1.state + shift;
            o.final_fee = o1.final_fee + shift;
        }
        state = o.state;
        fee_sum = fee_sum.add_num(Fr::one(), o.final_fee);
        fee_vars.push_back(o.final_fee);
    }
    const uint64_t epi_first = cs.n_aux;
    cs.record = true;  // only the epilogue's allocations are recorded
    cc::epilogue(cs, cx, state, p, fee_sum);
    cs.record = false;
    {
        std::vector<cc::Var> ext = {p.fee_token};
        ext.insert(ext.end(), fee_vars.begin(), fee_vars.end());
        if (!cc::compile_block(cs.recipes, 0, epi_first, cs.n_aux - epi_first, ext, &c->epi)) return BZK_ERR_BAD_ARG;
    }
    cs.recipes.clear();
    cs.recipes.shrink_to_fit();
    // rowptr[r] for r in [rows_lo, rows_hi) ends slot 1's rows: the head is the rows before it
    const uint64_t head = rows_lo - 1, tmpl = rows_hi - rows_lo, reps = n - 1;
    const uint64_t blocks[6] = {head, tmpl, reps, cs.n_rows - head - tmpl * reps, cs.n_inputs + first_block, n > 1 ? a_tx : c->slot_vars};
    memcpy(c->blocks, blocks, sizeof blocks);
    for (int s = 0; s < 3; s++) {
        c->nnz[s] = cs.m[s].col.size() + (blocked && n > 2 ? (n - 2) * (chunk_hi[s] - chunk_lo[s]) : 0);
        c->col[s].resize(cs.m[s].col.size());
        for (size_t i = 0; i < cs.m[s].col.size(); i++) {
            const cc::Var v = cs.m[s].col[i];
            c->col[s][i] = (uint32_t)((v & 1) ? cs.n_inputs + (v >> 1) : (v >> 1));
        }
        cs.m[s].col.clear();
        cs.m[s].col.shrink_to_fit();
    }
    *out = c.release();
    return BZK_OK;
}

extern "C" {

/* poseidon_blob: bazuka_b200/data/poseidon_params.bin (the table bzk_poseidon_load_params takes);
 * jubjub = {d, 8*BASE.x, 8*BASE.y} canonical */
int32_t bzk_mpn_update_circuit_compile(uint32_t log4_tree, uint32_t log4_token, uint32_t log4_batch, const uint8_t *poseidon_blob, size_t blob_len,
                                       const bzk_fr jubjub[3], bzk_mpn_circuit **out) {
    return update_circuit_compile(log4_tree, log4_token, log4_batch, poseidon_blob, blob_len, jubjub, false, out);
}
int32_t bzk_mpn_update_circuit_compile_blocked(uint32_t log4_tree, uint32_t log4_token, uint32_t log4_batch, const uint8_t *poseidon_blob,
                                               size_t blob_len, const bzk_fr jubjub[3], bzk_mpn_circuit **out) {
    return update_circuit_compile(log4_tree, log4_token, log4_batch, poseidon_blob, blob_len, jubjub, true, out);
}

/* out[9] = {head_rows, tmpl_rows, reps, tail_rows, var_lo, var_stride, stored nnz a, b, c}; update circuits only */
int32_t bzk_mpn_circuit_blocks(const bzk_mpn_circuit *c, uint64_t out[9]) {
    if (!c || !out || c->kind != 0) return BZK_ERR_BAD_ARG;
    memcpy(out, c->blocks, sizeof c->blocks);
    for (int s = 0; s < 3; s++) out[6 + s] = c->col[s].size();
    return BZK_OK;
}

int32_t bzk_mpn_circuit_free(bzk_mpn_circuit *c) {
    delete c;
    return BZK_OK;
}

/* shape[12] = {num_inputs, num_aux, num_constraints, nnz_a, nnz_b, nnz_c, p_aux, slot_vars, state_out, final_fee,
 *              epilogue_vars, 0} */
int32_t bzk_mpn_circuit_shape(const bzk_mpn_circuit *c, uint64_t shape[12]) {
    if (!c || !shape) return BZK_ERR_BAD_ARG;
    const uint64_t s[12] = {c->cs.n_inputs, c->cs.n_aux, c->cs.n_rows, c->kind ? c->col[0].size() : c->nnz[0], c->kind ? c->col[1].size() : c->nnz[1],
                            c->kind ? c->col[2].size() : c->nnz[2],
                            c->p_aux, c->slot_vars, c->state_out, c->final_fee, c->epi.ops.size() / 6, c->reveal_vars};
    memcpy(shape, s, sizeof s);
    return BZK_OK;
}

/* out[4] = {kind: 0 UpdateCircuit, 1 DepositCircuit, 2 WithdrawCircuit; log4_tree; log4_token; log4_batch} */
int32_t bzk_mpn_circuit_kind(const bzk_mpn_circuit *c, uint32_t out[4]) {
    if (!c || !out) return BZK_ERR_BAD_ARG;
    out[0] = c->kind; out[1] = c->A; out[2] = c->T; out[3] = c->B;
    return BZK_OK;
}

/* side = 0,1,2 (A,B,C): rowptr u64[ncons+1], col u32[nnz], val Fr[nnz] (Montgomery) — the arrays of bzk_r1cs_upload; of a
 * blocked compile, the stored rows head | template | tail (sizes from bzk_mpn_circuit_blocks) */
int32_t bzk_mpn_circuit_matrix(const bzk_mpn_circuit *c, uint32_t side, uint64_t *rowptr, uint32_t *col, bzk_fr *val) {
    if (!c || side > 2 || !rowptr || !col || !val) return BZK_ERR_BAD_ARG;
    memcpy(rowptr, c->cs.m[side].rowptr.data(), c->cs.m[side].rowptr.size() * 8);
    memcpy(col, c->col[side].data(), c->col[side].size() * 4);
    memcpy(val, c->cs.m[side].val.data(), c->cs.m[side].val.size() * sizeof(Fr));
    return BZK_OK;
}

/* which = 0 slot program, 1 epilogue program.  sizes[6] = {n_ops, n_lc, n_terms, n_coefs, n_raw, n_ext};
 * with non-null outputs the arrays are copied (ops int32[n_ops*6], lc_ptr int32[n_lc+1], lc_slot / lc_coef int32[n_terms],
 * coefs Fr[n_coefs] Montgomery) — the arguments of bzk_witness_program_upload */
int32_t bzk_mpn_circuit_program(const bzk_mpn_circuit *c, uint32_t which, uint64_t sizes[6], int32_t *ops, int32_t *lc_ptr, int32_t *lc_slot,
                                int32_t *lc_coef, bzk_fr *coefs) {
    if (!c || which > 2 || !sizes) return BZK_ERR_BAD_ARG;
    const cc::Program &P = which == 2 ? c->reveal : which ? c->epi : c->slot;
    const uint64_t s[6] = {P.ops.size() / 6, P.lc_ptr.size() - 1, P.lc_slot.size(), P.coefs.size(), P.n_raw, P.n_ext};
    memcpy(sizes, s, sizeof s);
    if (ops) memcpy(ops, P.ops.data(), P.ops.size() * 4);
    if (lc_ptr) memcpy(lc_ptr, P.lc_ptr.data(), P.lc_ptr.size() * 4);
    if (lc_slot) memcpy(lc_slot, P.lc_slot.data(), P.lc_slot.size() * 4);
    if (lc_coef) memcpy(lc_coef, P.lc_coef.data(), P.lc_coef.size() * 4);
    if (coefs) memcpy(coefs, P.coefs.data(), P.coefs.size() * sizeof(Fr));
    return BZK_OK;
}


/* kind: 1 = DepositCircuit, 2 = WithdrawCircuit.  Program 0 = phase 1 (the slot's transaction fields and calldata),
 * program 1 = phase 2 (the slot's state transition; externals per bzk_mpn_circuit_two_phase_info).  aux layout of the
 * batch = [5 public-input copies][phase 1 x n][reveal][phase 2 x n].
 * shape: slot_vars = phase-1 variables per slot, epilogue_vars = phase-2 variables per slot, last = reveal variables. */
int32_t bzk_mpn_dw_circuit_compile(uint32_t kind, uint32_t log4_tree, uint32_t log4_token, uint32_t log4_batch, const uint8_t *poseidon_blob,
                                   size_t blob_len, const bzk_fr jubjub[3], bzk_mpn_circuit **out) {
    if ((kind != 1 && kind != 2) || !out) return BZK_ERR_BAD_ARG;
    if (!poseidon_blob || !jubjub || blob_len < 12 || memcmp(poseidon_blob, "BZKPOSv1", 8) || log4_tree == 0 || log4_tree > 31 ||
        log4_token == 0 || log4_token > 8 || log4_batch > 6)
        return BZK_ERR_BAD_ARG;
    std::unique_ptr<bzk_mpn_circuit> c(new (std::nothrow) bzk_mpn_circuit);
    if (!c) return BZK_ERR_OOM;
    c->A = log4_tree; c->T = log4_token; c->B = log4_batch; c->kind = kind;
    cc::Ctx cx;
    if (!cc::load_constants(poseidon_blob, blob_len, jubjub, &cx)) return BZK_ERR_BAD_ARG;
    const uint64_t n = 1ull << (2 * log4_batch);
    // ---- the two slot programs: public inputs + phase 1 + phase 2 of ONE slot on a recording system
    {
        cc::CS rs;
        rs.record = true;
        cc::public_inputs(rs);
        c->p_aux = rs.n_aux;
        std::vector<cc::Number> row;
        cc::DepositWits dw;
        cc::WithdrawWits ww;
        if (kind == 1) dw = cc::deposit_phase1(rs, cx, &row); else ww = cc::withdraw_phase1(rs, cx, &row);
        c->slot_vars = rs.n_aux - c->p_aux;
        for (auto &nm : row) {
            if (nm.lc.t.size() != 1 || !(nm.lc.t[0].first & 1)) return BZK_ERR_BAD_ARG;
            c->row_local.push_back((int32_t)((nm.lc.t[0].first >> 1) - c->p_aux));
        }
        const uint64_t start2 = rs.n_aux;
        const cc::Var so = kind == 1 ? cc::deposit_phase2(rs, cx, log4_tree, log4_token, dw, cc::FAKE_STATE)
                                     : cc::withdraw_phase2(rs, cx, log4_tree, log4_token, ww, cc::FAKE_STATE);
        const uint64_t n2 = rs.n_aux - start2;
        c->state_out = (so >> 1) - start2;
        if (!cc::compile_block(rs.recipes, c->p_aux, c->p_aux, c->slot_vars, {}, &c->slot)) return BZK_ERR_BAD_ARG;
        // externals of phase 2 in order of first appearance: phase-1 variables of the slot (raw fields) and the entering state
        std::vector<cc::Var> ext;
        auto scan = [&](const cc::LC &lc) {
            for (auto &kv : lc.t) {
                const cc::Var v = kv.first;
                if (v == cc::ONE) continue;
                if ((v & 1) && (v >> 1) >= start2 && (v >> 1) < start2 + n2) continue;
                if (std::find(ext.begin(), ext.end(), v) == ext.end()) ext.push_back(v);
            }
        };
        for (uint64_t j = 0; j < n2; j++) {
            const cc::Recipe &r = rs.recipes[start2 + j];
            if (r.kind == cc::K_RAW || r.kind == cc::K_NOP) continue;
            scan(r.a);
            if (r.kind == cc::K_MUL || r.kind == cc::K_SELECT || r.kind == cc::K_JJ) scan(r.b);
            if (r.kind == cc::K_SELECT || r.kind == cc::K_JJ) scan(r.c);
            if (r.kind == cc::K_JJ) scan(r.d);
        }
        std::map<cc::Var, int32_t> raw_index;
        int32_t k = 0;
        for (uint64_t j = 0; j < c->slot_vars; j++)
            if (rs.recipes[c->p_aux + j].kind == cc::K_RAW) raw_index[2 * (c->p_aux + j) + 1] = k++;
        for (cc::Var v : ext) {
            if (v == cc::FAKE_STATE) c->ext_src.push_back(-1);
            else if (raw_index.count(v)) c->ext_src.push_back(raw_index[v]);
            else return BZK_ERR_BAD_ARG;  // phase 2 reads a derived phase-1 variable
        }
        if (!cc::compile_block(rs.recipes, start2, start2, n2, ext, &c->epi)) return BZK_ERR_BAD_ARG;
    }
    // ---- the whole batch: R1CS
    cc::CS &cs = c->cs;
    cc::PublicInputs p = cc::public_inputs(cs);
    std::vector<std::vector<cc::Number>> rows(n);
    std::vector<cc::DepositWits> dws;
    std::vector<cc::WithdrawWits> wws;
    for (uint64_t k = 0; k < n; k++) {
        if (kind == 1) dws.push_back(cc::deposit_phase1(cs, cx, &rows[k])); else wws.push_back(cc::withdraw_phase1(cs, cx, &rows[k]));
    }
    const uint64_t before_reveal = cs.n_aux;
    cs.record = true;  // only the reveal's allocations are recorded: its program's externals are the rows' variables
    cc::Number tx_root = cc::reveal_list_of_structs(cs, cx, rows);
    cs.record = false;
    c->reveal_vars = cs.n_aux - before_reveal;
    {
        std::vector<cc::Var> ext;
        for (auto &r : rows)
            for (auto &nm : r) ext.push_back(nm.lc.t[0].first);
        if (!cc::compile_block(cs.recipes, 0, before_reveal, c->reveal_vars, ext, &c->reveal)) return BZK_ERR_BAD_ARG;
        cs.recipes.clear();
        cs.recipes.shrink_to_fit();
    }
    cs.enforce(cc::LC(p.aux, Fr::one()), cc::LC(cc::ONE, Fr::one()), tx_root.lc);
    cc::Var state = p.state;
    for (uint64_t k = 0; k < n; k++)
        state = kind == 1 ? cc::deposit_phase2(cs, cx, log4_tree, log4_token, dws[k], state) : cc::withdraw_phase2(cs, cx, log4_tree, log4_token, wws[k], state);
    cs.enforce(cc::LC(state, Fr::one()), cc::LC(cc::ONE, Fr::one()), cc::LC(p.claimed, Fr::one()));
    for (int s = 0; s < 3; s++) {
        c->col[s].resize(cs.m[s].col.size());
        for (size_t i = 0; i < cs.m[s].col.size(); i++) {
            const cc::Var v = cs.m[s].col[i];
            c->col[s][i] = (uint32_t)((v & 1) ? cs.n_inputs + (v >> 1) : (v >> 1));
        }
        cs.m[s].col.clear();
        cs.m[s].col.shrink_to_fit();
    }
    *out = c.release();
    return BZK_OK;
}

/* two-phase circuits: row_local[n_row] (position of each revealed-row entry in the phase-1 block) and ext_src[n_ext]
 * (per phase-2 external: -1 = the state root entering the slot, k >= 0 = the slot's phase-1 RAW input number k).
 * counts[2] = {n_row, n_ext}; array outputs optional. */
int32_t bzk_mpn_circuit_two_phase_info(const bzk_mpn_circuit *c, uint64_t counts[2], int32_t *row_local, int32_t *ext_src) {
    if (!c || !counts) return BZK_ERR_BAD_ARG;
    counts[0] = c->row_local.size();
    counts[1] = c->ext_src.size();
    if (row_local) memcpy(row_local, c->row_local.data(), c->row_local.size() * 4);
    if (ext_src) memcpy(ext_src, c->ext_src.data(), c->ext_src.size() * 4);
    return BZK_OK;
}

}  // extern "C"
