// TEST INFRASTRUCTURE (CPU tier only) — never linked into libbzk.so.
//
// csrc/ed25519.cuh compiled for the host with BZK_HOST_DEVICE_TEXT, so the field arithmetic is the device text (32-bit limbs,
// explicit carries) and the square root, decompression, SHA-512, the reduction mod l, the group law and the predicate are the
// code the batch kernels of csrc/ed25519.cu run.  Field elements cross as 32-byte little-endian integers (inputs may be
// unreduced: they enter through to_mont, one Montgomery product by R^2).
#include <cstring>

#include "ed25519.cuh"

using namespace bzk;

namespace {
Fe25519 mont(const uint8_t *c) { return fe_load_bytes<Fe25519>(c).to_mont(); }
void canon(uint8_t *out, const Fe25519 &m) { const Fe25519 c = m.from_mont(); memcpy(out, c.l, 32); }
const EdNiels25519 *table() {
    static const std::vector<EdNiels25519> t = ed_base_table();
    return t.data();
}
}  // namespace

extern "C" {
// op 0: a * b, 1: a^2, 2: a^-1 (by the (p-2) power chain), 3: a + b, 4: a - b; canonical result
void shim_fe_op(int op, const uint8_t *a, const uint8_t *b, uint8_t *out) {
    const Fe25519 x = mont(a), y = mont(b);
    canon(out, op == 0 ? x * y : op == 1 ? x.sqr() : op == 2 ? fe_invert(x) : op == 3 ? x + y : x - y);
}
// sqrt_ratio_i(u, v): was_square, and the root it returns
int shim_sqrt_ratio_i(const uint8_t *u, const uint8_t *v, uint8_t *out) {
    Fe25519 r;
    const bool ok = sqrt_ratio_i(mont(u), mont(v), &r);
    canon(out, r);
    return ok ? 1 : 0;
}
void shim_sha512(const uint8_t *data, uint64_t len, uint8_t *out) { sha512_parts(data, 0, data, 0, data, len, out); }
// the same digest with the input split into three pieces (the prepare kernel's R || pk || M)
void shim_sha512_parts(const uint8_t *a, uint64_t na, const uint8_t *b, uint64_t nb, const uint8_t *c, uint64_t nc, uint8_t *out) {
    sha512_parts(a, na, b, nb, c, nc, out);
}
void shim_sc_from_hash(const uint8_t *h, uint8_t *out) { const Sc25519 k = sc_from_hash(h); memcpy(out, k.l, 32); }
int shim_decompress(const uint8_t *pk, uint8_t *x, uint8_t *y) {
    Fe25519 ax, ay;
    if (!ed_decompress(pk, &ax, &ay)) return 0;
    canon(x, ax);
    canon(y, ay);
    return 1;
}
// the batch kernels' verdict on one item: ed25519_prepare, then ed25519_finish over the fixed-base table
int shim_verify(const uint8_t *pk, const uint8_t *msg, uint64_t len, const uint8_t *sig) {
    Fe25519 ax, ay;
    Sc25519 k;
    if (!ed25519_prepare(pk, sig, msg, len, &ax, &ay, &k)) return 0;
    return ed25519_finish(ax, ay, k, sig, table()) ? 1 : 0;
}
}
