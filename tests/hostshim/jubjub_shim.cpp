// TEST INFRASTRUCTURE (CPU tier only) — never linked into libbzk.so.
//
// csrc/jubjub.cuh compiled for the host with BZK_HOST_DEVICE_TEXT, so the field arithmetic is the device text (32-bit limbs,
// explicit carries) and the group law, the square root, the windowed and fixed-base multiplications and the signature predicate
// are the code the batch kernels of csrc/jubjub.cu run.  Scalars cross as canonical 32-byte little-endian integers.
#include <cstring>

#include "jubjub.cuh"

using namespace bzk;

namespace {
Fr mont(const uint64_t *c) { Fr a; memcpy(a.l, c, 32); return a.to_mont(); }
Fr plain(const uint64_t *c) { Fr a; memcpy(a.l, c, 32); return a; }
void canon(uint64_t *out, const Fr &m) { const Fr c = m.from_mont(); memcpy(out, c.l, 32); }
void affine(uint64_t *out, const JJ &p) {
    const Fr zi = p.z.inv_gcd();
    canon(out, p.x * zi);
    canon(out + 4, p.y * zi);
}
std::vector<JJNiels> g_table;
Fr g_table_d;
const JJNiels *table(const Fr &d) {
    if (g_table.empty() || !(g_table_d == d)) { g_table = jj_fixed_base_table(d); g_table_d = d; }
    return g_table.data();
}
}  // namespace

extern "C" {
// y of PointCompressed(x, odd).decompress(); 0 where there is none
int shim_jj_decompress(const uint64_t *d, const uint64_t *x, int odd, uint64_t *y_out) {
    Fr y;
    if (!jj_decompress_root(mont(x), mont(d), &y)) return 0;
    canon(y_out, jj_with_parity(y, odd != 0));
    return 1;
}
// out = affine [k] (px, py) by the 4-bit window (k any 256-bit integer)
void shim_jj_mul(const uint64_t *d, const uint64_t *px, const uint64_t *py, const uint64_t *k, uint64_t *out) {
    affine(out, jj_mul(jj_from_affine(mont(px), mont(py)), plain(k), mont(d).dbl()));
}
// out = affine [k] BASE through the fixed-base table
void shim_jj_mul_fixed(const uint64_t *d, const uint64_t *k, uint64_t *out) { affine(out, jj_mul_fixed(table(mont(d)), plain(k))); }
// the batch kernels' verdict on one bzk_eddsa_item, given h = Poseidon(R.x, R.y, A.x, A.y, msg): canonical scalars, the key
// decompressed, then jj_eddsa_check with [s] BASE from the fixed-base table
int shim_eddsa_item(const uint64_t *d, const uint64_t *pk_x, int pk_odd, const uint64_t *msg, const uint64_t *rx, const uint64_t *ry, const uint64_t *s,
                    const uint64_t *h) {
    auto is_canonical = [](const uint64_t *c) { const Fr v = plain(c); return Fr::reduce_once(v) == v; };
    if (!is_canonical(pk_x) || !is_canonical(msg) || !is_canonical(rx) || !is_canonical(ry) || !is_canonical(s)) return 0;
    const Fr dm = mont(d);
    Fr ay;
    if (!jj_decompress_root(mont(pk_x), dm, &ay)) return 0;
    ay = jj_with_parity(ay, pk_odd != 0);
    return jj_eddsa_check(dm, mont(pk_x), ay, mont(rx), mont(ry), plain(h), jj_mul_fixed(table(dm), plain(s))) ? 1 : 0;
}
}
