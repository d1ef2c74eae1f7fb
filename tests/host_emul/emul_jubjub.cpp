// CPU unit-test harness of the PRODUCT's Jubjub header (zero_chain_b200/csrc/jubjub.cuh) compiled with ZK_HOST_EMUL:
// square root, extended-coordinate addition / doubling and the full decode, checked against the Python oracle by
// tests/test_host_emul_jubjub.py.  Test infrastructure only — never linked into libzkb200.so.
// Every value crosses as canonical Fr: 8 little-endian u32 words.
#define ZK_HOST_EMUL 1
#include "jubjub.cuh"
#include <string.h>

using namespace zkjj;

static Fr load(const uint32_t *a) { Fr x; memcpy(x.l, a, 32); return Fr::from_canonical(x); }
static void store(uint32_t *o, const Fr &x) { Fr c = x.to_canonical(); memcpy(o, c.l, 32); }
static Ext lift(const uint32_t *xy, const uint32_t *zc) {   // affine (x, y) scaled by z: (xz : yz : z : xyz)
    Fr x = load(xy), y = load(xy + 8), z = load(zc);
    Ext p;
    p.x = x * z; p.y = y * z; p.z = z; p.t = x * y * z;
    return p;
}
static void to_affine(const Ext &p, uint32_t *o) {
    Fr zi = p.z.inverse();
    store(o, p.x * zi); store(o + 8, p.y * zi);
}

extern "C" {
// 1 and a root of a, or 0 for a non-residue
int emu_jj_sqrt(const uint32_t *a, uint32_t *o) {
    Fr r;
    if (!fr_sqrt(load(a), r)) return 0;
    store(o, r);
    return 1;
}
// p, q: affine (x | y); zp, zq: the projective scale of each operand; o: affine p + q.  The T coordinate of the output
// is checked as well: returns 0 if T Z != X Y
int emu_jj_add(const uint32_t *p, const uint32_t *zp, const uint32_t *q, const uint32_t *zq, uint32_t *o) {
    Ext r = ext_add(lift(p, zp), lift(q, zq), jj_d2());
    to_affine(r, o);
    return r.t * r.z == r.x * r.y;
}
int emu_jj_dbl(const uint32_t *p, const uint32_t *zp, uint32_t *o) {
    Ext r = ext_dbl(lift(p, zp));
    to_affine(r, o);
    return r.t * r.z == r.x * r.y;
}
// [r_J] p is the identity?
int emu_jj_order_kills(const uint32_t *p) {
    uint32_t one[8] = {1, 0, 0, 0, 0, 0, 0, 0};
    return ext_is_identity(ext_mul_order(lift(p, one), jj_d2()));
}
// n encodings -> xy[16 i .. 16 i + 15] (canonical x | y), st[i]
void emu_jj_into_xy(const uint8_t *enc, size_t n, uint32_t *xy, uint8_t *st) {
    for (size_t i = 0; i < n; i++) {
        uint32_t w[8];
        memcpy(w, enc + 32 * i, 32);          // little-endian host: the byte order of the encoding
        Fr x, y;
        st[i] = (uint8_t)jubjub_into_xy(w, x, y);
        memcpy(xy + 16 * i, x.l, 32);
        memcpy(xy + 16 * i + 8, y.l, 32);
    }
}
}
