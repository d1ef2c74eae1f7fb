// RedJubjub signature verification with the Diversifier generator: what `impl Verify for RedjubjubSignature`
// (core/primitives/src/signature.rs:65-82) runs per extrinsic.
//
// Restates, verdict for verdict, PublicKey::try_from(signer) + PublicKey::verify (core/jubjub/src/redjubjub.rs:127-155):
//   c = H*(rbar || msg)   BLAKE2b-512 with personalization "Zcash_RedJubjubH" (redjubjub.rs:24-26, util.rs:5-11), then
//                         Fs::to_uniform: the digest as a little-endian 512-bit integer mod r_J (curve/fs.rs:587-592)
//   vk = Point::read(signer), R = Point::read(rbar)      no subgroup test (jubjub.cuh jubjub_read)
//   S = read_scalar(sbar)                                 rejected when S >= r_J
//   [8](c vk + R - S P_G) == O                            P_G = find_group_hash(b"r", "Zcash_PH") (redjubjub_consts.inc)
// c vk - S P_G comes out of one doubling chain over the 252 bits of c and S: each step doubles, then adds one of
// {O, vk, -P_G, vk - P_G} picked by the two bits, so every thread of a warp runs the same instructions.  All four table
// points are affine and carried as (y - x, y + x, 2d x y), which makes each addition 7 Fr products; vk - P_G is made affine
// with one inversion.  ~251 x 8 + 252 x 7 products for the chain, plus two Point::reads (~1 k each).
//
// Everything is inlined into the kernel (redjubjub.cu), like jubjub.cuh.  Thread-local arrays are only ever indexed with
// compile-time constants (the BLAKE2b rounds are unrolled, the scalar bits are shifted out of the top word), so nothing
// goes to local memory.  The same source compiles with ZK_HOST_EMUL for the CPU test (tests/host_emul/emul_redjubjub.cpp).
#pragma once
#include "jubjub.cuh"

namespace zkrj {
using namespace zkjj;

enum Verdict : uint8_t { RJ_BAD_EQUATION = 0, RJ_OK = 1, RJ_BAD_VK = 2, RJ_BAD_R = 3, RJ_BAD_S = 4 };

#include "redjubjub_consts.inc"

// ---- Fs: the Jubjub scalar field, r_J = 0x0e7db4ea...d6f72cb7 (fs.rs:14), 252 bits, R = 2^256 -------------------------
#ifndef ZK_HOST_EMUL
static __device__ __constant__ uint32_t ZK_FS_MOD[8] = {0xd6f72cb7u, 0xd0970e5eu, 0xccc81082u, 0xa6682093u,
                                                        0x01343b00u, 0x06673b01u, 0x6533afa9u, 0x0e7db4eau};
#endif
struct FsParams {
    static constexpr int N = 8;
    static constexpr uint32_t INV = 0xef788ef9u;   // -r_J^-1 mod 2^32
#ifndef ZK_HOST_EMUL
    ZK_DEV static uint32_t modc(int i) { return ZK_FS_MOD[i]; }
#else
    ZK_DEV static uint32_t modc(int i) { return mod(i); }
#endif
    ZK_DEV static constexpr uint32_t mod(int i) {
        constexpr uint32_t m[8] = {0xd6f72cb7u, 0xd0970e5eu, 0xccc81082u, 0xa6682093u, 0x01343b00u, 0x06673b01u, 0x6533afa9u, 0x0e7db4eau};
        return m[i];
    }
    ZK_DEV static constexpr uint32_t one(int i) {   // 2^256 mod r_J
        constexpr uint32_t m[8] = {0xb99607d9u, 0x25f80bb3u, 0x66b6e750u, 0xf315d62fu, 0xeb8814f4u, 0x932514eeu, 0x479155c6u, 0x09a6fc6fu};
        return m[i];
    }
    ZK_DEV static constexpr uint32_t r2(int i) {    // 2^512 mod r_J
        constexpr uint32_t m[8] = {0x95e57731u, 0x67719aa4u, 0x9ce3fc26u, 0x51b0cef0u, 0xc026e9a5u, 0x69dab7fau, 0x8d127688u, 0x04f6547bu};
        return m[i];
    }
};
typedef Fp<FsParams> Fs;

// Fs::to_uniform of a 64-byte digest given as 8 little-endian u64 words: lo + hi 2^256 mod r_J, returned as the canonical
// integer.  Two Montgomery products: (2^256 mod r_J) * lo = lo mod r_J and (2^512 mod r_J) * hi = hi 2^256 mod r_J.
// lo and hi are not reduced (they run up to 2^256 - 1 > 17 r_J), which is safe because each is the operand whose words
// are fed in one per row: with the left operand a < r_J < 2^252 every row adds less than 2^285 to a total that stays below
// 2^255, so the N + 1 accumulator words never overflow, and the result (a b + m r_J) / 2^256 < 2 r_J is brought below r_J by
// the final conditional subtraction.  The host-emulation test covers the all-ones digest.
ZK_DEV Fs fs_to_uniform(const uint64_t *d) {
    Fs lo, hi, one = Fs::one(), r2;
#pragma unroll
    for (int i = 0; i < 4; i++) {
        lo.l[2 * i] = (uint32_t)d[i]; lo.l[2 * i + 1] = (uint32_t)(d[i] >> 32);
        hi.l[2 * i] = (uint32_t)d[4 + i]; hi.l[2 * i + 1] = (uint32_t)(d[4 + i] >> 32);
    }
#pragma unroll
    for (int i = 0; i < 8; i++) r2.l[i] = FsParams::r2(i);
    return one * lo + r2 * hi;
}

// ---- BLAKE2b-512 (RFC 7693) with an empty key and salt and a 16-byte personalization --------------------------------
ZK_DEV constexpr uint64_t b2b_iv(int i) {
    constexpr uint64_t v[8] = {0x6a09e667f3bcc908ull, 0xbb67ae8584caa73bull, 0x3c6ef372fe94f82bull, 0xa54ff53a5f1d36f1ull,
                               0x510e527fade682d1ull, 0x9b05688c2b3e6c1full, 0x1f83d9abfb41bd6bull, 0x5be0cd19137e2179ull};
    return v[i];
}
ZK_DEV constexpr int b2b_sigma(int r, int i) {   // rounds 10 and 11 reuse the permutations of rounds 0 and 1
    constexpr uint8_t s[10][16] = {{0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15}, {14, 10, 4, 8, 9, 15, 13, 6, 1, 12, 0, 2, 11, 7, 5, 3},
                                   {11, 8, 12, 0, 5, 2, 15, 13, 10, 14, 3, 6, 7, 1, 9, 4}, {7, 9, 3, 1, 13, 12, 11, 14, 2, 6, 5, 10, 4, 0, 15, 8},
                                   {9, 0, 5, 7, 2, 4, 10, 15, 14, 1, 11, 12, 6, 8, 3, 13}, {2, 12, 6, 10, 0, 11, 8, 3, 4, 13, 7, 5, 15, 14, 1, 9},
                                   {12, 5, 1, 15, 14, 13, 4, 10, 0, 7, 6, 3, 9, 2, 8, 11}, {13, 11, 7, 14, 12, 1, 3, 9, 5, 0, 15, 4, 8, 6, 2, 10},
                                   {6, 15, 14, 9, 11, 3, 0, 8, 12, 2, 13, 7, 1, 4, 10, 5}, {10, 2, 8, 4, 7, 6, 1, 5, 15, 11, 9, 14, 3, 12, 13, 0}};
    return s[r % 10][i];
}
// "Zcash_RedJubjubH" as two little-endian words (redjubjub.rs:25)
constexpr uint64_t RJ_PERSONAL0 = 0x65525f687361635aull, RJ_PERSONAL1 = 0x4862756a62754a64ull;

// the 64-bit words compile to pairs of 32-bit registers: adds to add / addc, rotations to funnel shifts (by 32: a swap)
ZK_DEV uint64_t rotr64(uint64_t x, int n) { return (x >> n) | (x << (64 - n)); }
ZK_DEV void b2b_g(uint64_t &a, uint64_t &b, uint64_t &c, uint64_t &d, uint64_t x, uint64_t y) {
    a = a + b + x; d = rotr64(d ^ a, 32); c = c + d; b = rotr64(b ^ c, 24);
    a = a + b + y; d = rotr64(d ^ a, 16); c = c + d; b = rotr64(b ^ c, 63);
}
// F(h, m, t, last): all 12 rounds unrolled, so each m[sigma(r, i)] names a register
ZK_DEV void b2b_compress(uint64_t *h, const uint64_t *m, uint64_t t, bool last) {
    uint64_t v[16];
#pragma unroll
    for (int i = 0; i < 8; i++) { v[i] = h[i]; v[i + 8] = b2b_iv(i); }
    v[12] ^= t;                                   // the high word of the counter stays 0 (messages < 2^64 bytes)
    if (last) v[14] = ~v[14];
#pragma unroll
    for (int r = 0; r < 12; r++) {
        b2b_g(v[0], v[4], v[8], v[12], m[b2b_sigma(r, 0)], m[b2b_sigma(r, 1)]);
        b2b_g(v[1], v[5], v[9], v[13], m[b2b_sigma(r, 2)], m[b2b_sigma(r, 3)]);
        b2b_g(v[2], v[6], v[10], v[14], m[b2b_sigma(r, 4)], m[b2b_sigma(r, 5)]);
        b2b_g(v[3], v[7], v[11], v[15], m[b2b_sigma(r, 6)], m[b2b_sigma(r, 7)]);
        b2b_g(v[0], v[5], v[10], v[15], m[b2b_sigma(r, 8)], m[b2b_sigma(r, 9)]);
        b2b_g(v[1], v[6], v[11], v[12], m[b2b_sigma(r, 10)], m[b2b_sigma(r, 11)]);
        b2b_g(v[2], v[7], v[8], v[13], m[b2b_sigma(r, 12)], m[b2b_sigma(r, 13)]);
        b2b_g(v[3], v[4], v[9], v[14], m[b2b_sigma(r, 14)], m[b2b_sigma(r, 15)]);
    }
#pragma unroll
    for (int i = 0; i < 8; i++) h[i] ^= v[i] ^ v[i + 8];
}
// bytes [off, off + 8) of msg as a little-endian word, zero past mlen (byte loads: msg may start at any address)
ZK_DEV uint64_t msg_word(const uint8_t *msg, uint64_t mlen, uint64_t off) {
    uint64_t w = 0;
#pragma unroll
    for (int k = 0; k < 8; k++)
        if (off + k < mlen) w |= (uint64_t)msg[off + k] << (8 * k);
    return w;
}
// H*(rbar || msg) before the reduction: the 64-byte BLAKE2b digest as 8 little-endian words.  rbar: 4 little-endian words.
ZK_DEV void h_star_digest(const uint64_t *rbar, const uint8_t *msg, uint64_t mlen, uint64_t *h) {
#pragma unroll
    for (int i = 0; i < 8; i++) h[i] = b2b_iv(i);
    h[0] ^= 0x01010040ull;                        // digest length 64, key length 0, fanout 1, depth 1
    h[6] ^= RJ_PERSONAL0;
    h[7] ^= RJ_PERSONAL1;
    const uint64_t len = 32 + mlen, nblocks = (len + 127) / 128;
    for (uint64_t b = 0; b < nblocks; b++) {
        uint64_t m[16];
#pragma unroll
        for (int w = 0; w < 16; w++) m[w] = (b == 0 && w < 4) ? rbar[w & 3] : msg_word(msg, mlen, 128 * b + 8 * w - 32);
        const bool last = b + 1 == nblocks;
        b2b_compress(h, m, last ? len : 128 * (b + 1), last);
    }
}

// ---- the verification equation ----------------------------------------------------------------------------------------
struct Niels { Fr ymx, ypx, kt; };    // an affine point as (y - x, y + x, 2d x y)

ZK_DEV Niels niels_identity() { Niels q; q.ymx = Fr::one(); q.ypx = Fr::one(); q.kt = Fr::zero(); return q; }
ZK_DEV Niels niels_of(const Fr &x, const Fr &y, const Fr &d2) { Niels q; q.ymx = y - x; q.ypx = y + x; q.kt = x * y * d2; return q; }
ZK_DEV Niels niels_neg_pg() {
    Niels q;
#pragma unroll
    for (int i = 0; i < 8; i++) { q.ymx.l[i] = RJ_NEG_PG[0][i]; q.ypx.l[i] = RJ_NEG_PG[1][i]; q.kt.l[i] = RJ_NEG_PG[2][i]; }
    return q;
}
ZK_DEV Niels niels_select(bool c, const Niels &a, const Niels &b) {   // c ? a : b, without a branch
    Niels r;
#pragma unroll
    for (int i = 0; i < 8; i++) {
        r.ymx.l[i] = c ? a.ymx.l[i] : b.ymx.l[i];
        r.ypx.l[i] = c ? a.ypx.l[i] : b.ypx.l[i];
        r.kt.l[i] = c ? a.kt.l[i] : b.kt.l[i];
    }
    return r;
}
// add-2008-hwcd-3 (a = -1) with Z2 = 1 and the second operand's terms precomputed: 7 products
ZK_DEV Ext ext_madd(const Ext &p, const Niels &q) {
    Fr a = (p.y - p.x) * q.ymx;
    Fr b = (p.y + p.x) * q.ypx;
    Fr c = p.t * q.kt;
    Fr d = p.z.dbl();
    Fr e = b - a, f = d - c, g = d + c, h = b + a;
    Ext r;
    r.x = e * f; r.y = g * h; r.t = e * h; r.z = f * g;
    return r;
}
ZK_DEV void shl1(uint32_t *w) {
#pragma unroll
    for (int i = 7; i > 0; i--) w[i] = (w[i] << 1) | (w[i - 1] >> 31);
    w[0] <<= 1;
}

// PublicKey::try_from(vk) + PublicKey::verify(msg, sig, Diversifier) for one signature.  vk: 8 little-endian words;
// sig: 16 (rbar then sbar).  Returns the Verdict; when several checks fail, the first in the reference's order wins.
ZK_DEV int redjubjub_verify(const uint32_t *vk, const uint32_t *sig, const uint8_t *msg, uint64_t mlen) {
    uint32_t cw[8];
    {
        uint64_t rbar[4], dg[8];
#pragma unroll
        for (int i = 0; i < 4; i++) rbar[i] = (uint64_t)sig[2 * i] | ((uint64_t)sig[2 * i + 1] << 32);
        h_star_digest(rbar, msg, mlen, dg);
        const Fs c = fs_to_uniform(dg);
#pragma unroll
        for (int i = 0; i < 8; i++) cw[i] = c.l[i];
    }
    Ext a, r;
    if (jubjub_read(vk, a) != JJ_OK) return RJ_BAD_VK;
    if (jubjub_read(sig, r) != JJ_OK) return RJ_BAD_R;
    uint32_t sw[8];
    Fs s;
#pragma unroll
    for (int i = 0; i < 8; i++) sw[i] = s.l[i] = sig[8 + i];
    if (!Fs::canonical_lt_mod(s)) return RJ_BAD_S;

    const Fr d2 = jj_d2();
    const Niels nvk = niels_of(a.x, a.y, d2), npg = niels_neg_pg();
    Niels nboth;
    {
        Ext t = ext_madd(a, npg);                 // vk - P_G, made affine
        const Fr zi = t.z.inverse();
        nboth = niels_of(t.x * zi, t.y * zi, d2);
    }
    // c, S < r_J < 2^252: shift bit 251 up to bit 255, then take the top bits one at a time
#pragma unroll
    for (int i = 7; i > 0; i--) { cw[i] = (cw[i] << 4) | (cw[i - 1] >> 28); sw[i] = (sw[i] << 4) | (sw[i - 1] >> 28); }
    cw[0] <<= 4; sw[0] <<= 4;
    Ext acc = ext_identity();
#pragma unroll 1
    for (int i = 0; i < 252; i++) {
        if (i) acc = ext_dbl(acc);
        const bool bc = cw[7] >> 31, bs = sw[7] >> 31;
        shl1(cw); shl1(sw);
        const Niels q = niels_select(bc, niels_select(bs, nboth, nvk), niels_select(bs, npg, niels_identity()));
        acc = ext_madd(acc, q);
    }
    acc = ext_madd(acc, niels_of(r.x, r.y, d2));   // + R
    acc = ext_dbl(ext_dbl(ext_dbl(acc)));          // mul_by_cofactor
    return ext_is_identity(acc) ? RJ_OK : RJ_BAD_EQUATION;
}

}  // namespace zkrj
