// CPU unit-test harness of the PRODUCT's key-derivation functions in zero_chain_b200/csrc/hd_keys.cuh, compiled with
// ZK_HOST_EMUL: the hashes (the master hash, both 69-byte PRF messages, the 0x13 expansion, the 32-byte fingerprint), and
// whole rows run in the order zk_xsk_master_batch / zk_xsk_derive_batch / zk_xpgk_derive_batch run their passes (named
// parents, the parent pass, the row pass).  Checked against hashlib and the Python oracle by
// tests/test_host_emul_hd_keys.py.  Test infrastructure only — never linked into libzkb200.so.
#define ZK_HOST_EMUL 1
#include "hd_keys.cuh"
#include <string.h>
#include <vector>

using namespace zkhd;

static void words(const uint8_t *b, uint32_t *w) { hd_load(b, w); }
static void put64(uint8_t *out, const uint64_t *h, int n) {
    for (int i = 0; i < 8 * n; i++) out[i] = (uint8_t)(h[i / 8] >> (8 * (i % 8)));
}
static uint8_t *at(uint8_t *b, size_t i, int size) { return b ? b + (size_t)size * i : nullptr; }

extern "C" {
// the master sk and chain code of a seed
void emu_master_hash(const uint8_t *seed, uint64_t len, uint8_t *sk, uint8_t *chain) {
    uint32_t c[8];
    const Fs s = hd_master(seed, len, c);
    store_le_words(sk, s.l, 8);
    store_le_words(chain, c, 8);
}
// prf_expand_vec(c, [t, key, index LE]): the 64-byte digest
void emu_prf_child(const uint8_t *c, uint32_t t, const uint8_t *key, uint32_t index, uint8_t *out) {
    uint32_t cw[8], kw[8];
    uint64_t h[8];
    words(c, cw); words(key, kw);
    hd_prf_child(cw, t, kw, index, h);
    put64(out, h, 8);
}
// to_uniform(prf_expand(i_l, [0x13])) of the first 32 bytes of i (64 bytes)
void emu_tweak(const uint8_t *i, uint8_t *out) {
    uint64_t I[8];
    for (int k = 0; k < 8; k++) { I[k] = 0; for (int b = 0; b < 8; b++) I[k] |= (uint64_t)i[8 * k + b] << (8 * b); }
    const Fs t = hd_tweak(I);
    store_le_words(out, t.l, 8);
}
uint32_t emu_tag(const uint8_t *pgk) {
    uint32_t w[8];
    words(pgk, w);
    return hd_tag(w);
}

void emu_master(size_t n, const uint8_t *seeds, const uint64_t *off, uint8_t *xsks, uint8_t *xpgks, uint8_t *dks, uint8_t *eks) {
    for (size_t i = 0; i < n; i++)
        xsk_master(seeds + off[i], off[i + 1] - off[i], xsks + HD_XK_BYTES * i, at(xpgks, i, HD_XK_BYTES), at(dks, i, 32), at(eks, i, 32));
}

// -1, or the lowest named parent whose sk >= r_J (its rows unwritten)
long long emu_xsk_derive(size_t n_parents, const uint8_t *parents, size_t n, const uint32_t *pidx, const uint32_t *cidx, uint8_t *xsks,
                         uint8_t *xpgks, uint8_t *dks, uint8_t *eks, uint8_t *status) {
    std::vector<uint8_t> named(n_parents + 1, 0), pstatus(n_parents + 1, 0xEE);
    std::vector<uint32_t> penc(8 * n_parents + 8), ptag(n_parents + 1);
    for (size_t i = 0; i < n; i++)
        if (pidx[i] < n_parents) named[pidx[i]] = 1;
    long long bad = -1;
    for (size_t p = 0; p < n_parents; p++) {
        if (!named[p]) continue;
        uint32_t tag = 0;
        pstatus[p] = !xsk_parent(parents + HD_XK_BYTES * p, penc.data() + 8 * p, tag);
        ptag[p] = tag;
        if (pstatus[p] && bad < 0) bad = (long long)p;
    }
    for (size_t i = 0; i < n; i++) {
        const int st = xsk_row(parents, n_parents, pidx[i], cidx[i], penc.data(), ptag.data(), pstatus.data(), xsks + HD_XK_BYTES * i,
                               at(xpgks, i, HD_XK_BYTES), at(dks, i, 32), at(eks, i, 32));
        if (st >= 0) status[i] = (uint8_t)st;
    }
    return bad;
}

void emu_xpgk_derive(size_t n_parents, const uint8_t *parents, size_t n, const uint32_t *pidx, const uint32_t *cidx, uint8_t *xpgks,
                     uint8_t *dks, uint8_t *eks, uint8_t *status) {
    std::vector<uint8_t> named(n_parents + 1, 0), pstatus(n_parents + 1, 0xEE);
    std::vector<uint32_t> penc(8 * n_parents + 8), ptag(n_parents + 1), pniels(TB_ENTRY_WORDS * (n_parents + 1));
    for (size_t i = 0; i < n; i++)
        if (pidx[i] < n_parents) named[pidx[i]] = 1;
    for (size_t p = 0; p < n_parents; p++) {
        if (!named[p]) continue;
        uint32_t tag = 0;
        pstatus[p] = (uint8_t)xpgk_parent(parents + HD_XK_BYTES * p, penc.data() + 8 * p, pniels.data() + TB_ENTRY_WORDS * p, tag);
        ptag[p] = tag;
    }
    for (size_t i = 0; i < n; i++)
        status[i] = (uint8_t)xpgk_row(parents, n_parents, pidx[i], cidx[i], penc.data(), ptag.data(), pniels.data(), pstatus.data(),
                                      xpgks + HD_XK_BYTES * i, at(dks, i, 32), at(eks, i, 32));
}
}
