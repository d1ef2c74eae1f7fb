// CPU unit-test harness of the PRODUCT's transaction-building header (zero_chain_b200/csrc/tx_build.cuh) compiled with
// ZK_HOST_EMUL: BLAKE2s, the window tables, key derivation, GEpoch::group_hash, the confidential fields and signing, each
// in the layout of its zk_*_batch call, checked against the Python oracle by tests/test_host_emul_tx_build.py.  Test
// infrastructure only — never linked into libzkb200.so.
#define ZK_HOST_EMUL 1
#include "tx_build.cuh"
#include <string.h>

using namespace zktb;

extern "C" {
// BLAKE2s-256 of len bytes with the 8-byte personalization pers
void emu_tb_blake2s(const uint8_t *pers, const uint8_t *msg, uint32_t len, uint8_t *out) {
    uint32_t p[2], h[8];
    memcpy(p, pers, 8);
    b2s_256(p[0], p[1], len, [&](uint32_t k) {
        uint32_t w = 0;
        for (uint32_t b = 0; b < 4; b++)
            if (4 * k + b < len) w |= (uint32_t)msg[4 * k + b] << (8 * b);
        return w;
    }, h);
    memcpy(out, h, 32);
}
// the committed P_G window table, and the table tb_epoch_entry builds for the encoding g (a prime-order point)
void emu_tb_pg_table(uint32_t *out) { memcpy(out, TB_PG_TABLE, sizeof(TB_PG_TABLE)); }
int emu_tb_epoch_table(const uint8_t *g, uint32_t *out) {
    uint32_t enc[8];
    memcpy(enc, g, 32);
    Ext p;
    const int st = read_prime_order(enc, p);
    if (st != JJ_OK) return st;
    for (int e = 0; e < TB_WINDOWS * TB_DIGITS; e++) tb_epoch_entry(p, e, out + TB_ENTRY_WORDS * e);
    return JJ_OK;
}
void emu_tb_keys(size_t n, const uint8_t *seeds, const uint64_t *off, uint8_t *sks, uint8_t *dks, uint8_t *eks) {
    for (size_t i = 0; i < n; i++) {
        const Fs sk = spending_key(seeds + off[i], off[i + 1] - off[i]);
        const Fs dk = decryption_key(sk);
        uint32_t ek[8];
        ext_encode(pg_mul(dk), ek);
        memcpy(sks + 32 * i, sk.l, 32); memcpy(dks + 32 * i, dk.l, 32); memcpy(eks + 32 * i, ek, 32);
    }
}
// 1 and the tag byte, or 0
int emu_tb_g_epoch(uint32_t epoch, uint8_t *out, uint32_t *tag) {
    uint32_t enc[8];
    if (!g_epoch_hash(epoch, enc, *tag)) return 0;
    memcpy(out, enc, 32);
    return 1;
}
void emu_tb_fields(size_t n, const uint8_t *sks, const uint8_t *eks, const uint32_t *amounts, const uint32_t *fees, const uint8_t *rs,
                   const uint8_t *alphas, const uint8_t *g_epoch, uint8_t *fields, uint8_t *rsks, uint8_t *dks, uint8_t *status) {
    uint32_t sk[8], ek[8], r[8], al[8], scratch[28 * 8];
    static uint32_t table[TB_TABLE_WORDS];
    if (emu_tb_epoch_table(g_epoch, table) != JJ_OK) return;
    for (size_t i = 0; i < n; i++) {
        memcpy(sk, sks + 32 * i, 32); memcpy(ek, eks + 32 * i, 32); memcpy(r, rs + 32 * i, 32); memcpy(al, alphas + 32 * i, 32);
        status[i] = (uint8_t)confidential_fields(sk, ek, amounts[i], fees[i], r, al, g_epoch, table, scratch, 1, fields + 32 * TB_N_FIELDS * i,
                                                 rsks + 32 * i, dks + 32 * i);
    }
}
void emu_tb_sign(size_t n, const uint8_t *sks, const uint8_t *ts, const uint8_t *msgs, const uint64_t *off, uint8_t *sigs) {
    for (size_t i = 0; i < n; i++) {
        uint32_t sk[8], sig[16];
        uint64_t t[10];
        memcpy(sk, sks + 32 * i, 32);
        memcpy(t, ts + 80 * i, 80);
        redjubjub_sign(fs_words(sk), t, msgs + off[i], off[i + 1] - off[i], sig);
        memcpy(sigs + 64 * i, sig, 64);
    }
}
}
