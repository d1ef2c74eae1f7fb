/* TEST INFRASTRUCTURE (oracle) — the anonymous_transfer loop of modules/anonymous-balances in plain C99, one transaction
 * after another on one core, the way the runtime applies a block's extrinsics.  Not part of the product; the tests and
 * tools/anon_balances_bench.py build it through tests/jubjub_oracle/anon_coracle.py.
 *
 * It builds on the confidential-transfer oracle (balances_oracle.c, included as it is): Point::read + as_prime_order, the
 * byte-level Ciphertext add and the failing-account rule.  The storage is the arrays of zk_balances_anonymous_block,
 * updated in place; the statuses and the outputs are that call's (tests/jubjub_oracle/anon_balances.py states them). */
#include "balances_oracle.c"

#define RING 12

/* Returns -1, or the first account (in touch order) whose stored ciphertext does not read; nb / np / nf hold the state
 * on entry and on return.  seen: n_acct bytes of scratch. */
EXPORT long long ao_block(size_t n_acct, const uint8_t *keys, uint8_t *nb, uint8_t *np, uint8_t *nf, uint8_t *seen, size_t n_tx,
                          const uint32_t *members, const uint8_t *tx_points, const uint8_t *tx_extra, const uint8_t *g_epoch,
                          const uint8_t *applied, uint8_t *enc_balances, uint8_t *verify_points, uint8_t *status) {
    memset(seen, 0, n_acct);
    for (size_t k = 0; k < n_tx; k++) {
        const uint32_t *mem = members + RING * k;
        const uint8_t *pt = tx_points + 32 * (RING + 1) * k;
        uint8_t *eb = enc_balances + 64 * RING * k, *vp = verify_points + 32 * (4 * RING + 4) * k;
        int in_range = 1;
        for (int i = 0; i < RING; i++) in_range &= mem[i] < n_acct;
        if (!in_range) {
            memset(eb, 0, 64 * RING);
            memset(vp, 0, 32 * (4 * RING + 4));
            status[k] = 3;
            continue;
        }
        for (int i = 0; i < RING; i++) {                       /* rollover(e) for each enc_key (lib.rs:169-206) */
            const uint32_t a = mem[i];
            if (!seen[a]) {
                seen[a] = 1;
                if (((nf[a] & 1) && !ct_read_ok(nb + 64 * a)) || ((nf[a] & 2) && !ct_read_ok(np + 64 * a))) return a;
            }
            if (nf[a] & 4) {
                const uint8_t *pend = nf[a] & 2 ? np + 64 * a : CT_ZERO;
                if (nf[a] & 1) { if (ct_op(nb + 64 * a, pend, 1, nb + 64 * a)) return a; }
                else memcpy(nb + 64 * a, pend, 64);
                memset(np + 64 * a, 0, 64);
                nf[a] = (uint8_t)((nf[a] & ~6) | 1);
            }
        }
        /* acc, and verify_anonymous_proof's pushes (zk-system/src/lib.rs:118-165) */
        for (int i = 0; i < RING; i++) {
            const uint32_t a = mem[i];
            memcpy(eb + 64 * i, nf[a] & 1 ? nb + 64 * a : CT_ZERO, 64);
            memcpy(vp + 32 * i, keys + 32 * a, 32);
            memcpy(vp + 32 * (RING + i), pt + 32 * i, 32);
            memcpy(vp + 32 * (2 * RING + i), eb + 64 * i, 32);
            memcpy(vp + 32 * (3 * RING + i), eb + 64 * i + 32, 32);
        }
        memcpy(vp + 32 * (4 * RING), pt + 32 * RING, 32);
        memcpy(vp + 32 * (4 * RING + 1), tx_extra + 64 * k, 32);
        memcpy(vp + 32 * (4 * RING + 2), g_epoch, 32);
        memcpy(vp + 32 * (4 * RING + 3), tx_extra + 64 * k + 32, 32);
        ext_t q;
        int bad = 0;
        for (int i = 0; i <= RING; i++) bad |= read_prime(pt + 32 * i, &q);
        if (bad) { status[k] = 2; continue; }
        if (applied[k] != 1) { status[k] = 1; continue; }
        for (int i = 0; i < RING; i++) {                       /* add_pending_transfer (lib.rs:209-232) */
            const uint32_t a = mem[i];
            uint8_t c[64];
            memcpy(c, pt + 32 * i, 32);
            memcpy(c + 32, pt + 32 * RING, 32);
            if (nf[a] & 2) ct_op(np + 64 * a, c, 1, np + 64 * a);
            else { memcpy(np + 64 * a, c, 64); nf[a] |= 2; }
        }
        status[k] = 0;
    }
    /* a touched account's absent ciphertexts are zero bytes */
    for (size_t a = 0; a < n_acct; a++) {
        if (!seen[a]) continue;
        if (!(nf[a] & 1)) memset(nb + 64 * a, 0, 64);
        if (!(nf[a] & 2)) memset(np + 64 * a, 0, 64);
    }
    return -1;
}
