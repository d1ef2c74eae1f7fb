/* TEST INFRASTRUCTURE (oracle) — both calls of modules/anonymous-balances, anonymous_transfer and issue, in plain C99, one
 * transaction after another on one core, the way the runtime applies a block's extrinsics.  Not part of the product; the
 * tests and tools/anon_balances_bench.py build it through tests/jubjub_oracle/anon_issue_coracle.py.
 *
 * It includes the anonymous-transfer oracle (anon_balances_oracle.c, included as it is) and runs each stretch of
 * transfers between two issues through its ao_block; an issue (lib.rs:87-134) writes its issuer's balance in between.  The
 * storage is the arrays of zk_anonymous_calls_block, updated in place; the statuses and the outputs are that call's
 * (tests/jubjub_oracle/anon_issue.py states them). */
#include "anon_balances_oracle.c"

/* Returns -1, or the first account (in touch order) whose ciphertext stored before the block does not read; nb / np / nf
 * hold the state on entry and on return.  seen: n_acct bytes of scratch.  issued: written for applied issues only. */
EXPORT long long aio_block(size_t n_acct, const uint8_t *keys, uint8_t *nb, uint8_t *np, uint8_t *nf, uint8_t *seen, size_t n_tx,
                           const uint8_t *kind, const uint32_t *members, const uint8_t *tx_points, const uint8_t *tx_extra,
                           const uint8_t *g_epoch, const uint8_t *applied, uint8_t *enc_balances, uint8_t *verify_points, uint8_t *issued,
                           uint8_t *status) {
    /* the stored ciphertexts of every account a transfer touches must read, whatever an issue writes before the touch */
    memset(seen, 0, n_acct);
    for (size_t k = 0; k < n_tx; k++) {
        const uint32_t *mem = members + RING * k;
        int in_range = kind[k] == 0;
        for (int i = 0; i < RING; i++) in_range &= mem[i] < n_acct;
        for (int i = 0; in_range && i < RING; i++) {
            const uint32_t a = mem[i];
            if (seen[a]) continue;
            seen[a] = 1;
            if (((nf[a] & 1) && !ct_read_ok(nb + 64 * a)) || ((nf[a] & 2) && !ct_read_ok(np + 64 * a))) return a;
        }
    }
    size_t k0 = 0;                                              /* the start of the stretch of transfers */
    for (size_t k = 0; k <= n_tx; k++) {
        if (k < n_tx && kind[k] == 0) continue;
        if (k > k0) {
            long long bad = ao_block(n_acct, keys, nb, np, nf, seen, k - k0, members + RING * k0, tx_points + 32 * (RING + 1) * k0,
                                     tx_extra + 64 * k0, g_epoch, applied + k0, enc_balances + 64 * RING * k0,
                                     verify_points + 32 * (4 * RING + 4) * k0, status + k0);
            if (bad >= 0) return bad;
        }
        k0 = k + 1;
        if (k == n_tx) break;
        memset(enc_balances + 64 * RING * k, 0, 64 * RING);
        memset(verify_points + 32 * (4 * RING + 4) * k, 0, 32 * (4 * RING + 4));
        const uint32_t a = members[RING * k];
        const uint8_t *pt = tx_points + 32 * (RING + 1) * k;
        uint8_t ct[64];
        memcpy(ct, pt, 32);                                     /* total */
        memcpy(ct + 32, pt + 32 * RING, 32);                    /* randomness */
        if (kind[k] != 1 || a >= n_acct) { status[k] = 3; continue; }
        /* Ciphertext::from_left_right reads both points; adding Ciphertext::zero() writes them as Point::write does */
        if (!ct_read_ok(ct)) { status[k] = 2; continue; }
        if (applied[k] != 1) { status[k] = 1; continue; }
        ct_op(ct, CT_ZERO, 1, nb + 64 * a);                     /* EncryptedBalance::insert(issuer, total_ciphertext) */
        nf[a] |= 1;
        memcpy(issued + 64 * k, nb + 64 * a, 64);
        status[k] = 0;
    }
    return -1;
}
