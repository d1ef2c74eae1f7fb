/* TEST INFRASTRUCTURE (oracle) — the confidential-transfer loop of modules/encrypted-balances in plain C99, one transaction
 * after another on one core, the way the runtime applies a block's extrinsics.  Not part of the product; the tests and
 * tools/balances_bench.py build it through tests/jubjub_oracle/bal_coracle.py.
 *
 * It builds on the ElGamal oracle (elgamal_oracle.c, included as it is): Point::read + as_prime_order, the group law and
 * Point::write.  Every ciphertext operation works on bytes as core/primitives/src/ciphertext.rs:81-100 does: read both
 * operands, operate, write.  The storage is the arrays of zk_balances_confidential_block, updated in place; the statuses,
 * the outputs and the failing-account rule are that call's (tests/jubjub_oracle/balances.py states them). */
#include "elgamal_oracle.c"

/* Ciphertext::add (sign = 1) or sub (sign = -1) of 64-byte ciphertexts: 0 ok, 1 an operand does not read */
static int ct_op(const uint8_t *a, const uint8_t *b, int sign, uint8_t *out) {
    ext_t p[4];
    fr_t d2;
    jj_d2(&d2);
    for (int i = 0; i < 4; i++)
        if (read_prime(i < 2 ? a + 32 * i : b + 32 * (i - 2), &p[i])) return 1;
    for (int h = 0; h < 2; h++) {
        if (sign < 0) ext_neg(&p[2 + h], &p[2 + h]);
        ext_add(&p[h], &p[h], &p[2 + h], &d2);
    }
    ext_write(out, &p[0]);
    ext_write(out + 32, &p[1]);
    return 0;
}

static int ct_read_ok(const uint8_t *ct) {
    ext_t p;
    return !read_prime(ct, &p) && !read_prime(ct + 32, &p);
}

static const uint8_t CT_ZERO[64] = {1, [32] = 1};

/* Returns -1, or the first account (in touch order) whose stored ciphertext does not read; nb / np / nf hold the state
 * on entry and on return.  seen: n_acct bytes of scratch. */
EXPORT long long bo_block(size_t n_acct, uint8_t *nb, uint8_t *np, uint8_t *nf, uint8_t *seen, size_t n_tx, const uint32_t *sender,
                          const uint32_t *recipient, const uint8_t *tx_points, const uint8_t *applied, uint8_t *balance_sender,
                          uint8_t *balance_after, uint8_t *status) {
    memset(seen, 0, n_acct);
    for (size_t k = 0; k < n_tx; k++) {
        const uint32_t s = sender[k], r = recipient[k], who[2] = {s, r};
        const uint8_t *pt = tx_points + 128 * k;
        if (s >= n_acct || r >= n_acct) {
            memcpy(balance_sender + 64 * k, CT_ZERO, 64);
            status[k] = 3;
            continue;
        }
        for (int w = 0; w < 2; w++) {
            const uint32_t a = who[w];
            if (!seen[a]) {
                seen[a] = 1;
                if (((nf[a] & 1) && !ct_read_ok(nb + 64 * a)) || ((nf[a] & 2) && !ct_read_ok(np + 64 * a))) return a;
            }
            if (nf[a] & 4) {                                   /* rollover (lib.rs:133-172) */
                const uint8_t *pend = nf[a] & 2 ? np + 64 * a : CT_ZERO;
                if (nf[a] & 1) { if (ct_op(nb + 64 * a, pend, 1, nb + 64 * a)) return a; }
                else memcpy(nb + 64 * a, pend, 64);
                memset(np + 64 * a, 0, 64);
                nf[a] = (uint8_t)((nf[a] & ~6) | 1);
            }
        }
        memcpy(balance_sender + 64 * k, nf[s] & 1 ? nb + 64 * s : CT_ZERO, 64);
        ext_t q;
        int bad = 0;
        for (int i = 0; i < 4; i++) bad |= read_prime(pt + 32 * i, &q);
        if (bad) { status[k] = 2; continue; }
        if (!applied[k]) { status[k] = 1; continue; }
        /* sub_enc_balance (lib.rs:174-196): from_left_right, add, then sub when the balance is present */
        uint8_t amount[64], fee[64], apf[64], recv[64];
        memcpy(amount, pt, 32); memcpy(amount + 32, pt + 96, 32);
        memcpy(fee, pt + 64, 32); memcpy(fee + 32, pt + 96, 32);
        memcpy(recv, pt + 32, 32); memcpy(recv + 32, pt + 96, 32);
        ct_op(amount, fee, 1, apf);
        if (nf[s] & 1) ct_op(nb + 64 * s, apf, -1, nb + 64 * s);
        /* add_pending_transfer (lib.rs:198-222) */
        if (nf[r] & 2) ct_op(np + 64 * r, recv, 1, np + 64 * r);
        else { memcpy(np + 64 * r, recv, 64); nf[r] |= 2; }
        memcpy(balance_after + 64 * k, nf[s] & 1 ? nb + 64 * s : CT_ZERO, 64);
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
