/* TEST INFRASTRUCTURE (oracle) — the extrinsic loop of modules/encrypted-assets in plain C99, one transaction after another
 * on one core, the way the runtime applies a block's extrinsics.  Not part of the product; the tests and
 * tools/assets_bench.py build it through tests/jubjub_oracle/assets_coracle.py.
 *
 * It builds on the confidential-transfer oracle (balances_oracle.c, included as it is): the byte-level ciphertext operations
 * and the rollover.  The storage is the slot arrays of zk_assets_block, updated in place; the statuses, the outputs and the
 * failing-slot rule are that call's (tests/jubjub_oracle/assets.py states them). */
#include "balances_oracle.c"

/* Returns -1, or the first slot (in touch order) whose stored ciphertext does not read; nb / np / nf hold the state on
 * entry and on return.  seen: n_slots bytes of scratch.  balance_after, event_ct and event_flags are written only where
 * zk_assets_block writes them. */
EXPORT long long ao_block(size_t n_slots, uint8_t *nb, uint8_t *np, uint8_t *nf, uint8_t *seen, size_t n_tx, const uint8_t *kind,
                          const uint32_t *slot_a, const uint32_t *slot_b, const uint8_t *tx_points, const uint8_t *applied,
                          uint8_t *balance_sender, uint8_t *balance_after, uint8_t *event_ct, uint8_t *event_flags, uint8_t *status) {
    memset(seen, 0, n_slots);
    for (size_t k = 0; k < n_tx; k++) {
        const uint8_t kd = kind[k];
        const uint32_t a = slot_a[k], b = slot_b[k], who[2] = {a, b};
        const uint8_t *pt = tx_points + 128 * k;
        if (kd > 2 || a >= n_slots || (kd == 0 && b >= n_slots)) {
            if (kd == 0) memcpy(balance_sender + 64 * k, CT_ZERO, 64);
            else memset(balance_sender + 64 * k, 0, 64);
            status[k] = 3;
            continue;
        }
        for (int w = 0; w < (kd == 0 ? 2 : 1); w++) {
            const uint32_t s = who[w];
            if (!seen[s]) {
                seen[s] = 1;
                if (((nf[s] & 1) && !ct_read_ok(nb + 64 * s)) || ((nf[s] & 2) && !ct_read_ok(np + 64 * s))) return s;
            }
        }
        ext_t q;
        if (kd == 0) {                                     /* confidential_transfer (lib.rs:86-164) */
            for (int w = 0; w < 2; w++) {
                const uint32_t s = who[w];
                if (nf[s] & 4) {                           /* rollover (lib.rs:266-306) */
                    const uint8_t *pend = nf[s] & 2 ? np + 64 * s : CT_ZERO;
                    if (nf[s] & 1) { if (ct_op(nb + 64 * s, pend, 1, nb + 64 * s)) return s; }
                    else memcpy(nb + 64 * s, pend, 64);
                    memset(np + 64 * s, 0, 64);
                    nf[s] = (uint8_t)((nf[s] & ~6) | 1);
                }
            }
            memcpy(balance_sender + 64 * k, nf[a] & 1 ? nb + 64 * a : CT_ZERO, 64);
            int bad = 0;
            for (int i = 0; i < 4; i++) bad |= read_prime(pt + 32 * i, &q);
            if (bad) { status[k] = 2; continue; }
            if (applied[k] != 1) { status[k] = 1; continue; }
            uint8_t amount[64], fee[64], apf[64], recv[64];
            memcpy(amount, pt, 32); memcpy(amount + 32, pt + 96, 32);
            memcpy(fee, pt + 64, 32); memcpy(fee + 32, pt + 96, 32);
            memcpy(recv, pt + 32, 32); memcpy(recv + 32, pt + 96, 32);
            ct_op(amount, fee, 1, apf);
            if (nf[a] & 1) ct_op(nb + 64 * a, apf, -1, nb + 64 * a);
            if (nf[b] & 2) ct_op(np + 64 * b, recv, 1, np + 64 * b);
            else { memcpy(np + 64 * b, recv, 64); nf[b] |= 2; }
            memcpy(balance_after + 64 * k, nf[a] & 1 ? nb + 64 * a : CT_ZERO, 64);
            status[k] = 0;
            continue;
        }
        memset(balance_sender + 64 * k, 0, 64);
        if (kd == 1) {                                     /* issue (lib.rs:32-83) */
            if (read_prime(pt, &q) || read_prime(pt + 96, &q)) { status[k] = 2; continue; }
            if (applied[k] != 1) { status[k] = 1; continue; }
            uint8_t total[64];
            memcpy(total, pt, 32); memcpy(total + 32, pt + 96, 32);
            ct_op(total, CT_ZERO, 1, nb + 64 * a);         /* from_left_right: both halves read, then written */
            nf[a] |= 1;
            memcpy(event_ct + 128 * k, nb + 64 * a, 64);
            memset(event_ct + 128 * k + 64, 0, 64);
            event_flags[k] = 1;
        } else {                                           /* destroy (lib.rs:167-215) */
            if (applied[k] != 1) { status[k] = 1; continue; }
            for (int w = 0; w < 2; w++) {
                uint8_t *src = (w ? np : nb) + 64 * a;
                if (nf[a] & (1 << w)) memcpy(event_ct + 128 * k + 64 * w, src, 64);
                else memset(event_ct + 128 * k + 64 * w, 0, 64);
                memset(src, 0, 64);
            }
            event_flags[k] = nf[a] & 3;
            nf[a] &= (uint8_t)~3;
        }
        status[k] = 0;
    }
    /* a named slot's absent ciphertexts are zero bytes */
    for (size_t s = 0; s < n_slots; s++) {
        if (!seen[s]) continue;
        if (!(nf[s] & 1)) memset(nb + 64 * s, 0, 64);
        if (!(nf[s] & 2)) memset(np + 64 * s, 0, 64);
    }
    return -1;
}
