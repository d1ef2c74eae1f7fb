// Confidential-transfer balance updates of one block: what modules/encrypted-balances runs around each proof check.
//
// Restates the module's per-transaction loop (modules/encrypted-balances/src/lib.rs:25-96, 133-222) over a block:
//   rollover(sender), rollover(recipient)   at an account's first touch, when it is due: balance = (balance or zero) +
//                                           (pending or zero), present; pending absent
//   balance_sender                          the stored balance, or Ciphertext::zero() when absent (what the verifier reads)
//   sub_enc_balance                         applied transactions: balance -= (amount_sender + fee_sender, 2 randomness);
//                                           an absent balance stays absent (and_then)
//   add_pending_transfer                    applied transactions: pending(recipient) = (pending or nothing) +
//                                           (amount_recipient, randomness)
// Every ciphertext operation of the reference reads its points again (Point::read + as_prime_order) and writes the result
// (core/primitives/src/ciphertext.rs:81-100).  Here each point is read once, the arithmetic stays in extended coordinates,
// and each output is written once.  The epoch is fixed for the block, so an account's rollover comes before all of its
// in-block changes, and pending additions are never rolled inside the block.  Per account, then:
//   balance at transaction k = rolled balance - sum of its earlier applied sends
//   final pending            = rolled (or untouched) pending + sum of its applied receives
// The group law is associative and commutative and Point::write is canonical, so a segmented scan over the transactions
// grouped by account gives the sequential loop's bytes.
//
// The pipeline (balances.cu), one function here per thread of each pass:
//   bal_touch          keys of the two elements of each transaction (send: sender, receive: n_accounts + recipient) and
//                      the touched accounts
//   bal_decode         Point::read + as_prime_order of every transaction point and every touched account's ciphertexts
//   bal_tx             status and the (left, right) deltas of each transaction
//   bal_account        the rollover of each touched account
//   bal_radix_*        stable LSD radix sort of the elements by key (element ids are 2 k + kind, so the order inside a
//                      key is the transaction order)
//   bal_scan_*         segmented exclusive scan of the deltas in sorted order, BAL_SCAN_CHUNK elements per thread and
//                      level; the chunk aggregates are scanned the same way, level by level, so a chain may span any
//                      number of thread blocks
//   bal_tx_points / bal_acct_points   the projective outputs
//   bal_encode_chunk   Point::write of BAL_ENC_CHUNK points with one inversion (Montgomery's trick)
//   bal_finish_*       the output bytes
// Point state is passed through global memory between passes and held in registers inside them; nothing is indexed at
// run time in a thread-local array, so nothing goes to local memory.  The same source compiles with ZK_HOST_EMUL for the
// CPU test (tests/host_emul/emul_balances.cpp).
#pragma once
#include <stddef.h>
#include "elgamal.cuh"

namespace zkbal {
using namespace zkjj;
using zkeg::eg_read_prime_order;
using zkeg::ext_select;
using zkeg::load_le_words;

enum TxStatus : uint8_t { BAL_APPLIED = 0, BAL_NOT_APPLIED = 1, BAL_BAD_POINT = 2, BAL_BAD_INDEX = 3 };
constexpr uint8_t ACCT_BALANCE = 1, ACCT_PENDING = 2, ACCT_DUE = 4;
constexpr uint32_t BAL_MAX = 1u << 22;          // limit of n_tx and of n_accounts
constexpr int BAL_SCAN_CHUNK = 8;               // elements per thread and level of the scan
constexpr int BAL_ENC_CHUNK = 8;                // points per inversion
constexpr int BAL_SORT_TILE = 64;               // elements per thread of a radix pass
constexpr int BAL_RADIX_BITS = 8;
constexpr uint32_t BAL_RADIX = 1u << BAL_RADIX_BITS;

struct Pair { Ext l, r; };                      // a ciphertext (left, right)

ZK_DEV Pair pair_identity() { Pair p; p.l = ext_identity(); p.r = ext_identity(); return p; }
ZK_DEV Pair pair_add(const Pair &a, const Pair &b, const Fr &d2) { Pair s; s.l = ext_add(a.l, b.l, d2); s.r = ext_add(a.r, b.r, d2); return s; }
ZK_DEV Ext ext_neg(const Ext &p) { Ext q = p; q.x = p.x.neg(); q.t = p.t.neg(); return q; }
ZK_DEV Pair pair_sub(const Pair &a, const Pair &b, const Fr &d2) {
    Pair s; s.l = ext_add(a.l, ext_neg(b.l), d2); s.r = ext_add(a.r, ext_neg(b.r), d2); return s;
}
ZK_DEV Pair pair_select(bool c, const Pair &a, const Pair &b) {   // c ? a : b, without a branch
    Pair r; r.l = ext_select(c, a.l, b.l); r.r = ext_select(c, a.r, b.r); return r;
}

// A touched account whose stored ciphertext fails to read is reported in one word that holds the complement of the lowest
// such account: 0 (what the context's error words are cleared to) means none, and atomicMax keeps the lowest account.
ZK_DEV void bal_report_bad(uint32_t *bad, uint32_t a) {
#ifdef ZK_HOST_EMUL
    if (~a > *bad) *bad = ~a;
#else
    atomicMax(bad, ~a);
#endif
}

// ---- 1. keys and touched accounts --------------------------------------------------------------------------------------
// Element 2 k (the send) has key sender, element 2 k + 1 (the receive) n_accounts + recipient.  A transaction with an
// index out of range touches nothing: both its elements get the key 2 n_accounts, past every account.
ZK_DEV void bal_touch(size_t k, uint32_t n_acct, const uint32_t *sender, const uint32_t *recipient, uint32_t *keys, uint8_t *touched) {
    const uint32_t s = sender[k], r = recipient[k];
    const bool ok = s < n_acct && r < n_acct;
    keys[2 * k] = ok ? s : 2 * n_acct;
    keys[2 * k + 1] = ok ? n_acct + r : 2 * n_acct;
    if (ok) { touched[s] = 1; touched[r] = 1; }
}

// ---- 2. decoding -------------------------------------------------------------------------------------------------------
// Point p: p < 4 n_tx is transaction point p (amount_sender | amount_recipient | fee_sender | randomness); else point
// q = p - 4 n_tx is account q / 4's balance left / right (q % 4 = 0, 1) or pending left / right (2, 3), read only when the
// account is touched and the ciphertext present.  dec[p] = the point (the identity when not read), ok[p] = it read.
ZK_DEV void bal_decode(size_t p, size_t n_tx, const uint8_t *tx_points, const uint8_t *balances, const uint8_t *pendings,
                       const uint8_t *flags, const uint8_t *touched, Ext *dec, uint8_t *ok) {
    const uint8_t *src = nullptr;
    if (p < 4 * n_tx) {
        src = tx_points + 32 * p;
    } else {
        const size_t q = p - 4 * n_tx, a = q >> 2;
        const uint32_t j = (uint32_t)(q & 3);
        if (touched[a] && (flags[a] & (j < 2 ? ACCT_BALANCE : ACCT_PENDING)))
            src = (j < 2 ? balances : pendings) + 64 * a + 32 * (j & 1);
    }
    Ext pt = ext_identity();
    bool good = true;
    if (src) {
        uint32_t e[8];
        load_le_words(src, e);
        Ext r;
        good = eg_read_prime_order(e, r);
        if (good) pt = r;
    }
    dec[p] = pt;
    ok[p] = good;
}

// ---- 3. transactions ---------------------------------------------------------------------------------------------------
// Status (an index out of range first, then a rejected point, then the mask) and the deltas: delta[2 k] = the send
// (amount_sender + fee_sender, 2 randomness), delta[2 k + 1] = the receive (amount_recipient, randomness); the identity
// unless the transaction is applied.  recv_any[recipient] = 1 for an applied transaction.
ZK_DEV void bal_tx(size_t k, uint32_t n_acct, const uint32_t *sender, const uint32_t *recipient, const uint8_t *applied,
                   const Ext *dec, const uint8_t *ok, Pair *delta, uint8_t *status, uint8_t *recv_any) {
    const uint32_t s = sender[k], r = recipient[k];
    uint8_t st;
    if (s >= n_acct || r >= n_acct) st = BAL_BAD_INDEX;
    else if (!(ok[4 * k] && ok[4 * k + 1] && ok[4 * k + 2] && ok[4 * k + 3])) st = BAL_BAD_POINT;
    else st = applied[k] ? BAL_APPLIED : BAL_NOT_APPLIED;
    status[k] = st;
    Pair send = pair_identity(), recv = pair_identity();
    if (st == BAL_APPLIED) {
        const Fr d2 = jj_d2();
        const Ext rnd = dec[4 * k + 3];
        send.l = ext_add(dec[4 * k], dec[4 * k + 2], d2);
        send.r = ext_dbl(rnd);
        recv.l = dec[4 * k + 1];
        recv.r = rnd;
        recv_any[r] = 1;
    }
    delta[2 * k] = send;
    delta[2 * k + 1] = recv;
}

// ---- 4. rollover -------------------------------------------------------------------------------------------------------
// For touched account a: roll_b / roll_p = its balance and pending after the rollover, rflags[a] = which of them are
// present.  A stored ciphertext that fails to read is reported in *bad (bal_report_bad).
ZK_DEV void bal_account(size_t a, size_t n_tx, const uint8_t *flags, const uint8_t *touched, const Ext *dec, const uint8_t *ok,
                        Pair *roll_b, Pair *roll_p, uint8_t *rflags, uint32_t *bad) {
    if (!touched[a]) return;
    const size_t base = 4 * n_tx + 4 * a;
    if (!(ok[base] && ok[base + 1] && ok[base + 2] && ok[base + 3])) bal_report_bad(bad, (uint32_t)a);
    const uint8_t f = flags[a];
    Pair b, p;
    b.l = dec[base]; b.r = dec[base + 1];
    p.l = dec[base + 2]; p.r = dec[base + 3];
    if (f & ACCT_DUE) {
        roll_b[a] = pair_add(b, p, jj_d2());
        roll_p[a] = pair_identity();
        rflags[a] = ACCT_BALANCE;
    } else {
        roll_b[a] = b;
        roll_p[a] = p;
        rflags[a] = f & (ACCT_BALANCE | ACCT_PENDING);
    }
}

// ---- 5. stable radix sort of the elements by key -----------------------------------------------------------------------
// Pass over digit (key >> shift) & (BAL_RADIX - 1).  Thread t owns the elements [t BAL_SORT_TILE, (t + 1) BAL_SORT_TILE)
// and walks them in order, so the scatter keeps the order inside a digit.  hist: [digit][tile], zero before the count;
// its exclusive prefix sum is the cursor array of the scatter.  vals_in NULL: the element ids 0 .. n - 1.
ZK_DEV void bal_radix_hist(size_t t, size_t n, const uint32_t *keys, int shift, size_t n_tiles, uint32_t *hist) {
    const size_t i1 = (t + 1) * BAL_SORT_TILE < n ? (t + 1) * BAL_SORT_TILE : n;
    for (size_t i = t * BAL_SORT_TILE; i < i1; i++) hist[(size_t)((keys[i] >> shift) & (BAL_RADIX - 1)) * n_tiles + t]++;
}
ZK_DEV void bal_radix_scatter(size_t t, size_t n, const uint32_t *keys_in, const uint32_t *vals_in, int shift, size_t n_tiles,
                              uint32_t *cursor, uint32_t *keys_out, uint32_t *vals_out) {
    const size_t i1 = (t + 1) * BAL_SORT_TILE < n ? (t + 1) * BAL_SORT_TILE : n;
    for (size_t i = t * BAL_SORT_TILE; i < i1; i++) {
        const uint32_t key = keys_in[i];
        const uint32_t pos = cursor[(size_t)((key >> shift) & (BAL_RADIX - 1)) * n_tiles + t]++;
        keys_out[pos] = key;
        vals_out[pos] = vals_in ? vals_in[i] : (uint32_t)i;
    }
}

// ---- 6. segmented exclusive scan ---------------------------------------------------------------------------------------
// Level 0: the deltas in sorted order, v[idx[j]], with head[j] = 1 where a key starts.  Level l + 1: one item per chunk of
// level l, its aggregate (the sum from the chunk's last head, or the whole chunk) with head = the chunk holds a head.
ZK_DEV void bal_heads(size_t j, const uint32_t *keys, uint8_t *head) { head[j] = j == 0 || keys[j] != keys[j - 1]; }

ZK_DEV void bal_scan_up(size_t c, size_t n, const Pair *v, const uint32_t *idx, const uint8_t *head, Pair *agg, uint8_t *agg_head) {
    const Fr d2 = jj_d2();
    const size_t j1 = (c + 1) * BAL_SCAN_CHUNK < n ? (c + 1) * BAL_SCAN_CHUNK : n;
    Pair acc = pair_identity();
    uint8_t h = 0;
#pragma unroll 1
    for (size_t j = c * BAL_SCAN_CHUNK; j < j1; j++) {
        const bool hj = head[j];
        acc = pair_add(pair_select(hj, pair_identity(), acc), v[idx ? idx[j] : j], d2);
        h |= hj;
    }
    agg[c] = acc;
    agg_head[c] = h;
}
// out[j] = the sum of the items before j back to their segment's start.  carry: the level above's out (NULL: the identity).
// elements: a head starts its own segment (level 0); above, a head item's aggregate restarts the sum after it.
ZK_DEV void bal_scan_down(size_t c, size_t n, const Pair *v, const uint32_t *idx, const uint8_t *head, const Pair *carry, bool elements,
                          Pair *out) {
    const Fr d2 = jj_d2();
    const size_t j1 = (c + 1) * BAL_SCAN_CHUNK < n ? (c + 1) * BAL_SCAN_CHUNK : n;
    Pair run = carry ? carry[c] : pair_identity();
#pragma unroll 1
    for (size_t j = c * BAL_SCAN_CHUNK; j < j1; j++) {
        const bool hj = head[j];
        if (!elements) out[j] = run;
        run = pair_select(hj, pair_identity(), run);
        if (elements) out[j] = run;
        run = pair_add(run, v[idx ? idx[j] : j], d2);
    }
}

// ---- 7. outputs in projective form -------------------------------------------------------------------------------------
// Sorted element j.  A send writes its transaction's balance_sender and balance_after to pts[4 k .. 4 k + 4); the last
// element of a key writes the key's total to tot[key] and sets has[key].  The elements of a transaction with a bad index
// (key 2 n_accounts) write the identity for it.
ZK_DEV void bal_tx_points(size_t j, size_t n, uint32_t n_acct, const uint32_t *keys, const uint32_t *vals, const Pair *excl,
                          const Pair *delta, const Pair *roll_b, const uint8_t *rflags, const uint8_t *status, Ext *pts, Pair *tot,
                          uint8_t *has) {
    const uint32_t key = keys[j], e = vals[j];
    const size_t k = e >> 1;
    const Fr d2 = jj_d2();
    if (key >= 2 * n_acct) {
        if (!(e & 1))
#pragma unroll 1
            for (int i = 0; i < 4; i++) pts[4 * k + i] = ext_identity();
        return;
    }
    const bool send = !(e & 1), last = j + 1 == n || keys[j + 1] != key;
    const bool present = rflags[key < n_acct ? key : key - n_acct] & ACCT_BALANCE, applied = status[k] == BAL_APPLIED;
    // the left points, then the right ones: one Ext at a time keeps the live state small
#pragma unroll 1
    for (int h = 0; h < 2; h++) {
        const Ext x = (&excl[j].l)[h], d = (&delta[e].l)[h];
        if (send) {
            const Ext bs = present ? ext_add((&roll_b[key].l)[h], ext_neg(x), d2) : ext_identity();
            pts[4 * k + h] = bs;
            pts[4 * k + 2 + h] = present && applied ? ext_add(bs, ext_neg(d), d2) : ext_identity();
        }
        if (last) (&tot[key].l)[h] = ext_add(x, d, d2);
    }
    if (last) has[key] = 1;
}
// Account a's final balance and pending, at pts[4 n_tx + 4 a ..], and which are present (present[a]).  Every point of
// pts is written (the identity where there is nothing to encode), so that every Z of an encoding chunk is nonzero.
ZK_DEV void bal_acct_points(size_t a, size_t n_tx, uint32_t n_acct, const uint8_t *touched, const Pair *roll_b, const Pair *roll_p,
                            const uint8_t *rflags, const Pair *tot, const uint8_t *has, const uint8_t *recv_any, Ext *pts, uint8_t *present) {
    const size_t base = 4 * n_tx + 4 * a;
    if (!touched[a]) {
#pragma unroll 1
        for (int i = 0; i < 4; i++) pts[base + i] = ext_identity();
        return;
    }
    const Fr d2 = jj_d2();
    const uint8_t pr = rflags[a] | (recv_any[a] ? ACCT_PENDING : 0);
    const bool sent = has[a], received = has[n_acct + a];
#pragma unroll 1
    for (int h = 0; h < 2; h++) {
        Ext b = (&roll_b[a].l)[h];
        if (sent) b = ext_add(b, ext_neg((&tot[a].l)[h]), d2);
        pts[base + h] = pr & ACCT_BALANCE ? b : ext_identity();
        Ext p = (&roll_p[a].l)[h];
        if (received) p = ext_add(p, (&tot[n_acct + a].l)[h], d2);
        pts[base + 2 + h] = p;
    }
    present[a] = pr;
}

// ---- 8. Point::write with one inversion per chunk ----------------------------------------------------------------------
// Points [c BAL_ENC_CHUNK, ..) of pts to enc (8 words each).  The forward pass keeps the running product of the Z's in
// prefix; the backward pass turns it into each Z's inverse.
ZK_DEV void bal_encode_chunk(size_t c, size_t n, const Ext *pts, Fr *prefix, uint32_t *enc) {
    const size_t i0 = c * BAL_ENC_CHUNK;
    if (i0 >= n) return;
    const uint32_t cnt = n - i0 < BAL_ENC_CHUNK ? (uint32_t)(n - i0) : BAL_ENC_CHUNK;
    Fr acc = Fr::one();
#pragma unroll 1
    for (uint32_t j = 0; j < cnt; j++) {
        acc = acc * pts[i0 + j].z;
        prefix[i0 + j] = acc;
    }
    Fr inv = acc.inverse();
#pragma unroll 1
    for (uint32_t j = cnt; j-- > 0;) {
        const Ext *p = pts + i0 + j;
        const Fr zi = j ? prefix[i0 + j - 1] * inv : inv;
        inv = inv * p->z;
        jubjub_encode(p->x * zi, p->y * zi, enc + 8 * (i0 + j));
    }
}

// ---- 9. output bytes ---------------------------------------------------------------------------------------------------
// byte stores: device pointers passed in by the caller need not be word aligned
ZK_DEV void store_le_words(const uint32_t *w, size_t n_words, uint8_t *b) {
#pragma unroll 1
    for (size_t i = 0; i < n_words; i++)
#pragma unroll
        for (int k = 0; k < 4; k++) b[4 * i + k] = (uint8_t)(w[i] >> (8 * k));
}
ZK_DEV void bal_finish_tx(size_t k, const uint8_t *status, const uint32_t *enc, uint8_t *balance_sender, uint8_t *balance_after) {
    store_le_words(enc + 32 * k, 16, balance_sender + 64 * k);
    if (status[k] == BAL_APPLIED) store_le_words(enc + 32 * k + 16, 16, balance_after + 64 * k);
}
// Untouched accounts are copied through byte for byte.  A touched account's absent ciphertexts are written as zero bytes;
// its flags keep bits 3-7 and get the new presence bits, with bit 2 (due) cleared.
ZK_DEV void bal_finish_acct(size_t a, size_t n_tx, const uint8_t *touched, const uint8_t *balances, const uint8_t *pendings,
                            const uint8_t *flags, const uint8_t *present, const uint32_t *enc, uint8_t *new_balances,
                            uint8_t *new_pendings, uint8_t *new_flags) {
    if (!touched[a]) {
#pragma unroll 1
        for (int i = 0; i < 64; i++) { new_balances[64 * a + i] = balances[64 * a + i]; new_pendings[64 * a + i] = pendings[64 * a + i]; }
        new_flags[a] = flags[a];
        return;
    }
    const uint8_t pr = present[a];
    const uint32_t *e = enc + 8 * (4 * n_tx + 4 * a);
    if (pr & ACCT_BALANCE) store_le_words(e, 16, new_balances + 64 * a);
    else for (int i = 0; i < 64; i++) new_balances[64 * a + i] = 0;
    if (pr & ACCT_PENDING) store_le_words(e + 16, 16, new_pendings + 64 * a);
    else for (int i = 0; i < 64; i++) new_pendings[64 * a + i] = 0;
    new_flags[a] = (uint8_t)((flags[a] & ~(ACCT_BALANCE | ACCT_PENDING | ACCT_DUE)) | pr);
}

}  // namespace zkbal
