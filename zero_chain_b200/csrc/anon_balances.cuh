// Anonymous-transfer state updates of one block: what modules/anonymous-balances runs around each proof check.
//
// Restates the module's per-transaction loop (modules/anonymous-balances/src/lib.rs:23-82, 169-232) over a block:
//   rollover(e) for the 12 ring members     at an account's first touch, when it is due: balance = (balance or zero) +
//                                           (pending or zero), present; pending absent
//   acc[i]                                  member i's stored balance, or Ciphertext::zero() when absent (what
//                                           verify_anonymous_proof reads, modules/zk-system/src/lib.rs:118-165)
//   add_pending_transfer                    applied transactions, each member i: pending(e_i) = (pending or nothing) +
//                                           from_left_right(left_i, right_ciphertext)
// A transfer changes pending balances only, and the epoch is fixed for the block, so an account's balance changes at its
// first touch only: what the verifier reads does not depend on any verdict, and an account's final pending is its rolled
// (or untouched) pending plus the (left, right) of every applied (transaction, member) entry that names it.  The group
// law is commutative and Point::write is canonical, so the sum in any order gives the sequential loop's bytes.
//
// The pipeline (anon_balances.cu), one function here or in balances.cuh per thread of each pass:
//   an_touch           the touched accounts (a transaction touches its members when all 12 indices are in range)
//   an_decode          Point::read + as_prime_order of the 13 transaction points (bal_decode for the accounts' ciphertexts)
//   an_tx              status, and the 12 entries of each transaction: key n_accounts + member and delta (left_i, right)
//                      when applied, else key 2 n_accounts and the identity
//   bal_account        the rollover of each touched account
//   zk_bal_sort / zk_bal_scan   balances.cu's radix sort of the entries by key and segmented scan of their deltas
//   an_totals          each key's total (its last element's exclusive sum plus its own delta) to tot[key]
//   bal_acct_points / bal_encode_chunk / bal_finish_acct   the rolled balance and final pending of each account, encoded
//                      once per account with one inversion per BAL_ENC_CHUNK points, and the new account table
//   an_finish_tx       the 52 public-input encodings of each transaction, and its 12 acc ciphertexts
// The entries' keys sit where balances.cuh keeps a confidential transfer's receives (n_accounts + account), so
// bal_acct_points adds each key's total to the pending of its account unchanged.  The same source compiles with
// ZK_HOST_EMUL for the CPU test (tests/host_emul/emul_anon_balances.cpp).
#pragma once
#include "balances.cuh"

namespace zkbal {

constexpr int AN_RING = 12;                     // ring members per transaction (core/proofs/src/constants.rs:1)
constexpr int AN_TX_POINTS = AN_RING + 1;       // left_ciphertexts[0..12) | right_ciphertext
constexpr int AN_VERIFY_POINTS = 4 * AN_RING + 4;
constexpr uint32_t AN_MAX_TX = 1u << 18;        // limit of n_tx (n_accounts: BAL_MAX)
constexpr uint8_t AN_TRANSFER = 0, AN_ISSUE = 1;  // kinds of zk_anonymous_calls_block
constexpr uint32_t AN_NONE = 0xFFFFFFFFu;       // no transaction (past every index below AN_MAX_TX)

// ---- 1. touched accounts -----------------------------------------------------------------------------------------------
ZK_DEV bool an_ring_ok(size_t k, uint32_t n_acct, const uint32_t *members) {
    bool ok = true;
#pragma unroll 1
    for (int i = 0; i < AN_RING; i++) ok &= members[AN_RING * k + i] < n_acct;
    return ok;
}
ZK_DEV void an_touch(size_t k, uint32_t n_acct, const uint32_t *members, uint8_t *touched) {
    if (!an_ring_ok(k, n_acct, members)) return;
#pragma unroll 1
    for (int i = 0; i < AN_RING; i++) touched[members[AN_RING * k + i]] = 1;
}

// ---- 2. decoding -------------------------------------------------------------------------------------------------------
// Point p < 13 n_tx: transaction point p; else the account ciphertexts as bal_decode reads them, at dec / ok + 13 n_tx.
// kind (NULL: every transaction a transfer): an issue reads its slots 0 (total) and 12 (randomness) only, a transaction of
// an unknown kind nothing; a point not read is the identity, with ok set.
ZK_DEV void an_decode(size_t p, size_t n_tx, const uint8_t *tx_points, const uint8_t *balances, const uint8_t *pendings,
                      const uint8_t *flags, const uint8_t *touched, Ext *dec, uint8_t *ok, const uint8_t *kind = nullptr) {
    const size_t ntp = AN_TX_POINTS * n_tx;
    if (p >= ntp) {
        bal_decode(p - ntp, 0, nullptr, balances, pendings, flags, touched, dec + ntp, ok + ntp);
        return;
    }
    if (kind) {
        const size_t k = p / AN_TX_POINTS;
        const size_t i = p - AN_TX_POINTS * k;
        if (kind[k] > AN_ISSUE || (kind[k] == AN_ISSUE && i != 0 && i != AN_RING)) {
            dec[p] = ext_identity();
            ok[p] = 1;
            return;
        }
    }
    uint32_t e[8];
    load_le_words(tx_points + 32 * p, e);
    Ext r;
    const bool good = eg_read_prime_order(e, r);
    dec[p] = good ? r : ext_identity();
    ok[p] = good;
}

// ---- 3. transactions ---------------------------------------------------------------------------------------------------
// Status (an index out of range first, then a rejected point, then the mask: applied[k] == 1 only), and the entries
// 12 k + i.  recv_any[member] = 1 for an applied transaction.
ZK_DEV void an_tx(size_t k, uint32_t n_acct, const uint32_t *members, const uint8_t *applied, const Ext *dec, const uint8_t *ok,
                  uint32_t *keys, Pair *delta, uint8_t *status, uint8_t *recv_any) {
    uint8_t st;
    if (!an_ring_ok(k, n_acct, members)) {
        st = BAL_BAD_INDEX;
    } else {
        bool good = true;
#pragma unroll 1
        for (int i = 0; i < AN_TX_POINTS; i++) good &= ok[AN_TX_POINTS * k + i] != 0;
        st = !good ? BAL_BAD_POINT : applied[k] == 1 ? BAL_APPLIED : BAL_NOT_APPLIED;
    }
    status[k] = st;
    const bool app = st == BAL_APPLIED;
    const Ext right = app ? dec[AN_TX_POINTS * k + AN_RING] : ext_identity();
#pragma unroll 1
    for (int i = 0; i < AN_RING; i++) {
        const size_t e = AN_RING * k + i;
        const uint32_t m = members[e];
        keys[e] = app ? n_acct + m : 2 * n_acct;
        Pair d;
        d.l = app ? dec[AN_TX_POINTS * k + i] : ext_identity();
        d.r = right;
        delta[e] = d;
        if (app) recv_any[m] = 1;
    }
}

// ---- 4. per-key totals -------------------------------------------------------------------------------------------------
// Sorted element j: the last element of a key below 2 n_accounts writes the key's total to tot[key] and sets has[key].
ZK_DEV void an_totals(size_t j, size_t n, uint32_t n_acct, const uint32_t *keys, const uint32_t *vals, const Pair *excl,
                      const Pair *delta, Pair *tot, uint8_t *has) {
    const uint32_t key = keys[j];
    if (key >= 2 * n_acct || (j + 1 < n && keys[j + 1] == key)) return;
    const Fr d2 = jj_d2();
    const uint32_t e = vals[j];
#pragma unroll 1
    for (int h = 0; h < 2; h++) (&tot[key].l)[h] = ext_add((&excl[j].l)[h], (&delta[e].l)[h], d2);
    has[key] = 1;
}

// ---- 5. the verifier's inputs ------------------------------------------------------------------------------------------
// Slot s = 52 k + q of verify_points, in verify_anonymous_proof's push order: q < 12 the EncKey of member q, < 24 left
// ciphertext q - 12, < 36 the left point of member (q - 24)'s rolled balance, < 48 the right point of member (q - 36)'s,
// then right_ciphertext, rvk, g_epoch, nonce.  The balance slots also write their half of the member's acc ciphertext to
// enc_balances.  acct_enc: the account encodings of bal_encode_chunk (account a's rolled balance at words 32 a .. 32 a +
// 16: the identity pair, Ciphertext::zero(), when absent).  A transaction with an index out of range gets zero rows.
ZK_DEV void copy_bytes(const uint8_t *src, uint8_t *dst, int n) {
#pragma unroll 1
    for (int i = 0; i < n; i++) dst[i] = src[i];
}
// kind / rd (NULL without issues, an_issue_read): an issue's and an unknown kind's rows are zero too, and a balance slot
// reads the pair at word rd[12 k + i] of the encodings in place of 32 member.
ZK_DEV void an_finish_slot(size_t s, const uint32_t *members, const uint8_t *status, const uint8_t *enc_keys, const uint8_t *tx_points,
                           const uint8_t *tx_extra, const uint8_t *g_epoch, const uint32_t *acct_enc, uint8_t *enc_balances,
                           uint8_t *verify_points, const uint8_t *kind = nullptr, const uint32_t *rd = nullptr) {
    const size_t k = s / AN_VERIFY_POINTS;
    const int q = (int)(s - AN_VERIFY_POINTS * k);
    uint8_t *out = verify_points + 32 * s;
    const bool bal_slot = q >= 2 * AN_RING && q < 4 * AN_RING;
    const int i = q < 3 * AN_RING ? q - 2 * AN_RING : q - 3 * AN_RING;       // the member of a balance slot
    uint8_t *acc = enc_balances + 64 * (AN_RING * k + i) + (q < 3 * AN_RING ? 0 : 32);
    if (status[k] == BAL_BAD_INDEX || (kind && kind[k] != AN_TRANSFER)) {
#pragma unroll 1
        for (int b = 0; b < 32; b++) out[b] = 0;
        if (bal_slot)
#pragma unroll 1
            for (int b = 0; b < 32; b++) acc[b] = 0;
        return;
    }
    if (bal_slot) {
        const size_t w = rd ? rd[AN_RING * k + i] : 32 * (size_t)members[AN_RING * k + i];
        store_le_words(acct_enc + w + (q < 3 * AN_RING ? 0 : 8), 8, out);
        copy_bytes(out, acc, 32);
        return;
    }
    const uint8_t *src;
    if (q < AN_RING) src = enc_keys + 32 * (size_t)members[AN_RING * k + q];
    else if (q < 2 * AN_RING) src = tx_points + 32 * (AN_TX_POINTS * k + (q - AN_RING));
    else if (q == 4 * AN_RING) src = tx_points + 32 * (AN_TX_POINTS * k + AN_RING);
    else if (q == 4 * AN_RING + 1) src = tx_extra + 64 * k;
    else if (q == 4 * AN_RING + 2) src = g_epoch;
    else src = tx_extra + 64 * k + 32;
    copy_bytes(src, out, 32);
}

// ---- 6. issue (zk_anonymous_calls_block) ------------------------------------------------------------------------------
// issue(issuer, total, .., randomness, ..) (lib.rs:87-134) sets the issuer's balance to (total, randomness) and touches
// nothing else: no rollover, the pending and the due bit stay.  An issue's verdict reads only its own fields, and a
// transfer changes pending balances only, so a block that mixes both still needs no rounds.  The applied issues are
// sorted by issuer (zk_bal_sort: in block order inside an issuer); for account a with first transfer touch t_a
//   rolled balance    (the last issue before t_a, else the stored balance) + (pending when due): an_issue_account
//   balance read by k the last issue after t_a and before k, else the rolled balance: an_issue_read
//   final balance     the last issue after t_a (any issue when no transfer touches a), else the rolled balance
// The issues' (total, randomness) pairs are encoded with the accounts, transaction k's at points 4 n_accounts + 2 k.
ZK_DEV void an_min(uint32_t *p, uint32_t v) {
#ifdef ZK_HOST_EMUL
    if (v < *p) *p = v;
#else
    atomicMin(p, v);
#endif
}
// the touched accounts as an_touch, for transfers only, and first[member] = the first transfer that names it (first: all
// AN_NONE before)
ZK_DEV void an_call_touch(size_t k, uint32_t n_acct, const uint8_t *kind, const uint32_t *members, uint8_t *touched, uint32_t *first) {
    if (kind[k] != AN_TRANSFER || !an_ring_ok(k, n_acct, members)) return;
#pragma unroll 1
    for (int i = 0; i < AN_RING; i++) {
        const uint32_t m = members[AN_RING * k + i];
        touched[m] = 1;
        an_min(first + m, (uint32_t)k);
    }
}
// A transfer as an_tx.  Otherwise the status (3 an unknown kind or an issuer out of range, 2 total or randomness rejected,
// then the mask), no entries (key 2 n_accounts), the issue's sort key ikeys[k] (the issuer when applied, else n_accounts)
// and its pair ipts[2 k], ipts[2 k + 1] (the identity unless applied).
ZK_DEV void an_call_tx(size_t k, uint32_t n_acct, const uint8_t *kind, const uint32_t *members, const uint8_t *applied, const Ext *dec,
                       const uint8_t *ok, uint32_t *keys, Pair *delta, uint8_t *status, uint8_t *recv_any, uint32_t *ikeys, Ext *ipts) {
    const size_t p = AN_TX_POINTS * k;
    bool app = false;
    if (kind[k] == AN_TRANSFER) {
        an_tx(k, n_acct, members, applied, dec, ok, keys, delta, status, recv_any);
    } else {
        const uint32_t a = members[AN_RING * k];
        const uint8_t st = kind[k] != AN_ISSUE || a >= n_acct ? BAL_BAD_INDEX
                           : !(ok[p] && ok[p + AN_RING]) ? BAL_BAD_POINT
                           : applied[k] == 1 ? BAL_APPLIED : BAL_NOT_APPLIED;
        status[k] = st;
#pragma unroll 1
        for (int i = 0; i < AN_RING; i++) {
            keys[AN_RING * k + i] = 2 * n_acct;
            delta[AN_RING * k + i] = pair_identity();
        }
        app = st == BAL_APPLIED;
    }
    ikeys[k] = app ? members[AN_RING * k] : n_acct;
    ipts[2 * k] = app ? dec[p] : ext_identity();
    ipts[2 * k + 1] = app ? dec[p + AN_RING] : ext_identity();
}
ZK_DEV size_t an_lower_bound(const uint32_t *v, size_t lo, size_t hi, uint32_t x) {
    while (lo < hi) {
        const size_t mid = (lo + hi) / 2;
        if (v[mid] < x) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}
// the last applied issue to account a before transaction k (AN_NONE: the last of all), or AN_NONE; ikeys / ivals: the
// sorted issue keys and their transaction indices
ZK_DEV uint32_t an_last_issue(const uint32_t *ikeys, const uint32_t *ivals, size_t n_tx, uint32_t a, uint32_t k) {
    const size_t lo = an_lower_bound(ikeys, 0, n_tx, a), hi = an_lower_bound(ikeys, lo, n_tx, a + 1);
    const size_t j = an_lower_bound(ivals, lo, hi, k);
    return j > lo ? ivals[j - 1] : AN_NONE;
}
// bal_account with the issue before the first touch as the base, and fin[a] = the issue that holds the final balance (or
// AN_NONE).  dec / ok: all of an_decode's points.
ZK_DEV void an_issue_account(size_t a, size_t n_tx, const uint8_t *flags, const uint8_t *touched, const uint32_t *first,
                             const uint32_t *ikeys, const uint32_t *ivals, const Ext *dec, const uint8_t *ok, Pair *roll_b, Pair *roll_p,
                             uint8_t *rflags, uint32_t *fin, uint32_t *bad) {
    const size_t ntp = AN_TX_POINTS * n_tx;
    const bool t = touched[a];
    const uint32_t t0 = t ? first[a] : AN_NONE;
    const uint32_t last = an_last_issue(ikeys, ivals, n_tx, (uint32_t)a, AN_NONE);
    fin[a] = last != AN_NONE && (!t || last > t0) ? last : AN_NONE;
    if (!t) return;
    bal_account(a, 0, flags, touched, dec + ntp, ok + ntp, roll_b, roll_p, rflags, bad);
    const uint32_t j = an_last_issue(ikeys, ivals, n_tx, (uint32_t)a, t0);
    if (j == AN_NONE) return;
    Pair b;
    b.l = dec[AN_TX_POINTS * (size_t)j];
    b.r = dec[AN_TX_POINTS * (size_t)j + AN_RING];
    if (flags[a] & ACCT_DUE) {
        Pair p;
        p.l = dec[ntp + 4 * a + 2];
        p.r = dec[ntp + 4 * a + 3];
        b = pair_add(b, p, jj_d2());
    }
    roll_b[a] = b;
    rflags[a] |= ACCT_BALANCE;
}
// Entry e = 12 k + i: rd[e] = the word of the encodings where the balance member i of transfer k reads starts: the last
// issue to it after its first touch and before k (32 n_accounts + 16 j), else its rolled balance (32 member).
ZK_DEV void an_issue_read(size_t e, uint32_t n_acct, size_t n_tx, const uint8_t *kind, const uint8_t *status, const uint32_t *members,
                          const uint32_t *first, const uint32_t *ikeys, const uint32_t *ivals, uint32_t *rd) {
    const size_t k = e / AN_RING;
    if (kind[k] != AN_TRANSFER || status[k] == BAL_BAD_INDEX) {
        rd[e] = 0;
        return;
    }
    const uint32_t m = members[e];
    const uint32_t j = an_last_issue(ikeys, ivals, n_tx, m, (uint32_t)k);
    rd[e] = j != AN_NONE && j > first[m] ? 32 * n_acct + 16 * j : 32 * m;
}
// the Issued event's ciphertext of an applied issue
ZK_DEV void an_issued(size_t k, uint32_t n_acct, const uint8_t *kind, const uint8_t *status, const uint32_t *enc, uint8_t *issued) {
    if (kind[k] == AN_ISSUE && status[k] == BAL_APPLIED) store_le_words(enc + 32 * (size_t)n_acct + 16 * k, 16, issued + 64 * k);
}
// bal_finish_acct, then an account whose final balance is an issue's gets its encoding and bit 0 (an account no transfer
// touches keeps its pending bytes and its other flags)
ZK_DEV void an_issue_finish_acct(size_t a, uint32_t n_acct, const uint8_t *touched, const uint8_t *balances, const uint8_t *pendings,
                                 const uint8_t *flags, const uint8_t *present, const uint32_t *fin, const uint32_t *enc,
                                 uint8_t *new_balances, uint8_t *new_pendings, uint8_t *new_flags) {
    bal_finish_acct(a, 0, touched, balances, pendings, flags, present, enc, new_balances, new_pendings, new_flags);
    const uint32_t j = fin[a];
    if (j == AN_NONE) return;
    store_le_words(enc + 32 * (size_t)n_acct + 16 * (size_t)j, 16, new_balances + 64 * a);
    new_flags[a] |= ACCT_BALANCE;
}

}  // namespace zkbal
