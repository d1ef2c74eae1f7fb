// The verify / apply rounds of a block import (import.cu): zk_import_confidential_block and zk_import_assets_block.
//
// A transfer's proof is checked against the sender's balance at that transaction, and that balance depends on which of
// the sender's earlier transfers passed.  So every transfer starts undecided and counts as applied, and each round
//   1. runs the state pass (zk_balances_confidential_block / zk_assets_block) with the current mask,
//   2. compacts the undecided transfers (imp_flag, zk_bal_prefix_sum, imp_gather): their proofs, and their 11 verifier
//      points with slots 6-7 (balance_sender) taken from the state pass,
//   3. verifies the compacted rows (zk_groth16_verify_points_batch_device),
//   4. finds each chain's first failure (imp_fail: atomicMin over the failing rows) and decides every undecided transfer
//      up to and including it (imp_decide): the balances those read were exact.  The rest waits for the next round.
// A chain is the transfers of one key: the sender account, or the sender slot.  The undecided transfers of a chain are
// always a suffix of it, so "up to the first failure" is "k <= first_fail[key]".  A round without a failure decides every
// undecided transfer as passed, and its state pass is the final state; a round that leaves nothing undecided is followed
// by one last state pass.  Issues and destroys (zk_import_assets_block) carry the caller's verdicts from the start.
//
// zk_import_anonymous_block needs no rounds: an issue's proof reads only its own fields, and a transfer changes pending
// balances only, so nothing a proof is checked against depends on a transfer's verdict.  Its passes (section 5) are
//   1. imp_an_start: check each transaction's kind and indices, count issues and transfers, flag the issues;
//      zk_bal_prefix_sum turns the flags into each issue's compact row (a transfer's row is k - the issues before k),
//   2. imp_an_issue_row: each issue's 11 confidential points and its proof, verified with the confidential key,
//   3. imp_an_scatter: the issue verdicts into verdicts (transfers 0: not applied), then the state pass
//      (zk_anonymous_calls_block) with verdicts as the mask,
//   4. imp_an_gather: each transfer's 52 points from that pass and its proof, verified with the anonymous key,
//   5. imp_an_scatter: the transfer verdicts, then the state pass again.
// zk_import_asset_calls (section 6) puts the asset numbering and the slot resolution in front of zk_import_assets_block's
// rounds.  zk_import_block (section 7) runs the sections of all three pallets on one schedule, sharing the launches.
//
// Plain integer code, one function per item and thread of each pass; the same source compiles with ZK_HOST_EMUL for the
// CPU tests (tests/host_emul/emul_import.cpp, emul_import_anon.cpp, emul_import_assets.cpp), which run the passes as loops
// over the items.
#pragma once
#include <stddef.h>
#include <stdint.h>

#ifdef ZK_HOST_EMUL
#define ZK_IMP_DEV inline
#else
#define ZK_IMP_DEV __device__ __forceinline__
#endif

namespace zkimp {

constexpr uint8_t IMP_UNDECIDED = 0xFF;        // a transfer's verdict not known yet (the verifier's verdicts are 0..4)
constexpr uint32_t IMP_NONE = 0xFFFFFFFFu;
constexpr uint8_t IMP_TRANSFER = 0;            // zk_assets_block's kinds
constexpr uint8_t IMP_DESTROY = 2;
constexpr int IMP_POINTS = 11;                 // confidential_points: address_sender, address_recipient, amount_sender,
                                               // amount_recipient, randomness, fee_sender, balance_sender (2), rvk, g_epoch, nonce
constexpr int IMP_ROW = 32 * IMP_POINTS;       // bytes of a verifier row
constexpr int IMP_BS = 32 * 6;                 // offset of balance_sender in it
constexpr int IMP_WORDS = (IMP_ROW + 192) / 4; // 4-byte words of a row and a proof, gathered one per thread
// the counter block: read back by the host once per round
enum ImpCounter { IMP_FAILS = 0, IMP_LEFT = 1, IMP_BAD = 2, IMP_TRANSFERS = 3, IMP_COUNTERS = 4 };

ZK_IMP_DEV void imp_min(uint32_t *p, uint32_t v) {
#ifdef ZK_HOST_EMUL
    if (v < *p) *p = v;
#else
    atomicMin(p, v);
#endif
}
ZK_IMP_DEV void imp_inc(uint32_t *p) {
#ifdef ZK_HOST_EMUL
    ++*p;
#else
    atomicAdd(p, 1u);
#endif
}

// ---- 0. start ----------------------------------------------------------------------------------------------------------
// kind == NULL: every transaction is a transfer (the confidential block).  A transfer starts undecided and applied; its
// key_a (the chain key) and key_b must be < n_keys.  An issue or destroy takes fixed[k] as its verdict and is applied iff
// it is 1; an applied one's key_a must be < n_keys (a failed one touches nothing, whatever its slot).  Any fixed byte is
// taken as it is, IMP_UNDECIDED included: only a transfer is ever undecided (imp_undecided).  An unknown kind, or an index
// out of range, puts the lowest such transaction in cnt[IMP_BAD].  fixed and verdict may be the same array.
ZK_IMP_DEV void imp_start(size_t k, uint32_t n_keys, const uint8_t *kind, const uint32_t *key_a, const uint32_t *key_b,
                          const uint8_t *fixed, uint8_t *verdict, uint8_t *applied, uint32_t *cnt) {
    const uint8_t kd = kind ? kind[k] : IMP_TRANSFER;
    bool bad;
    if (kd == IMP_TRANSFER) {
        verdict[k] = IMP_UNDECIDED;
        applied[k] = 1;
        imp_inc(cnt + IMP_TRANSFERS);
        bad = key_a[k] >= n_keys || key_b[k] >= n_keys;
    } else {
        const uint8_t v = fixed[k];
        verdict[k] = v;
        applied[k] = v == 1;
        bad = kd > IMP_DESTROY || (v == 1 && key_a[k] >= n_keys);
    }
    if (bad) imp_min(cnt + IMP_BAD, (uint32_t)k);
}

// ---- 2. compaction -----------------------------------------------------------------------------------------------------
// A transfer's verdict byte holds IMP_UNDECIDED or the verifier's verdict; an issue's or destroy's holds the caller's byte,
// whatever it is, so the kind decides first.
ZK_IMP_DEV bool imp_undecided(size_t k, const uint8_t *kind, const uint8_t *verdict) {
    return (!kind || kind[k] == IMP_TRANSFER) && verdict[k] == IMP_UNDECIDED;
}
// flag[k] = 1 for an undecided transfer; zk_bal_prefix_sum turns the flags into each one's row of the round buffers
ZK_IMP_DEV void imp_flag(size_t k, const uint8_t *kind, const uint8_t *verdict, uint32_t *flag) { flag[k] = imp_undecided(k, kind, verdict); }

// Item i: word w = i % IMP_WORDS of transaction k = i / IMP_WORDS, when k is undecided: words [0, 88) are its verifier
// row, with bytes [192, 256) taken from balance_sender[k], words [88, 136) its proof, into row off + pos[k] of the round
// buffers (off: the section's first row in a launch shared with other sections).  Word 0 also records k as the
// section's row pos[k].  Byte copies: the caller's arrays need no alignment.
ZK_IMP_DEV void imp_gather(size_t i, const uint8_t *kind, const uint8_t *verdict, const uint32_t *pos, const uint8_t *rows, const uint8_t *proofs,
                           const uint8_t *balance_sender, uint32_t *idx, uint8_t *round_rows, uint8_t *round_proofs, size_t off = 0) {
    const size_t k = i / IMP_WORDS;
    const uint32_t w = (uint32_t)(i % IMP_WORDS);
    if (!imp_undecided(k, kind, verdict)) return;
    if (!w) idx[pos[k]] = (uint32_t)k;
    const size_t j = off + pos[k];
    const uint32_t o = 4 * w;
    const uint8_t *src;
    uint8_t *dst;
    if (o < IMP_ROW) {
        src = o >= IMP_BS && o < IMP_BS + 64 ? balance_sender + 64 * k + (o - IMP_BS) : rows + IMP_ROW * k + o;
        dst = round_rows + IMP_ROW * j + o;
    } else {
        src = proofs + 192 * k + (o - IMP_ROW);
        dst = round_proofs + 192 * j + (o - IMP_ROW);
    }
#pragma unroll
    for (int b = 0; b < 4; b++) dst[b] = src[b];
}

// the confidential state pass's tx_points (amount_sender | amount_recipient | fee_sender | randomness) from the rows:
// item i is word i % 32 of transaction i / 32, slots 2, 3, 5, 4
ZK_IMP_DEV void imp_tx_points(size_t i, const uint8_t *rows, uint8_t *tx_points) {
    const size_t k = i >> 5;
    const uint32_t w = (uint32_t)(i & 31), slot = w >> 3, from = slot < 2 ? 2 + slot : 7 - slot;
    const uint8_t *src = rows + IMP_ROW * k + 32 * from + 4 * (w & 7);
    uint8_t *dst = tx_points + 128 * k + 4 * w;
#pragma unroll
    for (int b = 0; b < 4; b++) dst[b] = src[b];
}

// ---- 4. decisions ------------------------------------------------------------------------------------------------------
// row j of the section's m: transaction idx[j] with verdict rv[off + j].  A failure lowers its chain's first_fail
// (IMP_NONE before the pass) and counts in cnt[IMP_FAILS].
ZK_IMP_DEV void imp_fail(size_t j, const uint32_t *idx, const uint32_t *key_a, const uint8_t *rv, uint32_t *first_fail, uint32_t *cnt,
                         size_t off = 0) {
    if (rv[off + j] == 1) return;
    const uint32_t k = idx[j];
    imp_min(first_fail + key_a[k], k);
    imp_inc(cnt + IMP_FAILS);
}
// after every imp_fail: a transaction at or before its chain's first failure takes its verdict, and is applied iff it
// passed; one after it stays undecided and applied, and counts in cnt[IMP_LEFT]
ZK_IMP_DEV void imp_decide(size_t j, const uint32_t *idx, const uint32_t *key_a, const uint8_t *rv, const uint32_t *first_fail,
                           uint8_t *verdict, uint8_t *applied, uint32_t *cnt, size_t off = 0) {
    const uint32_t k = idx[j];
    if (k <= first_fail[key_a[k]]) {
        verdict[k] = rv[off + j];
        applied[k] = rv[off + j] == 1;
    } else {
        imp_inc(cnt + IMP_LEFT);
    }
}

// ---- 5. zk_import_anonymous_block --------------------------------------------------------------------------------------
constexpr uint8_t IMP_AN_TRANSFER = 0, IMP_AN_ISSUE = 1;        // zk_anonymous_calls_block's kinds
constexpr int IMP_AN_RING = 12;
constexpr int IMP_AN_TX_POINTS = IMP_AN_RING + 1;               // left ciphertexts | right ciphertext
constexpr int IMP_AN_ROW = 32 * (4 * IMP_AN_RING + 4);          // bytes of a transfer's verifier row (52 points)
constexpr int IMP_AN_ISSUE_WORDS = (IMP_ROW + 192) / 4;         // an issue's row and proof, one 4-byte word per thread
constexpr int IMP_AN_WORDS = (IMP_AN_ROW + 192) / 4;            // a transfer's
constexpr int IMP_ISSUES = IMP_FAILS;                           // the counter block: issues in the slot the rounds count failures in

// kind == NULL: every transaction is a transfer.  A transfer's 12 members must be < n_acct; an issue's issuer (members[12 k])
// must be, and the block must have what an issue's verification reads (issues_ok: a confidential key and issue_fields).
// Any other kind is bad.  The lowest bad transaction goes to cnt[IMP_BAD]; flag[k] = 1 for an issue.
ZK_IMP_DEV void imp_an_start(size_t k, uint32_t n_acct, bool issues_ok, const uint8_t *kind, const uint32_t *members, uint32_t *flag,
                             uint32_t *cnt) {
    const uint8_t kd = kind ? kind[k] : IMP_AN_TRANSFER;
    const uint32_t *m = members + IMP_AN_RING * k;
    bool bad = false;
    if (kd == IMP_AN_TRANSFER) {
        for (int i = 0; i < IMP_AN_RING; i++) bad |= m[i] >= n_acct;
        imp_inc(cnt + IMP_TRANSFERS);
    } else if (kd == IMP_AN_ISSUE) {
        bad = !issues_ok || m[0] >= n_acct;
        imp_inc(cnt + IMP_ISSUES);
    } else {
        bad = true;
    }
    flag[k] = kd == IMP_AN_ISSUE;
    if (bad) imp_min(cnt + IMP_BAD, (uint32_t)k);
}

// Item i: word w = i % IMP_AN_ISSUE_WORDS of transaction k = i / IMP_AN_ISSUE_WORDS, when k is an issue; pos[k] is its row.
// Words [0, 88) are verify_confidential_proof's 11 points over (issuer, issuer, total, total, randomness, fee, balance, rvk,
// g_epoch, nonce): keys[issuer], tx_points slots 0 and 12, issue_fields (fee | balance), tx_extra (rvk | nonce) and g_epoch.
// Words [88, 136) are its proof.  Both go to row off + pos[k].  Byte copies: the caller's arrays need no alignment.
ZK_IMP_DEV void imp_an_issue_row(size_t i, const uint8_t *kind, const uint32_t *pos, const uint8_t *keys, const uint32_t *members,
                                 const uint8_t *tx_points, const uint8_t *issue_fields, const uint8_t *tx_extra, const uint8_t *g_epoch,
                                 const uint8_t *proofs, uint8_t *rows, uint8_t *round_proofs, size_t off = 0) {
    const size_t k = i / IMP_AN_ISSUE_WORDS;
    const uint32_t o = 4 * (uint32_t)(i % IMP_AN_ISSUE_WORDS);
    if (kind[k] != IMP_AN_ISSUE) return;
    const size_t j = off + pos[k];
    const uint8_t *src;
    uint8_t *dst;
    if (o < IMP_ROW) {
        const uint32_t slot = o / 32, b = o % 32;
        const uint8_t *tp = tx_points + 32 * IMP_AN_TX_POINTS * k;
        switch (slot) {
        case 0: case 1: src = keys + 32 * (size_t)members[IMP_AN_RING * k] + b; break;    // address_sender, address_recipient
        case 2: case 3: src = tp + b; break;                                               // total, twice
        case 4: src = tp + 32 * IMP_AN_RING + b; break;                                    // randomness
        case 5: case 6: case 7: src = issue_fields + 96 * k + (o - 32 * 5); break;         // fee, balance
        case 8: src = tx_extra + 64 * k + b; break;                                        // rvk
        case 9: src = g_epoch + b; break;
        default: src = tx_extra + 64 * k + 32 + b; break;                                  // nonce
        }
        dst = rows + IMP_ROW * j + o;
    } else {
        src = proofs + 192 * k + (o - IMP_ROW);
        dst = round_proofs + 192 * j + (o - IMP_ROW);
    }
#pragma unroll
    for (int b = 0; b < 4; b++) dst[b] = src[b];
}

// pos is the exclusive prefix sum of the flags "not a transfer" (an anonymous issue; an asset issue or destroy), so
// pos[k] is such a transaction's compact row and k - pos[k] a transfer's.
// issues: verdicts[k] = rv[off + pos[k]] at a non-transfer and 0 at a transfer (not applied in the first state pass);
// otherwise verdicts[k] = rv[off + k - pos[k]] at a transfer, the others unchanged.
ZK_IMP_DEV void imp_an_scatter(size_t k, bool issues, const uint8_t *kind, const uint32_t *pos, const uint8_t *rv, uint8_t *verdicts,
                               size_t off = 0) {
    const bool issue = kind[k] != IMP_AN_TRANSFER;
    if (issues)
        verdicts[k] = issue ? rv[off + pos[k]] : 0;
    else if (!issue)
        verdicts[k] = rv[off + k - pos[k]];
}

// Item i: word o / 4 of transaction k's row_bytes-byte row (src_rows) and 192-byte proof, when k is a non-transfer (issues)
// or a transfer (!issues): into compact row off + pos[k] or off + k - pos[k] of rows / round_proofs.
ZK_IMP_DEV void imp_compact(size_t i, uint32_t row_bytes, bool issues, const uint8_t *kind, const uint32_t *pos, const uint8_t *src_rows,
                            const uint8_t *proofs, uint8_t *rows, uint8_t *round_proofs, size_t off = 0) {
    const uint32_t words = (row_bytes + 192) / 4;
    const size_t k = i / words;
    const uint32_t o = 4 * (uint32_t)(i % words);
    if ((kind[k] != IMP_AN_TRANSFER) != issues) return;
    const size_t j = off + (issues ? pos[k] : k - pos[k]);
    const uint8_t *src;
    uint8_t *dst;
    if (o < row_bytes) {
        src = src_rows + (size_t)row_bytes * k + o;
        dst = rows + (size_t)row_bytes * j + o;
    } else {
        src = proofs + 192 * k + (o - row_bytes);
        dst = round_proofs + 192 * j + (o - row_bytes);
    }
#pragma unroll
    for (int b = 0; b < 4; b++) dst[b] = src[b];
}

// Item i: word w = i % IMP_AN_WORDS of transaction k = i / IMP_AN_WORDS, when k is a transfer: words [0, 416) are its 52
// points from the state pass's verify_points, words [416, 464) its proof, into row k - pos[k].
ZK_IMP_DEV void imp_an_gather(size_t i, const uint8_t *kind, const uint32_t *pos, const uint8_t *verify_points, const uint8_t *proofs,
                              uint8_t *rows, uint8_t *round_proofs) {
    imp_compact(i, IMP_AN_ROW, false, kind, pos, verify_points, proofs, rows, round_proofs);
}

// ---- 6. zk_import_asset_calls ------------------------------------------------------------------------------------------
// The passes in front of zk_import_assets_block's rounds, from the slot table as the module stores it and the extrinsic
// fields (import.cu's asset_calls_run):
//   1. imp_as_start: check each kind, flag the issues and destroys; imp_as_row_insert / imp_as_row_dup: the table's rows
//      into the hash table, and the lowest row whose key repeats an earlier row's.  The host reads the counter block.
//   2. zk_bal_prefix_sum + imp_compact: the issue and destroy rows and proofs, verified; imp_an_scatter: their verdicts.
//   3. imp_as_issue_flag + zk_bal_prefix_sum: each passing issue's number among them; imp_as_refs: its asset id, and the
//      (asset id, key) every transaction references at positions 2k (slot_a) and 2k + 1 (slot_b).
//   4. imp_as_ref_insert: the references into the hash table; imp_as_new + zk_bal_prefix_sum: each new key's row, in the
//      order of its first reference; imp_as_slot: slot_a / slot_b, and each new row's (id, key), zero ciphertexts and flags.
//      imp_as_tx_points: the state pass's tx_points.  The host reads the counter block again (new rows, id overflow).
// The hash table: open addressing with linear probing over `cap` uint32 entries, IMP_NONE when empty.  An entry holds a
// handle: r < n_slots is table row r, n_slots + p is reference p.  Inserting a handle whose key is present lowers the
// entry to the least handle of that key (imp_min), so once every insert is done the entry is the key's table row if it
// has one, and its first reference otherwise, whatever order the threads ran in.  Keys are compared in full.
constexpr uint8_t IMP_ISSUE = 1;
constexpr uint32_t IMP_ASSET_ID_MAX = 0xFFFFFFFFu;
// the counter block of zk_import_asset_calls: the issues and destroys, the new rows, and the lowest transaction with an
// unknown kind, table row repeating an earlier one, and passing issue whose id would pass IMP_ASSET_ID_MAX
enum ImpAsCounter { IMP_AS_FIXED = 0, IMP_AS_NEW = 1, IMP_AS_BAD = 2, IMP_AS_DUP = 3, IMP_AS_OVF = 4, IMP_AS_COUNTERS = 5 };

// the keys behind the handles: a table row's (slot_ids[r], slot_keys[r]); reference p's (ref_id[p], slot p & 1 of row p / 2)
struct ImpAsKeys {
    const uint32_t *slot_ids;
    const uint8_t *slot_keys;
    const uint32_t *ref_id;
    const uint8_t *rows;
    uint32_t n_slots;
};
ZK_IMP_DEV uint32_t imp_as_id(const ImpAsKeys &t, uint32_t h) { return h < t.n_slots ? t.slot_ids[h] : t.ref_id[h - t.n_slots]; }
ZK_IMP_DEV const uint8_t *imp_as_key(const ImpAsKeys &t, uint32_t h) {
    if (h < t.n_slots) return t.slot_keys + 32 * (size_t)h;
    const uint32_t p = h - t.n_slots;
    return t.rows + IMP_ROW * (size_t)(p >> 1) + 32 * (p & 1);
}
ZK_IMP_DEV bool imp_as_equal(const ImpAsKeys &t, uint32_t a, uint32_t b) {
    if (imp_as_id(t, a) != imp_as_id(t, b)) return false;
    const uint8_t *x = imp_as_key(t, a), *y = imp_as_key(t, b);
    uint32_t diff = 0;
    for (int i = 0; i < 32; i++) diff |= x[i] ^ y[i];
    return !diff;
}
// FNV-1a over the id's 4 little-endian bytes and the key's 32, then murmur3's finaliser
ZK_IMP_DEV uint32_t imp_as_hash(uint32_t id, const uint8_t *key) {
    uint32_t h = 2166136261u;
    for (int i = 0; i < 4; i++) h = (h ^ ((id >> (8 * i)) & 0xFF)) * 16777619u;
    for (int i = 0; i < 32; i++) h = (h ^ key[i]) * 16777619u;
    h ^= h >> 16; h *= 0x85ebca6bu; h ^= h >> 13; h *= 0xc2b2ae35u; h ^= h >> 16;
    return h;
}
// entries for n keys: a power of two, at most half full
inline size_t imp_as_capacity(size_t n) {
    size_t c = 64;
    while (c < 2 * n) c <<= 1;
    return c;
}
// The emulation build may override both, e.g. a constant hash and n + 1 entries put every key into one probe chain.
#ifndef ZK_IAS_HASH
#define ZK_IAS_HASH(id, key) imp_as_hash(id, key)
#endif
#ifndef ZK_IAS_CAPACITY
#define ZK_IAS_CAPACITY(n) imp_as_capacity(n)
#endif

ZK_IMP_DEV uint32_t imp_cas(uint32_t *p, uint32_t cmp, uint32_t v) {
#ifdef ZK_HOST_EMUL
    const uint32_t old = *p;
    if (old == cmp) *p = v;
    return old;
#else
    return atomicCAS(p, cmp, v);
#endif
}
ZK_IMP_DEV uint32_t imp_as_first(const ImpAsKeys &t, uint32_t h, uint32_t cap) {
    return (uint32_t)(ZK_IAS_HASH(imp_as_id(t, h), imp_as_key(t, h)) % cap);
}
// handle h into the table (cap > the number of distinct keys, so an empty entry is always ahead)
ZK_IMP_DEV void imp_as_insert(const ImpAsKeys &t, uint32_t h, uint32_t *table, uint32_t cap) {
    for (uint32_t e = imp_as_first(t, h, cap);; e = e + 1 == cap ? 0 : e + 1) {
        const uint32_t cur = imp_cas(table + e, IMP_NONE, h);
        if (cur == IMP_NONE) return;
        if (imp_as_equal(t, cur, h)) {
            imp_min(table + e, h);
            return;
        }
    }
}
// after every insert: the entry of h's key (IMP_NONE for a key never inserted)
ZK_IMP_DEV uint32_t imp_as_find(const ImpAsKeys &t, uint32_t h, const uint32_t *table, uint32_t cap) {
    for (uint32_t e = imp_as_first(t, h, cap);; e = e + 1 == cap ? 0 : e + 1) {
        const uint32_t cur = table[e];
        if (cur == IMP_NONE || imp_as_equal(t, cur, h)) return cur;
    }
}

// an unknown kind puts k in cnt[IMP_AS_BAD]; flag[k] = 1 for an issue or destroy, counted in cnt[IMP_AS_FIXED]
ZK_IMP_DEV void imp_as_start(size_t k, const uint8_t *kind, uint32_t *flag, uint32_t *cnt) {
    const uint8_t kd = kind[k];
    if (kd > IMP_DESTROY) imp_min(cnt + IMP_AS_BAD, (uint32_t)k);
    flag[k] = kd == IMP_ISSUE || kd == IMP_DESTROY;
    if (flag[k]) imp_inc(cnt + IMP_AS_FIXED);
}
ZK_IMP_DEV void imp_as_row_insert(size_t r, const ImpAsKeys &t, uint32_t *table, uint32_t cap) { imp_as_insert(t, (uint32_t)r, table, cap); }
// after every row insert: a row whose entry holds an earlier row repeats that row's key
ZK_IMP_DEV void imp_as_row_dup(size_t r, const ImpAsKeys &t, const uint32_t *table, uint32_t cap, uint32_t *cnt) {
    if (imp_as_find(t, (uint32_t)r, table, cap) != r) imp_min(cnt + IMP_AS_DUP, (uint32_t)r);
}

// flag[k] = 1 for a passing issue; zk_bal_prefix_sum turns the flags into the passing issues before k
ZK_IMP_DEV void imp_as_issue_flag(size_t k, const uint8_t *kind, const uint8_t *verdicts, uint32_t *flag) {
    flag[k] = kind[k] == IMP_ISSUE && verdicts[k] == 1;
}
// The references of transaction k and a passing issue's id, next_id + ipos[k]; one past IMP_ASSET_ID_MAX puts k in
// cnt[IMP_AS_OVF].  asset_ids[k] is that id at a passing issue and 0 elsewhere.  Reference 2k: a transfer's (asset_id,
// sender), a passing issue's (id, issuer), a passing destroy's (asset_id, owner); 2k + 1: a transfer's (asset_id,
// recipient).  ref_on[p] = 0 where there is none.
ZK_IMP_DEV void imp_as_refs(size_t k, uint32_t next_id, const uint8_t *kind, const uint32_t *asset_id, const uint8_t *verdicts,
                            const uint32_t *ipos, uint32_t *asset_ids, uint32_t *ref_id, uint8_t *ref_on, uint32_t *cnt) {
    const uint8_t kd = kind[k];
    const bool pass = verdicts[k] == 1;
    uint32_t id = asset_id[k], issued = 0;
    if (kd == IMP_ISSUE && pass) {
        const uint64_t v = (uint64_t)next_id + ipos[k];
        if (v > IMP_ASSET_ID_MAX) imp_min(cnt + IMP_AS_OVF, (uint32_t)k);
        id = issued = (uint32_t)v;
    }
    asset_ids[k] = issued;
    ref_id[2 * k] = ref_id[2 * k + 1] = id;
    ref_on[2 * k] = kd == IMP_TRANSFER || pass;
    ref_on[2 * k + 1] = kd == IMP_TRANSFER;
}
ZK_IMP_DEV void imp_as_ref_insert(size_t p, const uint8_t *ref_on, const ImpAsKeys &t, uint32_t *table, uint32_t cap) {
    if (ref_on[p]) imp_as_insert(t, t.n_slots + (uint32_t)p, table, cap);
}
// after every reference insert: flag[p] = 1 where reference p is its key's first and the key is in no table row, counted
// in cnt[IMP_AS_NEW]; zk_bal_prefix_sum turns the flags into each new key's row past n_slots
ZK_IMP_DEV void imp_as_new(size_t p, const uint8_t *ref_on, const ImpAsKeys &t, const uint32_t *table, uint32_t cap, uint32_t *flag,
                           uint32_t *cnt) {
    const uint32_t h = t.n_slots + (uint32_t)p;
    flag[p] = ref_on[p] && imp_as_find(t, h, table, cap) == h;
    if (flag[p]) imp_inc(cnt + IMP_AS_NEW);
}
// reference p's slot into slot_a[p / 2] (p even) or slot_b[p / 2] (IMP_NONE: no reference).  A new key's first reference
// also writes its row: (id, key) into new_ids / new_keys, zero ciphertexts into balances / pendings, and flags.
ZK_IMP_DEV void imp_as_slot(size_t p, const uint8_t *ref_on, const ImpAsKeys &t, const uint32_t *table, uint32_t cap, const uint32_t *newpos,
                            uint8_t flags, uint32_t *slot_a, uint32_t *slot_b, uint32_t *new_ids, uint8_t *new_keys, uint8_t *balances,
                            uint8_t *pendings, uint8_t *slot_flags) {
    uint32_t slot = IMP_NONE;
    if (ref_on[p]) {
        const uint32_t h = t.n_slots + (uint32_t)p, e = imp_as_find(t, h, table, cap);
        slot = e < t.n_slots ? e : t.n_slots + newpos[e - t.n_slots];
        if (e == h) {
            const uint8_t *key = imp_as_key(t, h);
            new_ids[slot] = t.ref_id[p];
            for (int i = 0; i < 32; i++) new_keys[32 * (size_t)slot + i] = key[i];
            for (int i = 0; i < 64; i++) balances[64 * (size_t)slot + i] = pendings[64 * (size_t)slot + i] = 0;
            slot_flags[slot] = flags;
        }
    }
    (p & 1 ? slot_b : slot_a)[p >> 1] = slot;
}
// zk_assets_block's tx_points: a transfer's as imp_tx_points; an issue's total | 0 | 0 | randomness (slots 2 and 4); a
// destroy's zero
ZK_IMP_DEV void imp_as_tx_points(size_t i, const uint8_t *kind, const uint8_t *rows, uint8_t *tx_points) {
    const uint8_t kd = kind[i >> 5];
    const uint32_t at = (uint32_t)(i & 31) >> 3;
    if (kd == IMP_TRANSFER || (kd == IMP_ISSUE && (at == 0 || at == 3))) {
        imp_tx_points(i, rows, tx_points);
        return;
    }
#pragma unroll
    for (int b = 0; b < 4; b++) tx_points[4 * i + b] = 0;
}

// ---- 7. zk_import_block -----------------------------------------------------------------------------------------------
// One launch verifies the rows of several sections (the confidential transfers, the asset calls, the anonymous issues)
// that use one key: each section compacts its rows behind the ones before it (imp_gather / imp_compact / imp_an_issue_row
// with off, the rows of the sections before it), the verifier runs once over them all, and each section reads its
// verdicts at its own offset (imp_fail / imp_decide / imp_an_scatter with off), over its own chain keys.  A section's
// rows are a contiguous run of the launch, so no verdict of one section is read by another.
// the lowest extrinsic whose signature verdict is not 1 into *first (IMP_NONE before the pass)
ZK_IMP_DEV void imp_sig_first(size_t i, const uint8_t *verdicts, uint32_t *first) {
    if (verdicts[i] != 1) imp_min(first, (uint32_t)i);
}
// after imp_sig_first: that extrinsic's verdict into *code (1 when every signature passes)
ZK_IMP_DEV void imp_sig_code(const uint8_t *verdicts, const uint32_t *first, uint32_t *code) {
    *code = *first != IMP_NONE ? verdicts[*first] : 1;
}
// a 32-byte little-endian z below r_J?  Every z is checked before the batch verdict is read, as zk_redjubjub_batch_verify
// checks them before it computes anything.
ZK_IMP_DEV bool imp_fs_canonical(const uint8_t *b) {
    const uint64_t r[4] = {0xd0970e5ed6f72cb7ull, 0xa6682093ccc81082ull, 0x06673b0101343b00ull, 0x0e7db4ea6533afa9ull};
#pragma unroll
    for (int w = 3; w >= 0; w--) {
        uint64_t v = 0;
#pragma unroll
        for (int k = 7; k >= 0; k--) v = v << 8 | b[8 * w + k];
        if (v != r[w]) return v < r[w];
    }
    return false;
}
// the lowest extrinsic whose z_i >= r_J into *first (IMP_NONE before the pass)
ZK_IMP_DEV void imp_sig_z(size_t i, const uint8_t *zs, uint32_t *first) {
    if (!imp_fs_canonical(zs + 32 * i)) imp_min(first, (uint32_t)i);
}

}  // namespace zkimp
