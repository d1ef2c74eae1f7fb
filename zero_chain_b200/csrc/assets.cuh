// Encrypted-asset calls of one block: what modules/encrypted-assets runs around each proof check.
//
// Restates the module's per-extrinsic loop (modules/encrypted-assets/src/lib.rs:32-215, 266-358) over a block whose state is
// keyed by slot, one slot per (AssetId, EncKey):
//   confidential_transfer  rollover(sender), rollover(recipient) at a due slot's first transfer touch: balance = (balance
//                          or zero) + (pending or zero), present; pending absent.  The verifier reads the sender's balance
//                          (Ciphertext::zero() when absent); applied: balance -= (amount_sender + fee_sender, 2 randomness),
//                          an absent balance staying absent; pending(recipient) += (amount_recipient, randomness)
//   issue                  applied: balance(issuer slot) = from_left_right(total, randomness); no rollover, the pending
//                          transfer and the due state are not touched
//   destroy                applied: take the balance and the pending transfer (both absent after); no rollover
// Issue and destroy overwrite, so a slot's balance and pending values are no longer one group sum over the block.  They
// are group sums between restarts: the elements of a transaction (AS_ELEMS per transaction, in this order) are
//   0, 1  balance / pending of slot_a: a rollover (heads), an applied issue (balance head) or an applied destroy (heads)
//   2, 3  balance / pending of slot_b: its rollover (heads)
//   4     the send on slot_a's balance (a transfer; the negated delta when applied, else the identity)
//   5     the receive on slot_b's pending (a transfer; the delta when applied, else the identity)
// keyed as balances.cuh does (balance: slot, pending: n_slots + slot; 2 n_slots: no element).  A head starts a segment and
// carries its own starting value as its delta: the issued total, the identity for an absent value, or the rolled pair.  A
// segment that starts where a key starts, without a head, starts from the stored value.  Before a slot's first transfer
// touch only issues and destroys act on it, so the rolled pair is read off the element just before each rollover head on
// its key (a head, whose value is its delta) or the stored value.  After the stable sort, an integer prefix sum of (key
// change | head) numbers the segments, and balances.cu's segmented scan, keyed by those numbers, restarts at every head.
// Presence belongs to a segment: a balance segment keeps its head's presence; a pending segment is present when its head
// is or it receives anything applied.
//
// The pipeline (assets.cu), one function here per thread of each pass:
//   as_touch        the touched slots, and each slot's first transfer (atomicMin)
//   bal_decode      Point::read + as_prime_order of every transaction point and every touched slot's ciphertexts
//   as_tx           status, keys, element bits and deltas of each transaction
//   as_slot         the stored values of each slot, by key (absent: the identity)
//   zk_bal_sort     stable radix sort of the elements by key
//   as_pos          each element's sorted position, and the segment-start counters
//   as_roll         the rolled pair of each rollover head
//   zk_bal_prefix_sum, as_segkeys   segment numbers
//   zk_bal_scan     segmented exclusive scan of the deltas, keyed by segment
//   as_seg          each segment's start (presence, stored base) and received flag; the last element of each key
//   as_tx_points / as_slot_points   the projective outputs
//   bal_encode_chunk                Point::write with one inversion per BAL_ENC_CHUNK points
//   as_finish_tx / as_finish_slot   the output bytes
// As in balances.cuh, point state passes through global memory between passes and stays in registers inside them.  The
// same source compiles with ZK_HOST_EMUL for the CPU test (tests/host_emul/emul_assets.cpp).
#pragma once
#include "balances.cuh"

namespace zkbal {

enum AssetKind : uint8_t { AS_TRANSFER = 0, AS_ISSUE = 1, AS_DESTROY = 2 };
constexpr uint32_t AS_MAX_TX = 1u << 20;        // limit of n_tx (AS_ELEMS n_tx elements in the sort); n_slots <= BAL_MAX
constexpr int AS_ELEMS = 6;                     // elements per transaction
constexpr uint32_t AS_NONE = 0xFFFFFFFFu;
// element bits
constexpr uint8_t AS_HEAD = 1, AS_HEAD_PRESENT = 2, AS_ROLL = 4, AS_RECV = 8;
// segment bits: the value at the start is present; the segment starts from the stored value
constexpr uint8_t AS_SEG_PRESENT = 1, AS_SEG_STORED = 2;

ZK_DEV void as_min(uint32_t *p, uint32_t v) {
#ifdef ZK_HOST_EMUL
    if (v < *p) *p = v;
#else
    atomicMin(p, v);
#endif
}

ZK_DEV bool as_valid(uint8_t kind, uint32_t a, uint32_t b, uint32_t n) {
    return kind <= AS_DESTROY && a < n && (kind != AS_TRANSFER || b < n);
}

// ---- 1. touched slots --------------------------------------------------------------------------------------------------
// touched: referenced by a transaction whose kind and slots are valid; first[slot]: the first transfer touching it
// (AS_NONE before the pass).  A slot's rollover, when due, belongs to that transfer.
ZK_DEV void as_touch(size_t k, uint32_t n, const uint8_t *kind, const uint32_t *slot_a, const uint32_t *slot_b, uint8_t *touched,
                     uint32_t *first) {
    const uint8_t kd = kind[k];
    const uint32_t a = slot_a[k], b = slot_b[k];
    if (!as_valid(kd, a, b, n)) return;
    touched[a] = 1;
    if (kd == AS_TRANSFER) {
        touched[b] = 1;
        as_min(first + a, (uint32_t)k);
        as_min(first + b, (uint32_t)k);
    }
}

// ---- 3. transactions ---------------------------------------------------------------------------------------------------
// Status (an invalid kind or slot, then a rejected point the call reads, then the mask: applied iff applied[k] == 1), and
// the six elements' keys, bits and deltas.  A rollover head's delta is filled in by as_roll.
ZK_DEV void as_tx(size_t k, uint32_t n, const uint8_t *kind, const uint32_t *slot_a, const uint32_t *slot_b, const uint8_t *applied,
                  const uint8_t *flags, const uint32_t *first, const Ext *dec, const uint8_t *ok, uint32_t *keys, uint8_t *ebits,
                  Pair *delta, uint8_t *status) {
    const uint8_t kd = kind[k];
    const uint32_t a = slot_a[k], b = slot_b[k];
    const size_t e = AS_ELEMS * k, p = 4 * k;
    uint8_t st;
    if (!as_valid(kd, a, b, n)) st = BAL_BAD_INDEX;
    else if (kd == AS_TRANSFER ? !(ok[p] && ok[p + 1] && ok[p + 2] && ok[p + 3]) : kd == AS_ISSUE ? !(ok[p] && ok[p + 3]) : false)
        st = BAL_BAD_POINT;
    else st = applied[k] == 1 ? BAL_APPLIED : BAL_NOT_APPLIED;
    status[k] = st;
#pragma unroll
    for (int i = 0; i < AS_ELEMS; i++) { keys[e + i] = 2 * n; ebits[e + i] = 0; delta[e + i] = pair_identity(); }
    if (st == BAL_BAD_INDEX) return;
    if (kd == AS_TRANSFER) {
        if (first[a] == k && (flags[a] & ACCT_DUE)) {
            keys[e] = a; ebits[e] = AS_HEAD | AS_HEAD_PRESENT | AS_ROLL;
            keys[e + 1] = n + a; ebits[e + 1] = AS_HEAD;
        }
        if (b != a && first[b] == k && (flags[b] & ACCT_DUE)) {
            keys[e + 2] = b; ebits[e + 2] = AS_HEAD | AS_HEAD_PRESENT | AS_ROLL;
            keys[e + 3] = n + b; ebits[e + 3] = AS_HEAD;
        }
        keys[e + 4] = a;
        keys[e + 5] = n + b;
        if (st == BAL_APPLIED) {
            const Fr d2 = jj_d2();
            const Ext rnd = dec[p + 3];
            Pair send, recv;
            send.l = ext_neg(ext_add(dec[p], dec[p + 2], d2));
            send.r = ext_neg(ext_dbl(rnd));
            recv.l = dec[p + 1];
            recv.r = rnd;
            delta[e + 4] = send;
            delta[e + 5] = recv;
            ebits[e + 5] = AS_RECV;
        }
    } else if (st == BAL_APPLIED) {
        keys[e] = a;
        if (kd == AS_ISSUE) {
            ebits[e] = AS_HEAD | AS_HEAD_PRESENT;
            Pair t;
            t.l = dec[p];
            t.r = dec[p + 3];
            delta[e] = t;
        } else {
            ebits[e] = AS_HEAD;
            keys[e + 1] = n + a; ebits[e + 1] = AS_HEAD;
        }
    }
}

// ---- 4. stored values --------------------------------------------------------------------------------------------------
// base[slot] = the stored balance, base[n + slot] = the stored pending (the identity when absent or untouched).  A touched
// slot whose stored ciphertext fails to read is reported in *bad.
ZK_DEV void as_slot(size_t a, size_t n_tx, uint32_t n, const uint8_t *touched, const Ext *dec, const uint8_t *ok, Pair *base,
                    uint32_t *bad) {
    const size_t q = 4 * n_tx + 4 * a;
    if (touched[a] && !(ok[q] && ok[q + 1] && ok[q + 2] && ok[q + 3])) bal_report_bad(bad, (uint32_t)a);
    Pair b, p;
    b.l = dec[q]; b.r = dec[q + 1];
    p.l = dec[q + 2]; p.r = dec[q + 3];
    base[a] = b;
    base[n + a] = p;
}

// ---- 6. sorted positions and segment starts ----------------------------------------------------------------------------
ZK_DEV bool as_starts(size_t j, const uint32_t *skeys, const uint32_t *svals, const uint8_t *ebits) {
    return j == 0 || skeys[j] != skeys[j - 1] || (ebits[svals[j]] & AS_HEAD);
}
ZK_DEV void as_pos(size_t j, const uint32_t *skeys, const uint32_t *svals, const uint8_t *ebits, uint32_t *pos, uint32_t *cnt) {
    pos[svals[j]] = (uint32_t)j;
    cnt[j] = as_starts(j, skeys, svals, ebits);
}

// ---- 7. rollover heads -------------------------------------------------------------------------------------------------
// Item i: transaction i / 2's rollover of slot_a (i even) or slot_b (odd), when it has one.  The value before it on each
// key is the element just before it (an issue's or a destroy's head, whose value is its delta) or the stored value; the
// rolled balance is their sum (absent values are the identity).
ZK_DEV void as_roll(size_t i, const uint32_t *skeys, const uint32_t *svals, const uint8_t *ebits, const uint32_t *pos, const Pair *base,
                    Pair *delta) {
    const size_t e = AS_ELEMS * (i >> 1) + 2 * (i & 1);
    if (!(ebits[e] & AS_ROLL)) return;
    const Fr d2 = jj_d2();
    const uint32_t jb = pos[e], jp = pos[e + 1], kb = skeys[jb], kp = skeys[jp];
    const Pair &b = jb && skeys[jb - 1] == kb ? delta[svals[jb - 1]] : base[kb];
    const Pair &p = jp && skeys[jp - 1] == kp ? delta[svals[jp - 1]] : base[kp];
    delta[e] = pair_add(b, p, d2);
}

// ---- 8. segment numbers ------------------------------------------------------------------------------------------------
// cnt: the exclusive prefix sum of the segment starts; seg[j] = cnt[j] + (j starts a segment), in place: segment seg[j] - 1
ZK_DEV void as_segkeys(size_t j, const uint32_t *skeys, const uint32_t *svals, const uint8_t *ebits, uint32_t *seg) {
    seg[j] += as_starts(j, skeys, svals, ebits);
}

// ---- 10. segments ------------------------------------------------------------------------------------------------------
// The first element of a segment writes how the segment starts: from its head (present or not) or from the stored value
// (with the stored presence).  An applied receive sets seg_recv.  The last element of a key writes its position to last.
ZK_DEV void as_seg(size_t j, size_t ne, uint32_t n, const uint32_t *skeys, const uint32_t *svals, const uint32_t *seg, const uint8_t *ebits,
                   const uint8_t *flags, uint8_t *seg_info, uint8_t *seg_recv, uint32_t *last) {
    const uint32_t key = skeys[j], s = seg[j] - 1;
    const uint8_t eb = ebits[svals[j]];
    if (key >= 2 * n) return;
    if (j == 0 || seg[j - 1] != seg[j]) {
        const uint8_t stored = flags[key < n ? key : key - n] & (key < n ? ACCT_BALANCE : ACCT_PENDING);
        seg_info[s] = eb & AS_HEAD ? (eb & AS_HEAD_PRESENT ? AS_SEG_PRESENT : 0) : (uint8_t)(AS_SEG_STORED | (stored ? AS_SEG_PRESENT : 0));
    }
    if (eb & AS_RECV) seg_recv[s] = 1;
    if (j + 1 == ne || skeys[j + 1] != key) last[key] = (uint32_t)j;
}

// ---- 11. outputs in projective form ------------------------------------------------------------------------------------
// Half h (left 0, right 1) of the value before (after = false) or after sorted element j, whatever its presence.
ZK_DEV Ext as_value(size_t j, int h, bool after, const uint32_t *skeys, const uint32_t *svals, const uint32_t *seg, const uint8_t *seg_info,
                    const Pair *base, const Pair *excl, const Pair *delta, const Fr &d2) {
    Ext v = (&excl[j].l)[h];
    if (seg_info[seg[j] - 1] & AS_SEG_STORED) v = ext_add((&base[skeys[j]].l)[h], v, d2);
    if (after) v = ext_add(v, (&delta[svals[j]].l)[h], d2);
    return v;
}
// Is the value after sorted element j present?  pending: whether j's key is a pending key.
ZK_DEV bool as_present(size_t j, bool pending, const uint32_t *seg, const uint8_t *seg_info, const uint8_t *seg_recv) {
    const uint32_t s = seg[j] - 1;
    return (seg_info[s] & AS_SEG_PRESENT) || (pending && seg_recv[s]);
}

// Transaction k's four points at pts[4 k ..]: a transfer's balance_sender and balance_after, an applied issue's total,
// an applied destroy's taken balance and pending (the value before its head: the element before it on the key, or the
// stored value); the identity elsewhere.  evf[k]: which of a destroy's taken values are present (an issue: 1).
ZK_DEV void as_tx_points(size_t k, uint32_t n, const uint8_t *kind, const uint8_t *status, const uint32_t *skeys, const uint32_t *svals,
                         const uint32_t *pos, const uint32_t *seg, const uint8_t *seg_info, const uint8_t *seg_recv, const uint8_t *flags,
                         const Pair *base, const Pair *excl, const Pair *delta, Ext *pts, uint8_t *evf) {
    const uint8_t kd = kind[k], st = status[k];
    const size_t e = AS_ELEMS * k;
    const Fr d2 = jj_d2();
    uint8_t f = 0;
#pragma unroll 1
    for (int i = 0; i < 4; i++) pts[4 * k + i] = ext_identity();
    if (st == BAL_BAD_INDEX) {
    } else if (kd == AS_TRANSFER) {
        const uint32_t j = pos[e + 4];
        const bool present = as_present(j, false, seg, seg_info, seg_recv);
        if (present) {
#pragma unroll 1
            for (int h = 0; h < 2; h++) {
                const Ext bs = as_value(j, h, false, skeys, svals, seg, seg_info, base, excl, delta, d2);
                pts[4 * k + h] = bs;
                if (st == BAL_APPLIED) pts[4 * k + 2 + h] = ext_add(bs, (&delta[svals[j]].l)[h], d2);
            }
        }
    } else if (st == BAL_APPLIED && kd == AS_ISSUE) {
        pts[4 * k] = delta[e].l;
        pts[4 * k + 1] = delta[e].r;
        f = 1;
    } else if (st == BAL_APPLIED) {
#pragma unroll 1
        for (int w = 0; w < 2; w++) {
            const uint32_t j = pos[e + w], key = skeys[j];
            const bool prev = j && skeys[j - 1] == key;
            const bool present = prev ? as_present(j - 1, w == 1, seg, seg_info, seg_recv)
                                      : (flags[key < n ? key : key - n] & (w ? ACCT_PENDING : ACCT_BALANCE)) != 0;
            if (!present) continue;
            f |= (uint8_t)(1 << w);
#pragma unroll 1
            for (int h = 0; h < 2; h++)
                pts[4 * k + 2 * w + h] = prev ? as_value(j - 1, h, true, skeys, svals, seg, seg_info, base, excl, delta, d2) : (&base[key].l)[h];
        }
    }
    evf[k] = f;
}
// Slot a's final balance and pending at pts[4 n_tx + 4 a ..] (the value after the last element of each key, or the stored
// value), and which are present (present[a]).
ZK_DEV void as_slot_points(size_t a, size_t n_tx, uint32_t n, const uint8_t *touched, const uint8_t *flags, const uint32_t *skeys,
                           const uint32_t *svals, const uint32_t *last, const uint32_t *seg, const uint8_t *seg_info, const uint8_t *seg_recv,
                           const Pair *base, const Pair *excl, const Pair *delta, Ext *pts, uint8_t *present) {
    const size_t q = 4 * n_tx + 4 * a;
#pragma unroll 1
    for (int i = 0; i < 4; i++) pts[q + i] = ext_identity();
    if (!touched[a]) return;
    const Fr d2 = jj_d2();
    uint8_t pr = 0;
#pragma unroll 1
    for (int w = 0; w < 2; w++) {
        const uint32_t key = w ? n + (uint32_t)a : (uint32_t)a, j = last[key];
        const bool p = j != AS_NONE ? as_present(j, w == 1, seg, seg_info, seg_recv) : (flags[a] & (w ? ACCT_PENDING : ACCT_BALANCE)) != 0;
        if (!p) continue;
        pr |= (uint8_t)(1 << w);
#pragma unroll 1
        for (int h = 0; h < 2; h++)
            pts[q + 2 * w + h] = j != AS_NONE ? as_value(j, h, true, skeys, svals, seg, seg_info, base, excl, delta, d2) : (&base[key].l)[h];
    }
    present[a] = pr;
}

// ---- 14. output bytes --------------------------------------------------------------------------------------------------
// balance_sender: a transfer's row (Ciphertext::zero() for an invalid slot), 64 zero bytes for the other kinds;
// balance_after: applied transfers; event_ct / event_flags: applied issues (the total ciphertext | 64 zero bytes, 1) and
// applied destroys (taken balance | taken pending, an absent one as 64 zero bytes; which are present).
ZK_DEV void as_finish_tx(size_t k, const uint8_t *kind, const uint8_t *status, const uint8_t *evf, const uint32_t *enc,
                         uint8_t *balance_sender, uint8_t *balance_after, uint8_t *event_ct, uint8_t *event_flags) {
    const uint8_t kd = kind[k], st = status[k];
    const uint32_t *row = enc + 32 * k;
    if (kd == AS_TRANSFER) {
        store_le_words(row, 16, balance_sender + 64 * k);
        if (st == BAL_APPLIED) store_le_words(row + 16, 16, balance_after + 64 * k);
        return;
    }
#pragma unroll 1
    for (int i = 0; i < 64; i++) balance_sender[64 * k + i] = 0;
    if (st != BAL_APPLIED) return;
    const uint8_t f = evf[k];
#pragma unroll 1
    for (int w = 0; w < 2; w++) {
        if (f & (1 << w)) store_le_words(row + 16 * w, 16, event_ct + 128 * k + 64 * w);
        else for (int i = 0; i < 64; i++) event_ct[128 * k + 64 * w + i] = 0;
    }
    event_flags[k] = f;
}
// As bal_finish_acct, except that bit 2 (due) is cleared only for a slot a transfer touched.
ZK_DEV void as_finish_slot(size_t a, size_t n_tx, const uint8_t *touched, const uint32_t *first, const uint8_t *balances,
                           const uint8_t *pendings, const uint8_t *flags, const uint8_t *present, const uint32_t *enc,
                           uint8_t *new_balances, uint8_t *new_pendings, uint8_t *new_flags) {
    bal_finish_acct(a, n_tx, touched, balances, pendings, flags, present, enc, new_balances, new_pendings, new_flags);
    if (touched[a] && first[a] == AS_NONE) new_flags[a] |= flags[a] & ACCT_DUE;
}

}  // namespace zkbal
