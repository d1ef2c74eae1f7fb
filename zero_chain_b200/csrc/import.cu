// Block imports with their verify / apply rounds on the device (import.cuh): zk_import_confidential_block and
// zk_import_assets_block, and their _device forms.  One engine, run_rounds, parameterised by the state pass (balances.cu's
// zk_balances_confidential_block_device or assets.cu's zk_assets_block_device) and by the chain key (the sender account or
// the sender slot).  Everything stays on the context's stream between the first upload and the last download; the host
// reads a block of four counters before the first round (transfers, and the lowest transaction with a bad index) and after
// each round (failures, transfers left undecided), which is all it needs to launch the next round.
// zk_import_anonymous_block and its _device form (anon_run) take no rounds: a fixed sequence of verifications and state
// passes (import.cuh section 5), with one read of the counter block to size the two verifications.
// zk_import_asset_calls and its _device form (asset_calls_run): import.cuh section 6's passes, then assets_run.
//
// The round buffers live in the context (ctx->imp); the host forms stage their arrays in ctx->imp_io.
#include "internal.h"
#include "anon_balances.cuh"
#include "assets.cuh"
#include "import.cuh"

using namespace zkimp;

constexpr int BT = 256;                 // threads per block
constexpr size_t PREFIX_TOTALS = 1024;  // workspace words of zk_bal_prefix_sum

#define IMP_FOR(i, n) for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < (n); i = (n))

static __global__ void __launch_bounds__(BT) k_imp_start(size_t n_tx, uint32_t n_keys, const uint8_t *__restrict__ kind,
                                                         const uint32_t *__restrict__ key_a, const uint32_t *__restrict__ key_b,
                                                         const uint8_t *fixed, uint8_t *verdict,   // may alias
                                                         uint8_t *__restrict__ applied, uint32_t *cnt) {
    IMP_FOR(k, n_tx) imp_start(k, n_keys, kind, key_a, key_b, fixed, verdict, applied, cnt);
}
static __global__ void __launch_bounds__(BT) k_imp_tx_points(size_t n, const uint8_t *__restrict__ rows, uint8_t *__restrict__ tx_points) {
    IMP_FOR(i, n) imp_tx_points(i, rows, tx_points);
}
static __global__ void __launch_bounds__(BT) k_imp_flag(size_t n_tx, const uint8_t *__restrict__ kind, const uint8_t *__restrict__ verdict,
                                                        uint32_t *__restrict__ flag) {
    IMP_FOR(k, n_tx) imp_flag(k, kind, verdict, flag);
}
static __global__ void __launch_bounds__(BT) k_imp_gather(size_t n, const uint8_t *__restrict__ kind, const uint8_t *__restrict__ verdict,
                                                          const uint32_t *__restrict__ pos,
                                                          const uint8_t *__restrict__ rows, const uint8_t *__restrict__ proofs,
                                                          const uint8_t *__restrict__ balance_sender, uint32_t *__restrict__ idx,
                                                          uint8_t *__restrict__ round_rows, uint8_t *__restrict__ round_proofs) {
    IMP_FOR(i, n) imp_gather(i, kind, verdict, pos, rows, proofs, balance_sender, idx, round_rows, round_proofs);
}
static __global__ void __launch_bounds__(BT) k_imp_fail(size_t m, const uint32_t *__restrict__ idx, const uint32_t *__restrict__ key_a,
                                                        const uint8_t *__restrict__ rv, uint32_t *first_fail, uint32_t *cnt) {
    IMP_FOR(j, m) imp_fail(j, idx, key_a, rv, first_fail, cnt);
}
static __global__ void __launch_bounds__(BT) k_imp_decide(size_t m, const uint32_t *__restrict__ idx, const uint32_t *__restrict__ key_a,
                                                          const uint8_t *__restrict__ rv, const uint32_t *__restrict__ first_fail,
                                                          uint8_t *__restrict__ verdict, uint8_t *__restrict__ applied, uint32_t *cnt) {
    IMP_FOR(j, m) imp_decide(j, idx, key_a, rv, first_fail, verdict, applied, cnt);
}

// zk_import_anonymous_block
static __global__ void __launch_bounds__(BT) k_imp_an_start(size_t n_tx, uint32_t n_acct, bool issues_ok, const uint8_t *__restrict__ kind,
                                                            const uint32_t *__restrict__ members, uint32_t *__restrict__ flag, uint32_t *cnt) {
    IMP_FOR(k, n_tx) imp_an_start(k, n_acct, issues_ok, kind, members, flag, cnt);
}
static __global__ void __launch_bounds__(BT) k_imp_an_issue_row(size_t n, const uint8_t *__restrict__ kind, const uint32_t *__restrict__ pos,
                                                                const uint8_t *__restrict__ keys, const uint32_t *__restrict__ members,
                                                                const uint8_t *__restrict__ tx_points, const uint8_t *__restrict__ issue_fields,
                                                                const uint8_t *__restrict__ tx_extra, const uint8_t *__restrict__ g_epoch,
                                                                const uint8_t *__restrict__ proofs, uint8_t *__restrict__ rows,
                                                                uint8_t *__restrict__ round_proofs) {
    IMP_FOR(i, n) imp_an_issue_row(i, kind, pos, keys, members, tx_points, issue_fields, tx_extra, g_epoch, proofs, rows, round_proofs);
}
static __global__ void __launch_bounds__(BT) k_imp_an_scatter(size_t n_tx, bool issues, const uint8_t *__restrict__ kind,
                                                              const uint32_t *__restrict__ pos, const uint8_t *__restrict__ rv,
                                                              uint8_t *__restrict__ verdicts) {
    IMP_FOR(k, n_tx) imp_an_scatter(k, issues, kind, pos, rv, verdicts);
}
static __global__ void __launch_bounds__(BT) k_imp_an_gather(size_t n, const uint8_t *__restrict__ kind, const uint32_t *__restrict__ pos,
                                                             const uint8_t *__restrict__ verify_points, const uint8_t *__restrict__ proofs,
                                                             uint8_t *__restrict__ rows, uint8_t *__restrict__ round_proofs) {
    IMP_FOR(i, n) imp_an_gather(i, kind, pos, verify_points, proofs, rows, round_proofs);
}

// zk_import_asset_calls
static __global__ void __launch_bounds__(BT) k_imp_as_start(size_t n_tx, const uint8_t *__restrict__ kind, uint32_t *__restrict__ flag,
                                                            uint32_t *cnt) {
    IMP_FOR(k, n_tx) imp_as_start(k, kind, flag, cnt);
}
static __global__ void __launch_bounds__(BT) k_imp_as_row_insert(size_t n_slots, ImpAsKeys t, uint32_t *table, uint32_t cap) {
    IMP_FOR(r, n_slots) imp_as_row_insert(r, t, table, cap);
}
static __global__ void __launch_bounds__(BT) k_imp_as_row_dup(size_t n_slots, ImpAsKeys t, const uint32_t *__restrict__ table, uint32_t cap,
                                                              uint32_t *cnt) {
    IMP_FOR(r, n_slots) imp_as_row_dup(r, t, table, cap, cnt);
}
static __global__ void __launch_bounds__(BT) k_imp_as_compact(size_t n, const uint8_t *__restrict__ kind, const uint32_t *__restrict__ pos,
                                                              const uint8_t *__restrict__ rows, const uint8_t *__restrict__ proofs,
                                                              uint8_t *__restrict__ round_rows, uint8_t *__restrict__ round_proofs) {
    IMP_FOR(i, n) imp_compact(i, IMP_ROW, true, kind, pos, rows, proofs, round_rows, round_proofs);
}
static __global__ void __launch_bounds__(BT) k_imp_as_issue_flag(size_t n_tx, const uint8_t *__restrict__ kind,
                                                                 const uint8_t *__restrict__ verdicts, uint32_t *__restrict__ flag) {
    IMP_FOR(k, n_tx) imp_as_issue_flag(k, kind, verdicts, flag);
}
static __global__ void __launch_bounds__(BT) k_imp_as_refs(size_t n_tx, uint32_t next_id, const uint8_t *__restrict__ kind,
                                                           const uint32_t *__restrict__ asset_id, const uint8_t *__restrict__ verdicts,
                                                           const uint32_t *__restrict__ ipos, uint32_t *__restrict__ asset_ids,
                                                           uint32_t *__restrict__ ref_id, uint8_t *__restrict__ ref_on, uint32_t *cnt) {
    IMP_FOR(k, n_tx) imp_as_refs(k, next_id, kind, asset_id, verdicts, ipos, asset_ids, ref_id, ref_on, cnt);
}
static __global__ void __launch_bounds__(BT) k_imp_as_ref_insert(size_t n_ref, const uint8_t *__restrict__ ref_on, ImpAsKeys t, uint32_t *table,
                                                                 uint32_t cap) {
    IMP_FOR(p, n_ref) imp_as_ref_insert(p, ref_on, t, table, cap);
}
static __global__ void __launch_bounds__(BT) k_imp_as_new(size_t n_ref, const uint8_t *__restrict__ ref_on, ImpAsKeys t,
                                                          const uint32_t *__restrict__ table, uint32_t cap, uint32_t *__restrict__ flag,
                                                          uint32_t *cnt) {
    IMP_FOR(p, n_ref) imp_as_new(p, ref_on, t, table, cap, flag, cnt);
}
static __global__ void __launch_bounds__(BT) k_imp_as_slot(size_t n_ref, const uint8_t *__restrict__ ref_on, ImpAsKeys t,
                                                           const uint32_t *__restrict__ table, uint32_t cap, const uint32_t *__restrict__ newpos,
                                                           uint8_t flags, uint32_t *__restrict__ slot_a, uint32_t *__restrict__ slot_b,
                                                           uint32_t *__restrict__ new_ids, uint8_t *__restrict__ new_keys,
                                                           uint8_t *__restrict__ balances, uint8_t *__restrict__ pendings,
                                                           uint8_t *__restrict__ slot_flags) {
    IMP_FOR(p, n_ref) imp_as_slot(p, ref_on, t, table, cap, newpos, flags, slot_a, slot_b, new_ids, new_keys, balances, pendings, slot_flags);
}
static __global__ void __launch_bounds__(BT) k_imp_as_tx_points(size_t n, const uint8_t *__restrict__ kind, const uint8_t *__restrict__ rows,
                                                                uint8_t *__restrict__ tx_points) {
    IMP_FOR(i, n) imp_as_tx_points(i, kind, rows, tx_points);
}

static unsigned grid(size_t n) { return (unsigned)(n ? (n + BT - 1) / BT : 1); }

struct ImpWork {
    uint8_t *applied, *rv, *balance_sender, *round_rows, *round_proofs, *tx_points;
    uint32_t *pos, *idx, *first_fail, *cnt, *totals;
};

static size_t carve(Carve &c, ImpWork &w, size_t n_tx, size_t n_keys, bool tx_points) {
    w.cnt = c.take<uint32_t>(IMP_COUNTERS); w.totals = c.take<uint32_t>(PREFIX_TOTALS);
    w.applied = c.take<uint8_t>(n_tx); w.rv = c.take<uint8_t>(n_tx); w.balance_sender = c.take<uint8_t>(64 * n_tx);
    w.round_rows = c.take<uint8_t>(IMP_ROW * n_tx); w.round_proofs = c.take<uint8_t>(192 * n_tx);
    w.tx_points = tx_points ? c.take<uint8_t>(128 * n_tx) : nullptr;
    w.pos = c.take<uint32_t>(n_tx); w.idx = c.take<uint32_t>(n_tx); w.first_fail = c.take<uint32_t>(n_keys);
    return c.off;
}

// the counter block to the host; zk_check_err_flag synchronises the stream and reports a touched account or slot that
// failed to read in the state pass
static int read_counters(zk_ctx *ctx, const uint32_t *d_cnt, uint32_t *cnt, size_t n = IMP_COUNTERS) {
    ZK_CUDA(cudaMemcpyAsync(cnt, d_cnt, n * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
    return zk_check_err_flag(ctx);
}

// The rounds of import.cuh over n_tx transactions.  state(w) enqueues the state pass with the mask w.applied, writing each
// transfer's balance_sender to w.balance_sender (and reading w.tx_points, when asked for); kind == NULL: every transaction
// is a transfer.  All arrays are device pointers.  rounds: the verification launches.
template <class State>
static int run_rounds(zk_ctx *ctx, const char *fn, const zk_pvk *pvk, size_t n_keys, size_t n_tx, const uint8_t *kind,
                      const uint32_t *key_a, const uint32_t *key_b, const uint8_t *rows, const uint8_t *proofs, const uint8_t *fixed,
                      uint8_t *verdicts, bool tx_points, unsigned *rounds, State state) {
    cudaStream_t st = ctx->stream;
    ImpWork w;
    Carve sizing;
    ZK_TRY(ctx->imp.reserve(carve(sizing, w, n_tx, n_keys, tx_points)));
    Carve c;
    c.base = ctx->imp.as<uint8_t>();
    carve(c, w, n_tx, n_keys, tx_points);
    if (rounds) *rounds = 0;
    if (!n_tx) {
        ZK_TRY(state(w));
        return zk_check_err_flag(ctx);
    }
    uint32_t cnt[IMP_COUNTERS];
    ZK_CUDA(cudaMemsetAsync(w.cnt, 0, IMP_COUNTERS * sizeof(uint32_t), st));
    ZK_CUDA(cudaMemsetAsync(w.cnt + IMP_BAD, 0xFF, sizeof(uint32_t), st));
    k_imp_start<<<grid(n_tx), BT, 0, st>>>(n_tx, (uint32_t)n_keys, kind, key_a, key_b, fixed, verdicts, w.applied, w.cnt);
    if (w.tx_points) k_imp_tx_points<<<grid(32 * n_tx), BT, 0, st>>>(32 * n_tx, rows, w.tx_points);
    ZK_CUDA(cudaGetLastError());
    ZK_TRY(read_counters(ctx, w.cnt, cnt));
    if (cnt[IMP_BAD] != IMP_NONE) {
        zk_set_error("%s: transaction %u: an index out of range%s", fn, cnt[IMP_BAD], kind ? " or an unknown kind" : "");
        return ZK_ERR_INVALID;
    }
    size_t m = cnt[IMP_TRANSFERS];                 // undecided transfers
    for (unsigned r = 0;; r++) {
        ZK_TRY(state(w));
        if (!m) break;                             // nothing undecided: this state pass is the final state
        if (rounds) *rounds = r + 1;
        k_imp_flag<<<grid(n_tx), BT, 0, st>>>(n_tx, kind, verdicts, w.pos);
        ZK_CUDA(cudaGetLastError());
        ZK_TRY(zk_bal_prefix_sum(ctx, w.pos, n_tx, w.totals));
        k_imp_gather<<<grid(IMP_WORDS * n_tx), BT, 0, st>>>(IMP_WORDS * n_tx, kind, verdicts, w.pos, rows, proofs, w.balance_sender, w.idx,
                                                             w.round_rows, w.round_proofs);
        ZK_CUDA(cudaGetLastError());
        ZK_TRY(zk_groth16_verify_points_batch_device(ctx, pvk, m, w.round_proofs, w.round_rows, IMP_POINTS, w.rv));
        ZK_CUDA(cudaMemsetAsync(w.first_fail, 0xFF, n_keys * sizeof(uint32_t), st));
        ZK_CUDA(cudaMemsetAsync(w.cnt, 0, 2 * sizeof(uint32_t), st));       // IMP_FAILS, IMP_LEFT
        k_imp_fail<<<grid(m), BT, 0, st>>>(m, w.idx, key_a, w.rv, w.first_fail, w.cnt);
        k_imp_decide<<<grid(m), BT, 0, st>>>(m, w.idx, key_a, w.rv, w.first_fail, verdicts, w.applied, w.cnt);
        ZK_CUDA(cudaGetLastError());
        ZK_TRY(read_counters(ctx, w.cnt, cnt));
        if (!cnt[IMP_FAILS]) return ZK_OK;         // every balance of this round was exact: its state pass is final
        m = cnt[IMP_LEFT];
    }
    return zk_check_err_flag(ctx);
}

// the verifier's own check (MalformedVerifyingKey: a key for other than n_points points), before any work: a call with no
// proofs makes only that check
static int check_key(zk_ctx *ctx, const zk_pvk *pvk, size_t n_points = IMP_POINTS) {
    return zk_groth16_verify_points_batch_device(ctx, pvk, 0, nullptr, nullptr, n_points, nullptr);
}

// ---- confidential transfers --------------------------------------------------------------------------------------------
static int conf_args(const char *fn, zk_ctx *ctx, const zk_pvk *pvk, size_t n_accounts, const void *balances, const void *pendings,
                     const void *acct_flags, size_t n_tx, const void *sender, const void *recipient, const void *rows, const void *proofs,
                     const void *verdicts, const void *balance_after, const void *tx_status, const void *new_balances,
                     const void *new_pendings, const void *new_flags) {
    if (!ctx || !pvk || (n_accounts && (!balances || !pendings || !acct_flags || !new_balances || !new_pendings || !new_flags)) ||
        (n_tx && (!sender || !recipient || !rows || !proofs || !verdicts || !balance_after || !tx_status))) {
        zk_set_error("%s: NULL argument", fn);
        return ZK_ERR_INVALID;
    }
    if (n_accounts > zkbal::BAL_MAX || n_tx > zkbal::BAL_MAX) {
        zk_set_error("%s: n_accounts = %zu, n_tx = %zu: each must be at most %u", fn, n_accounts, n_tx, zkbal::BAL_MAX);
        return ZK_ERR_INVALID;
    }
    return ZK_OK;
}

static int conf_run(zk_ctx *ctx, const char *fn, const zk_pvk *pvk, size_t n_accounts, const uint8_t *balances, const uint8_t *pendings,
                    const uint8_t *acct_flags, size_t n_tx, const uint32_t *sender, const uint32_t *recipient, const uint8_t *rows,
                    const uint8_t *proofs, uint8_t *verdicts, uint8_t *balance_after, uint8_t *tx_status, uint8_t *new_balances,
                    uint8_t *new_pendings, uint8_t *new_flags, unsigned *rounds) {
    auto state = [&](const ImpWork &w) -> int {
        // balance_after is written for applied transfers only, and a later round may apply fewer
        if (n_tx) ZK_CUDA(cudaMemsetAsync(balance_after, 0, 64 * n_tx, ctx->stream));
        return zk_balances_confidential_block_device(ctx, n_accounts, balances, pendings, acct_flags, n_tx, sender, recipient, w.tx_points,
                                                     w.applied, w.balance_sender, balance_after, tx_status, new_balances, new_pendings,
                                                     new_flags);
    };
    return run_rounds(ctx, fn, pvk, n_accounts, n_tx, nullptr, sender, recipient, rows, proofs, nullptr, verdicts, true, rounds, state);
}

extern "C" int zk_import_confidential_block_device(zk_ctx *ctx, const zk_pvk *pvk, size_t n_accounts, const uint8_t *d_balances,
                                                   const uint8_t *d_pendings, const uint8_t *d_acct_flags, size_t n_tx,
                                                   const uint32_t *d_sender, const uint32_t *d_recipient, const uint8_t *d_rows,
                                                   const uint8_t *d_proofs, uint8_t *d_verdicts, uint8_t *d_balance_after,
                                                   uint8_t *d_tx_status, uint8_t *d_new_balances, uint8_t *d_new_pendings,
                                                   uint8_t *d_new_flags, unsigned *rounds) {
    const char *fn = "zk_import_confidential_block_device";
    ZK_TRY(conf_args(fn, ctx, pvk, n_accounts, d_balances, d_pendings, d_acct_flags, n_tx, d_sender, d_recipient, d_rows, d_proofs,
                     d_verdicts, d_balance_after, d_tx_status, d_new_balances, d_new_pendings, d_new_flags));
    ZK_TRY(check_key(ctx, pvk));
    if (rounds) *rounds = 0;
    if (!n_accounts && !n_tx) return ZK_OK;
    ZK_TRY(zk_use_device(ctx));
    return conf_run(ctx, fn, pvk, n_accounts, d_balances, d_pendings, d_acct_flags, n_tx, d_sender, d_recipient, d_rows, d_proofs,
                    d_verdicts, d_balance_after, d_tx_status, d_new_balances, d_new_pendings, d_new_flags, rounds);
}

extern "C" int zk_import_confidential_block(zk_ctx *ctx, const zk_pvk *pvk, size_t n_accounts, const uint8_t *balances,
                                            const uint8_t *pendings, const uint8_t *acct_flags, size_t n_tx, const uint32_t *sender,
                                            const uint32_t *recipient, const uint8_t *rows, const uint8_t *proofs, uint8_t *verdicts,
                                            uint8_t *balance_after, uint8_t *tx_status, uint8_t *new_balances, uint8_t *new_pendings,
                                            uint8_t *new_flags, unsigned *rounds) {
    const char *fn = "zk_import_confidential_block";
    ZK_TRY(conf_args(fn, ctx, pvk, n_accounts, balances, pendings, acct_flags, n_tx, sender, recipient, rows, proofs, verdicts,
                     balance_after, tx_status, new_balances, new_pendings, new_flags));
    ZK_TRY(check_key(ctx, pvk));
    if (rounds) *rounds = 0;
    if (!n_accounts && !n_tx) return ZK_OK;
    ZK_TRY(zk_use_device(ctx));
    cudaStream_t st = ctx->stream;
    const size_t na = n_accounts;
    Carve c;
    for (int pass = 0; pass < 2; pass++) {     // inputs, then outputs
        if (pass) c = Carve{ctx->imp_io.as<uint8_t>(), 0};
        uint8_t *b = c.take<uint8_t>(64 * na), *p = c.take<uint8_t>(64 * na), *f = c.take<uint8_t>(na);
        uint32_t *s = c.take<uint32_t>(n_tx), *r = c.take<uint32_t>(n_tx);
        uint8_t *rw = c.take<uint8_t>(IMP_ROW * n_tx), *pf = c.take<uint8_t>(192 * n_tx), *v = c.take<uint8_t>(n_tx),
                *ba = c.take<uint8_t>(64 * n_tx), *ts = c.take<uint8_t>(n_tx), *nb = c.take<uint8_t>(64 * na),
                *npd = c.take<uint8_t>(64 * na), *nf = c.take<uint8_t>(na);
        if (!pass) { ZK_TRY(ctx->imp_io.reserve(c.off)); continue; }
        if (na) {
            ZK_CUDA(cudaMemcpyAsync(b, balances, 64 * na, cudaMemcpyHostToDevice, st));
            ZK_CUDA(cudaMemcpyAsync(p, pendings, 64 * na, cudaMemcpyHostToDevice, st));
            ZK_CUDA(cudaMemcpyAsync(f, acct_flags, na, cudaMemcpyHostToDevice, st));
        }
        if (n_tx) {
            ZK_CUDA(cudaMemcpyAsync(s, sender, 4 * n_tx, cudaMemcpyHostToDevice, st));
            ZK_CUDA(cudaMemcpyAsync(r, recipient, 4 * n_tx, cudaMemcpyHostToDevice, st));
            ZK_CUDA(cudaMemcpyAsync(rw, rows, IMP_ROW * n_tx, cudaMemcpyHostToDevice, st));
            ZK_CUDA(cudaMemcpyAsync(pf, proofs, 192 * n_tx, cudaMemcpyHostToDevice, st));
        }
        ZK_TRY(conf_run(ctx, fn, pvk, na, b, p, f, n_tx, s, r, rw, pf, v, ba, ts, nb, npd, nf, rounds));
        if (n_tx) {
            ZK_CUDA(cudaMemcpyAsync(verdicts, v, n_tx, cudaMemcpyDeviceToHost, st));
            ZK_CUDA(cudaMemcpyAsync(balance_after, ba, 64 * n_tx, cudaMemcpyDeviceToHost, st));
            ZK_CUDA(cudaMemcpyAsync(tx_status, ts, n_tx, cudaMemcpyDeviceToHost, st));
        }
        if (na) {
            ZK_CUDA(cudaMemcpyAsync(new_balances, nb, 64 * na, cudaMemcpyDeviceToHost, st));
            ZK_CUDA(cudaMemcpyAsync(new_pendings, npd, 64 * na, cudaMemcpyDeviceToHost, st));
            ZK_CUDA(cudaMemcpyAsync(new_flags, nf, na, cudaMemcpyDeviceToHost, st));
        }
    }
    ZK_CUDA(cudaStreamSynchronize(st));
    return ZK_OK;
}

// ---- encrypted-asset calls ---------------------------------------------------------------------------------------------
static int assets_args(const char *fn, zk_ctx *ctx, const zk_pvk *pvk, size_t n_slots, const void *balances, const void *pendings,
                       const void *slot_flags, size_t n_tx, const void *kind, const void *slot_a, const void *slot_b, const void *tx_points,
                       const void *rows, const void *proofs, const void *fixed_verdicts, const void *verdicts, const void *balance_after,
                       const void *event_ct, const void *event_flags, const void *tx_status, const void *new_balances,
                       const void *new_pendings, const void *new_flags) {
    if (!ctx || !pvk || (n_slots && (!balances || !pendings || !slot_flags || !new_balances || !new_pendings || !new_flags)) ||
        (n_tx && (!kind || !slot_a || !slot_b || !tx_points || !rows || !proofs || !fixed_verdicts || !verdicts || !balance_after ||
                  !event_ct || !event_flags || !tx_status))) {
        zk_set_error("%s: NULL argument", fn);
        return ZK_ERR_INVALID;
    }
    if (n_slots > zkbal::BAL_MAX || n_tx > zkbal::AS_MAX_TX) {
        zk_set_error("%s: n_slots = %zu, n_tx = %zu: at most %u slots and %u transactions", fn, n_slots, n_tx, zkbal::BAL_MAX,
                     zkbal::AS_MAX_TX);
        return ZK_ERR_INVALID;
    }
    return ZK_OK;
}

static int assets_run(zk_ctx *ctx, const char *fn, const zk_pvk *pvk, size_t n_slots, const uint8_t *balances, const uint8_t *pendings,
                      const uint8_t *slot_flags, size_t n_tx, const uint8_t *kind, const uint32_t *slot_a, const uint32_t *slot_b,
                      const uint8_t *tx_points, const uint8_t *rows, const uint8_t *proofs, const uint8_t *fixed_verdicts, uint8_t *verdicts,
                      uint8_t *balance_after, uint8_t *event_ct, uint8_t *event_flags, uint8_t *tx_status, uint8_t *new_balances,
                      uint8_t *new_pendings, uint8_t *new_flags, unsigned *rounds) {
    auto state = [&](const ImpWork &w) -> int {
        // balance_after and the events are written for applied transactions only, and a later round may apply fewer
        if (n_tx) {
            ZK_CUDA(cudaMemsetAsync(balance_after, 0, 64 * n_tx, ctx->stream));
            ZK_CUDA(cudaMemsetAsync(event_ct, 0, 128 * n_tx, ctx->stream));
            ZK_CUDA(cudaMemsetAsync(event_flags, 0, n_tx, ctx->stream));
        }
        return zk_assets_block_device(ctx, n_slots, balances, pendings, slot_flags, n_tx, kind, slot_a, slot_b, tx_points, w.applied,
                                      w.balance_sender, balance_after, event_ct, event_flags, tx_status, new_balances, new_pendings, new_flags);
    };
    return run_rounds(ctx, fn, pvk, n_slots, n_tx, kind, slot_a, slot_b, rows, proofs, fixed_verdicts, verdicts, false, rounds, state);
}

extern "C" int zk_import_assets_block_device(zk_ctx *ctx, const zk_pvk *pvk, size_t n_slots, const uint8_t *d_balances,
                                             const uint8_t *d_pendings, const uint8_t *d_slot_flags, size_t n_tx, const uint8_t *d_kind,
                                             const uint32_t *d_slot_a, const uint32_t *d_slot_b, const uint8_t *d_tx_points,
                                             const uint8_t *d_rows, const uint8_t *d_proofs, const uint8_t *d_fixed_verdicts,
                                             uint8_t *d_verdicts, uint8_t *d_balance_after, uint8_t *d_event_ct, uint8_t *d_event_flags,
                                             uint8_t *d_tx_status, uint8_t *d_new_balances, uint8_t *d_new_pendings, uint8_t *d_new_flags,
                                             unsigned *rounds) {
    const char *fn = "zk_import_assets_block_device";
    ZK_TRY(assets_args(fn, ctx, pvk, n_slots, d_balances, d_pendings, d_slot_flags, n_tx, d_kind, d_slot_a, d_slot_b, d_tx_points, d_rows,
                       d_proofs, d_fixed_verdicts, d_verdicts, d_balance_after, d_event_ct, d_event_flags, d_tx_status, d_new_balances,
                       d_new_pendings, d_new_flags));
    ZK_TRY(check_key(ctx, pvk));
    if (rounds) *rounds = 0;
    if (!n_slots && !n_tx) return ZK_OK;
    ZK_TRY(zk_use_device(ctx));
    return assets_run(ctx, fn, pvk, n_slots, d_balances, d_pendings, d_slot_flags, n_tx, d_kind, d_slot_a, d_slot_b, d_tx_points, d_rows,
                      d_proofs, d_fixed_verdicts, d_verdicts, d_balance_after, d_event_ct, d_event_flags, d_tx_status, d_new_balances,
                      d_new_pendings, d_new_flags, rounds);
}

extern "C" int zk_import_assets_block(zk_ctx *ctx, const zk_pvk *pvk, size_t n_slots, const uint8_t *balances, const uint8_t *pendings,
                                      const uint8_t *slot_flags, size_t n_tx, const uint8_t *kind, const uint32_t *slot_a,
                                      const uint32_t *slot_b, const uint8_t *tx_points, const uint8_t *rows, const uint8_t *proofs,
                                      const uint8_t *fixed_verdicts, uint8_t *verdicts, uint8_t *balance_after, uint8_t *event_ct,
                                      uint8_t *event_flags, uint8_t *tx_status, uint8_t *new_balances, uint8_t *new_pendings,
                                      uint8_t *new_flags, unsigned *rounds) {
    const char *fn = "zk_import_assets_block";
    ZK_TRY(assets_args(fn, ctx, pvk, n_slots, balances, pendings, slot_flags, n_tx, kind, slot_a, slot_b, tx_points, rows, proofs,
                       fixed_verdicts, verdicts, balance_after, event_ct, event_flags, tx_status, new_balances, new_pendings, new_flags));
    ZK_TRY(check_key(ctx, pvk));
    if (rounds) *rounds = 0;
    if (!n_slots && !n_tx) return ZK_OK;
    ZK_TRY(zk_use_device(ctx));
    cudaStream_t st = ctx->stream;
    const size_t ns = n_slots;
    Carve c;
    for (int pass = 0; pass < 2; pass++) {     // inputs, then outputs
        if (pass) c = Carve{ctx->imp_io.as<uint8_t>(), 0};
        uint8_t *b = c.take<uint8_t>(64 * ns), *p = c.take<uint8_t>(64 * ns), *f = c.take<uint8_t>(ns);
        uint32_t *sa = c.take<uint32_t>(n_tx), *sb = c.take<uint32_t>(n_tx);
        uint8_t *kd = c.take<uint8_t>(n_tx), *tp = c.take<uint8_t>(128 * n_tx), *rw = c.take<uint8_t>(IMP_ROW * n_tx),
                *pf = c.take<uint8_t>(192 * n_tx), *fx = c.take<uint8_t>(n_tx), *v = c.take<uint8_t>(n_tx), *ba = c.take<uint8_t>(64 * n_tx),
                *ev = c.take<uint8_t>(128 * n_tx), *ef = c.take<uint8_t>(n_tx), *ts = c.take<uint8_t>(n_tx), *nb = c.take<uint8_t>(64 * ns),
                *npd = c.take<uint8_t>(64 * ns), *nf = c.take<uint8_t>(ns);
        if (!pass) { ZK_TRY(ctx->imp_io.reserve(c.off)); continue; }
        if (ns) {
            ZK_CUDA(cudaMemcpyAsync(b, balances, 64 * ns, cudaMemcpyHostToDevice, st));
            ZK_CUDA(cudaMemcpyAsync(p, pendings, 64 * ns, cudaMemcpyHostToDevice, st));
            ZK_CUDA(cudaMemcpyAsync(f, slot_flags, ns, cudaMemcpyHostToDevice, st));
        }
        if (n_tx) {
            ZK_CUDA(cudaMemcpyAsync(sa, slot_a, 4 * n_tx, cudaMemcpyHostToDevice, st));
            ZK_CUDA(cudaMemcpyAsync(sb, slot_b, 4 * n_tx, cudaMemcpyHostToDevice, st));
            ZK_CUDA(cudaMemcpyAsync(kd, kind, n_tx, cudaMemcpyHostToDevice, st));
            ZK_CUDA(cudaMemcpyAsync(tp, tx_points, 128 * n_tx, cudaMemcpyHostToDevice, st));
            ZK_CUDA(cudaMemcpyAsync(rw, rows, IMP_ROW * n_tx, cudaMemcpyHostToDevice, st));
            ZK_CUDA(cudaMemcpyAsync(pf, proofs, 192 * n_tx, cudaMemcpyHostToDevice, st));
            ZK_CUDA(cudaMemcpyAsync(fx, fixed_verdicts, n_tx, cudaMemcpyHostToDevice, st));
        }
        ZK_TRY(assets_run(ctx, fn, pvk, ns, b, p, f, n_tx, kd, sa, sb, tp, rw, pf, fx, v, ba, ev, ef, ts, nb, npd, nf, rounds));
        if (n_tx) {
            ZK_CUDA(cudaMemcpyAsync(verdicts, v, n_tx, cudaMemcpyDeviceToHost, st));
            ZK_CUDA(cudaMemcpyAsync(balance_after, ba, 64 * n_tx, cudaMemcpyDeviceToHost, st));
            ZK_CUDA(cudaMemcpyAsync(event_ct, ev, 128 * n_tx, cudaMemcpyDeviceToHost, st));
            ZK_CUDA(cudaMemcpyAsync(event_flags, ef, n_tx, cudaMemcpyDeviceToHost, st));
            ZK_CUDA(cudaMemcpyAsync(tx_status, ts, n_tx, cudaMemcpyDeviceToHost, st));
        }
        if (ns) {
            ZK_CUDA(cudaMemcpyAsync(new_balances, nb, 64 * ns, cudaMemcpyDeviceToHost, st));
            ZK_CUDA(cudaMemcpyAsync(new_pendings, npd, 64 * ns, cudaMemcpyDeviceToHost, st));
            ZK_CUDA(cudaMemcpyAsync(new_flags, nf, ns, cudaMemcpyDeviceToHost, st));
        }
    }
    ZK_CUDA(cudaStreamSynchronize(st));
    return ZK_OK;
}

// ---- encrypted-asset calls from the extrinsic fields -------------------------------------------------------------------
// The passes of import.cuh section 6, then assets_run on the grown table with the issue and destroy verdicts fixed.  The
// host reads the counter block twice before the rounds: after imp_as_start, since the number of issues and destroys sizes
// their verification, and after imp_as_slot, since the number of new rows sizes the state pass.
static_assert(IMP_TRANSFER == zkbal::AS_TRANSFER && IMP_ISSUE == zkbal::AS_ISSUE && IMP_DESTROY == zkbal::AS_DESTROY,
              "import.cuh's kinds are assets.cuh's");

struct AsWork {
    uint8_t *round_rows, *round_proofs, *rv, *ref_on, *tx_points, *balances, *pendings, *flags;
    uint32_t *cnt, *totals, *pos, *ipos, *ref_id, *newpos, *table, *slot_a, *slot_b;
};

// n_rows = n_slots + 2 n_tx: the table grown by a new row at every reference at most
static size_t carve(Carve &c, AsWork &w, size_t n_tx, size_t n_rows, size_t cap) {
    w.cnt = c.take<uint32_t>(IMP_AS_COUNTERS); w.totals = c.take<uint32_t>(PREFIX_TOTALS);
    w.round_rows = c.take<uint8_t>(IMP_ROW * n_tx); w.round_proofs = c.take<uint8_t>(192 * n_tx); w.rv = c.take<uint8_t>(n_tx);
    w.pos = c.take<uint32_t>(n_tx); w.ipos = c.take<uint32_t>(n_tx); w.ref_id = c.take<uint32_t>(2 * n_tx); w.ref_on = c.take<uint8_t>(2 * n_tx);
    w.newpos = c.take<uint32_t>(2 * n_tx); w.table = c.take<uint32_t>(cap); w.slot_a = c.take<uint32_t>(n_tx); w.slot_b = c.take<uint32_t>(n_tx);
    w.tx_points = c.take<uint8_t>(128 * n_tx);
    w.balances = c.take<uint8_t>(64 * n_rows); w.pendings = c.take<uint8_t>(64 * n_rows); w.flags = c.take<uint8_t>(n_rows);
    return c.off;
}

static int asset_calls_args(const char *fn, zk_ctx *ctx, const zk_pvk *pvk, size_t n_slots, const void *slot_ids, const void *slot_keys,
                            const void *balances, const void *pendings, const void *slot_flags, size_t n_tx, const void *kind,
                            const void *asset_id, const void *rows, const void *proofs, const void *verdicts, const void *asset_ids,
                            const void *balance_after, const void *event_ct, const void *event_flags, const void *tx_status,
                            const void *new_slot_ids, const void *new_slot_keys, const void *new_balances, const void *new_pendings,
                            const void *new_flags, const void *n_slots_out) {
    if (!ctx || !pvk || !n_slots_out || (n_slots && (!slot_ids || !slot_keys || !balances || !pendings || !slot_flags)) ||
        (n_tx && (!kind || !asset_id || !rows || !proofs || !verdicts || !asset_ids || !balance_after || !event_ct || !event_flags ||
                  !tx_status)) ||
        ((n_slots || n_tx) && (!new_slot_ids || !new_slot_keys || !new_balances || !new_pendings || !new_flags))) {
        zk_set_error("%s: NULL argument", fn);
        return ZK_ERR_INVALID;
    }
    if (n_slots > zkbal::BAL_MAX || n_tx > zkbal::AS_MAX_TX) {
        zk_set_error("%s: n_slots = %zu, n_tx = %zu: at most %u slots and %u transactions", fn, n_slots, n_tx, zkbal::BAL_MAX,
                     zkbal::AS_MAX_TX);
        return ZK_ERR_INVALID;
    }
    return ZK_OK;
}

// All arrays are device pointers; the table outputs have room for n_slots + 2 n_tx rows.
static int asset_calls_run(zk_ctx *ctx, const char *fn, const zk_pvk *pvk, size_t n_slots, const uint32_t *slot_ids, const uint8_t *slot_keys,
                           const uint8_t *balances, const uint8_t *pendings, const uint8_t *slot_flags, uint32_t next_asset_id,
                           uint8_t new_slot_flags, size_t n_tx, const uint8_t *kind, const uint32_t *asset_id, const uint8_t *rows,
                           const uint8_t *proofs, uint8_t *verdicts, uint32_t *asset_ids, uint8_t *balance_after, uint8_t *event_ct,
                           uint8_t *event_flags, uint8_t *tx_status, uint32_t *new_slot_ids, uint8_t *new_slot_keys, uint8_t *new_balances,
                           uint8_t *new_pendings, uint8_t *new_flags, size_t *n_slots_out, unsigned *rounds) {
    cudaStream_t st = ctx->stream;
    const size_t n_ref = 2 * n_tx, n_rows = n_slots + n_ref, cap = ZK_IAS_CAPACITY(n_rows);
    AsWork w;
    Carve sizing;
    ZK_TRY(ctx->imp_as.reserve(carve(sizing, w, n_tx, n_rows, cap)));
    Carve c;
    c.base = ctx->imp_as.as<uint8_t>();
    carve(c, w, n_tx, n_rows, cap);
    const ImpAsKeys keys{slot_ids, slot_keys, w.ref_id, rows, (uint32_t)n_slots};
    uint32_t cnt[IMP_AS_COUNTERS];

    // 1. kinds, and the table's rows into the hash table
    ZK_CUDA(cudaMemsetAsync(w.cnt, 0, IMP_AS_BAD * sizeof(uint32_t), st));
    ZK_CUDA(cudaMemsetAsync(w.cnt + IMP_AS_BAD, 0xFF, (IMP_AS_COUNTERS - IMP_AS_BAD) * sizeof(uint32_t), st));
    ZK_CUDA(cudaMemsetAsync(w.table, 0xFF, cap * sizeof(uint32_t), st));
    if (n_tx) k_imp_as_start<<<grid(n_tx), BT, 0, st>>>(n_tx, kind, w.pos, w.cnt);
    k_imp_as_row_insert<<<grid(n_slots), BT, 0, st>>>(n_slots, keys, w.table, (uint32_t)cap);
    k_imp_as_row_dup<<<grid(n_slots), BT, 0, st>>>(n_slots, keys, w.table, (uint32_t)cap, w.cnt);
    ZK_CUDA(cudaGetLastError());
    ZK_TRY(read_counters(ctx, w.cnt, cnt, IMP_AS_COUNTERS));
    if (cnt[IMP_AS_BAD] != IMP_NONE) {
        zk_set_error("%s: transaction %u: an unknown kind", fn, cnt[IMP_AS_BAD]);
        return ZK_ERR_INVALID;
    }
    if (cnt[IMP_AS_DUP] != IMP_NONE) {
        zk_set_error("%s: slot row %u repeats an earlier row's (asset id, key)", fn, cnt[IMP_AS_DUP]);
        return ZK_ERR_INVALID;
    }

    if (n_tx) {
        // 2. the issues and destroys, verified; their verdicts fixed (transfers 0 until the rounds start them)
        const size_t m = cnt[IMP_AS_FIXED];
        ZK_CUDA(cudaMemsetAsync(verdicts, 0, n_tx, st));
        if (m) {
            ZK_TRY(zk_bal_prefix_sum(ctx, w.pos, n_tx, w.totals));
            k_imp_as_compact<<<grid(IMP_WORDS * n_tx), BT, 0, st>>>(IMP_WORDS * n_tx, kind, w.pos, rows, proofs, w.round_rows, w.round_proofs);
            ZK_CUDA(cudaGetLastError());
            ZK_TRY(zk_groth16_verify_points_batch_device(ctx, pvk, m, w.round_proofs, w.round_rows, IMP_POINTS, w.rv));
            k_imp_an_scatter<<<grid(n_tx), BT, 0, st>>>(n_tx, true, kind, w.pos, w.rv, verdicts);
        }
        // 3. asset ids and references
        k_imp_as_issue_flag<<<grid(n_tx), BT, 0, st>>>(n_tx, kind, verdicts, w.ipos);
        ZK_CUDA(cudaGetLastError());
        ZK_TRY(zk_bal_prefix_sum(ctx, w.ipos, n_tx, w.totals));
        k_imp_as_refs<<<grid(n_tx), BT, 0, st>>>(n_tx, next_asset_id, kind, asset_id, verdicts, w.ipos, asset_ids, w.ref_id, w.ref_on, w.cnt);
        // 4. the references into the hash table; new rows numbered in the order of their first reference
        k_imp_as_ref_insert<<<grid(n_ref), BT, 0, st>>>(n_ref, w.ref_on, keys, w.table, (uint32_t)cap);
        k_imp_as_new<<<grid(n_ref), BT, 0, st>>>(n_ref, w.ref_on, keys, w.table, (uint32_t)cap, w.newpos, w.cnt);
        ZK_CUDA(cudaGetLastError());
        ZK_TRY(zk_bal_prefix_sum(ctx, w.newpos, n_ref, w.totals));
    }
    // the table's rows, then the new ones behind them
    if (n_slots) {
        ZK_CUDA(cudaMemcpyAsync(w.balances, balances, 64 * n_slots, cudaMemcpyDeviceToDevice, st));
        ZK_CUDA(cudaMemcpyAsync(w.pendings, pendings, 64 * n_slots, cudaMemcpyDeviceToDevice, st));
        ZK_CUDA(cudaMemcpyAsync(w.flags, slot_flags, n_slots, cudaMemcpyDeviceToDevice, st));
        ZK_CUDA(cudaMemcpyAsync(new_slot_ids, slot_ids, 4 * n_slots, cudaMemcpyDeviceToDevice, st));
        ZK_CUDA(cudaMemcpyAsync(new_slot_keys, slot_keys, 32 * n_slots, cudaMemcpyDeviceToDevice, st));
    }
    if (n_tx) {
        const uint8_t flags = (uint8_t)(new_slot_flags & ~(zkbal::ACCT_BALANCE | zkbal::ACCT_PENDING));
        k_imp_as_slot<<<grid(n_ref), BT, 0, st>>>(n_ref, w.ref_on, keys, w.table, (uint32_t)cap, w.newpos, flags, w.slot_a, w.slot_b,
                                                  new_slot_ids, new_slot_keys, w.balances, w.pendings, w.flags);
        k_imp_as_tx_points<<<grid(32 * n_tx), BT, 0, st>>>(32 * n_tx, kind, rows, w.tx_points);
        ZK_CUDA(cudaGetLastError());
        ZK_TRY(read_counters(ctx, w.cnt, cnt, IMP_AS_COUNTERS));
        if (cnt[IMP_AS_OVF] != IMP_NONE) {
            zk_set_error("%s: transaction %u: the issue's asset id would pass 2^32 - 1", fn, cnt[IMP_AS_OVF]);
            return ZK_ERR_INVALID;
        }
    }
    const size_t ns = n_slots + cnt[IMP_AS_NEW];
    if (ns > zkbal::BAL_MAX) {
        zk_set_error("%s: %zu slots after the block's new ones: at most %u", fn, ns, zkbal::BAL_MAX);
        return ZK_ERR_INVALID;
    }
    *n_slots_out = ns;
    // 5. the rounds, the issue and destroy verdicts fixed in verdicts itself
    return assets_run(ctx, fn, pvk, ns, w.balances, w.pendings, w.flags, n_tx, kind, w.slot_a, w.slot_b, w.tx_points, rows, proofs, verdicts,
                      verdicts, balance_after, event_ct, event_flags, tx_status, new_balances, new_pendings, new_flags, rounds);
}

extern "C" int zk_import_asset_calls_device(zk_ctx *ctx, const zk_pvk *pvk, size_t n_slots, const uint32_t *d_slot_ids,
                                            const uint8_t *d_slot_keys, const uint8_t *d_balances, const uint8_t *d_pendings,
                                            const uint8_t *d_slot_flags, uint32_t next_asset_id, uint8_t new_slot_flags, size_t n_tx,
                                            const uint8_t *d_kind, const uint32_t *d_asset_id, const uint8_t *d_rows, const uint8_t *d_proofs,
                                            uint8_t *d_verdicts, uint32_t *d_asset_ids, uint8_t *d_balance_after, uint8_t *d_event_ct,
                                            uint8_t *d_event_flags, uint8_t *d_tx_status, uint32_t *d_new_slot_ids, uint8_t *d_new_slot_keys,
                                            uint8_t *d_new_balances, uint8_t *d_new_pendings, uint8_t *d_new_flags, size_t *n_slots_out,
                                            unsigned *rounds) {
    const char *fn = "zk_import_asset_calls_device";
    ZK_TRY(asset_calls_args(fn, ctx, pvk, n_slots, d_slot_ids, d_slot_keys, d_balances, d_pendings, d_slot_flags, n_tx, d_kind, d_asset_id,
                            d_rows, d_proofs, d_verdicts, d_asset_ids, d_balance_after, d_event_ct, d_event_flags, d_tx_status, d_new_slot_ids,
                            d_new_slot_keys, d_new_balances, d_new_pendings, d_new_flags, n_slots_out));
    ZK_TRY(check_key(ctx, pvk));
    if (rounds) *rounds = 0;
    *n_slots_out = 0;
    if (!n_slots && !n_tx) return ZK_OK;
    ZK_TRY(zk_use_device(ctx));
    return asset_calls_run(ctx, fn, pvk, n_slots, d_slot_ids, d_slot_keys, d_balances, d_pendings, d_slot_flags, next_asset_id, new_slot_flags,
                           n_tx, d_kind, d_asset_id, d_rows, d_proofs, d_verdicts, d_asset_ids, d_balance_after, d_event_ct, d_event_flags,
                           d_tx_status, d_new_slot_ids, d_new_slot_keys, d_new_balances, d_new_pendings, d_new_flags, n_slots_out, rounds);
}

extern "C" int zk_import_asset_calls(zk_ctx *ctx, const zk_pvk *pvk, size_t n_slots, const uint32_t *slot_ids, const uint8_t *slot_keys,
                                     const uint8_t *balances, const uint8_t *pendings, const uint8_t *slot_flags, uint32_t next_asset_id,
                                     uint8_t new_slot_flags, size_t n_tx, const uint8_t *kind, const uint32_t *asset_id, const uint8_t *rows,
                                     const uint8_t *proofs, uint8_t *verdicts, uint32_t *asset_ids, uint8_t *balance_after, uint8_t *event_ct,
                                     uint8_t *event_flags, uint8_t *tx_status, uint32_t *new_slot_ids, uint8_t *new_slot_keys,
                                     uint8_t *new_balances, uint8_t *new_pendings, uint8_t *new_flags, size_t *n_slots_out,
                                     unsigned *rounds) {
    const char *fn = "zk_import_asset_calls";
    ZK_TRY(asset_calls_args(fn, ctx, pvk, n_slots, slot_ids, slot_keys, balances, pendings, slot_flags, n_tx, kind, asset_id, rows, proofs,
                            verdicts, asset_ids, balance_after, event_ct, event_flags, tx_status, new_slot_ids, new_slot_keys, new_balances,
                            new_pendings, new_flags, n_slots_out));
    ZK_TRY(check_key(ctx, pvk));
    if (rounds) *rounds = 0;
    *n_slots_out = 0;
    if (!n_slots && !n_tx) return ZK_OK;
    ZK_TRY(zk_use_device(ctx));
    cudaStream_t st = ctx->stream;
    const size_t ns = n_slots, nr = n_slots + 2 * n_tx;
    Carve c;
    for (int pass = 0; pass < 2; pass++) {     // inputs, then outputs
        if (pass) c = Carve{ctx->imp_io.as<uint8_t>(), 0};
        uint32_t *si = c.take<uint32_t>(ns);
        uint8_t *sk = c.take<uint8_t>(32 * ns), *b = c.take<uint8_t>(64 * ns), *p = c.take<uint8_t>(64 * ns), *f = c.take<uint8_t>(ns),
                *kd = c.take<uint8_t>(n_tx);
        uint32_t *ai = c.take<uint32_t>(n_tx);
        uint8_t *rw = c.take<uint8_t>(IMP_ROW * n_tx), *pf = c.take<uint8_t>(192 * n_tx), *v = c.take<uint8_t>(n_tx);
        uint32_t *ids = c.take<uint32_t>(n_tx);
        uint8_t *ba = c.take<uint8_t>(64 * n_tx), *ev = c.take<uint8_t>(128 * n_tx), *ef = c.take<uint8_t>(n_tx), *ts = c.take<uint8_t>(n_tx);
        uint32_t *nsi = c.take<uint32_t>(nr);
        uint8_t *nsk = c.take<uint8_t>(32 * nr), *nb = c.take<uint8_t>(64 * nr), *npd = c.take<uint8_t>(64 * nr), *nf = c.take<uint8_t>(nr);
        if (!pass) { ZK_TRY(ctx->imp_io.reserve(c.off)); continue; }
        if (ns) {
            ZK_CUDA(cudaMemcpyAsync(si, slot_ids, 4 * ns, cudaMemcpyHostToDevice, st));
            ZK_CUDA(cudaMemcpyAsync(sk, slot_keys, 32 * ns, cudaMemcpyHostToDevice, st));
            ZK_CUDA(cudaMemcpyAsync(b, balances, 64 * ns, cudaMemcpyHostToDevice, st));
            ZK_CUDA(cudaMemcpyAsync(p, pendings, 64 * ns, cudaMemcpyHostToDevice, st));
            ZK_CUDA(cudaMemcpyAsync(f, slot_flags, ns, cudaMemcpyHostToDevice, st));
        }
        if (n_tx) {
            ZK_CUDA(cudaMemcpyAsync(kd, kind, n_tx, cudaMemcpyHostToDevice, st));
            ZK_CUDA(cudaMemcpyAsync(ai, asset_id, 4 * n_tx, cudaMemcpyHostToDevice, st));
            ZK_CUDA(cudaMemcpyAsync(rw, rows, IMP_ROW * n_tx, cudaMemcpyHostToDevice, st));
            ZK_CUDA(cudaMemcpyAsync(pf, proofs, 192 * n_tx, cudaMemcpyHostToDevice, st));
        }
        size_t n_out = 0;
        ZK_TRY(asset_calls_run(ctx, fn, pvk, ns, si, sk, b, p, f, next_asset_id, new_slot_flags, n_tx, kd, ai, rw, pf, v, ids, ba, ev, ef, ts,
                               nsi, nsk, nb, npd, nf, &n_out, rounds));
        if (n_tx) {
            ZK_CUDA(cudaMemcpyAsync(verdicts, v, n_tx, cudaMemcpyDeviceToHost, st));
            ZK_CUDA(cudaMemcpyAsync(asset_ids, ids, 4 * n_tx, cudaMemcpyDeviceToHost, st));
            ZK_CUDA(cudaMemcpyAsync(balance_after, ba, 64 * n_tx, cudaMemcpyDeviceToHost, st));
            ZK_CUDA(cudaMemcpyAsync(event_ct, ev, 128 * n_tx, cudaMemcpyDeviceToHost, st));
            ZK_CUDA(cudaMemcpyAsync(event_flags, ef, n_tx, cudaMemcpyDeviceToHost, st));
            ZK_CUDA(cudaMemcpyAsync(tx_status, ts, n_tx, cudaMemcpyDeviceToHost, st));
        }
        if (n_out) {
            ZK_CUDA(cudaMemcpyAsync(new_slot_ids, nsi, 4 * n_out, cudaMemcpyDeviceToHost, st));
            ZK_CUDA(cudaMemcpyAsync(new_slot_keys, nsk, 32 * n_out, cudaMemcpyDeviceToHost, st));
            ZK_CUDA(cudaMemcpyAsync(new_balances, nb, 64 * n_out, cudaMemcpyDeviceToHost, st));
            ZK_CUDA(cudaMemcpyAsync(new_pendings, npd, 64 * n_out, cudaMemcpyDeviceToHost, st));
            ZK_CUDA(cudaMemcpyAsync(new_flags, nf, n_out, cudaMemcpyDeviceToHost, st));
        }
        ZK_CUDA(cudaStreamSynchronize(st));
        *n_slots_out = n_out;
    }
    return ZK_OK;
}

// ---- anonymous-balances calls ------------------------------------------------------------------------------------------
// The fixed sequence of import.cuh section 5; no rounds.  The host reads the counter block once, after imp_an_start: the
// number of issues and of transfers sizes the two verifications.
static_assert(IMP_AN_RING == zkbal::AN_RING && IMP_AN_ROW == 32 * zkbal::AN_VERIFY_POINTS, "import.cuh's ring layout is anon_balances.cuh's");
static_assert(IMP_AN_TRANSFER == zkbal::AN_TRANSFER && IMP_AN_ISSUE == zkbal::AN_ISSUE, "import.cuh's kinds are anon_balances.cuh's");

struct AnonImpWork {
    uint8_t *verify_points, *rows, *round_proofs, *rv;
    uint32_t *pos, *cnt, *totals;
};

// rows holds the compacted issue rows (352 B each) in one verification and the transfer rows (1664 B) in the other
static size_t carve(Carve &c, AnonImpWork &w, size_t n_tx) {
    w.cnt = c.take<uint32_t>(IMP_COUNTERS); w.totals = c.take<uint32_t>(PREFIX_TOTALS);
    w.verify_points = c.take<uint8_t>(IMP_AN_ROW * n_tx); w.rows = c.take<uint8_t>(IMP_AN_ROW * n_tx);
    w.round_proofs = c.take<uint8_t>(192 * n_tx); w.rv = c.take<uint8_t>(n_tx); w.pos = c.take<uint32_t>(n_tx);
    return c.off;
}

static int anon_args(const char *fn, zk_ctx *ctx, const zk_pvk *anon_pvk, size_t n_accounts, const void *keys, const void *balances,
                     const void *pendings, const void *acct_flags, size_t n_tx, const void *members, const void *tx_points, const void *tx_extra,
                     const void *g_epoch, const void *proofs, const void *verdicts, const void *enc_balances, const void *issued,
                     const void *tx_status, const void *new_balances, const void *new_pendings, const void *new_flags) {
    if (!ctx || !anon_pvk || (n_accounts && (!keys || !balances || !pendings || !acct_flags || !new_balances || !new_pendings || !new_flags)) ||
        (n_tx && (!members || !tx_points || !tx_extra || !g_epoch || !proofs || !verdicts || !enc_balances || !issued || !tx_status))) {
        zk_set_error("%s: NULL argument", fn);
        return ZK_ERR_INVALID;
    }
    if (n_accounts > zkbal::BAL_MAX || n_tx > zkbal::AN_MAX_TX) {
        zk_set_error("%s: n_accounts = %zu, n_tx = %zu: at most %u accounts and %u transactions", fn, n_accounts, n_tx, zkbal::BAL_MAX,
                     zkbal::AN_MAX_TX);
        return ZK_ERR_INVALID;
    }
    return ZK_OK;
}

// the keys' shapes (MalformedVerifyingKey), before any work
static int anon_keys(zk_ctx *ctx, const zk_pvk *anon_pvk, const zk_pvk *conf_pvk) {
    ZK_TRY(check_key(ctx, anon_pvk, zkbal::AN_VERIFY_POINTS));
    return conf_pvk ? check_key(ctx, conf_pvk) : ZK_OK;
}

// All arrays are device pointers; kind NULL: every transaction is a transfer.
static int anon_run(zk_ctx *ctx, const char *fn, const zk_pvk *anon_pvk, const zk_pvk *conf_pvk, size_t n_acct, const uint8_t *keys,
                    const uint8_t *balances, const uint8_t *pendings, const uint8_t *acct_flags, size_t n_tx, const uint8_t *kind,
                    const uint32_t *members, const uint8_t *tx_points, const uint8_t *tx_extra, const uint8_t *issue_fields,
                    const uint8_t *g_epoch, const uint8_t *proofs, uint8_t *verdicts, uint8_t *enc_balances, uint8_t *issued,
                    uint8_t *tx_status, uint8_t *new_balances, uint8_t *new_pendings, uint8_t *new_flags) {
    cudaStream_t st = ctx->stream;
    AnonImpWork w;
    Carve sizing;
    ZK_TRY(ctx->imp.reserve(carve(sizing, w, n_tx)));
    Carve c;
    c.base = ctx->imp.as<uint8_t>();
    carve(c, w, n_tx);
    // the issue verdicts, when there are issues, select the passes of zk_anonymous_calls_block; without issues the state
    // pass is zk_balances_anonymous_block's, as the Python driver runs it
    bool issues = false;
    auto state = [&]() -> int {
        if (issues)
            return zk_anonymous_calls_block_device(ctx, n_acct, keys, balances, pendings, acct_flags, n_tx, kind, members, tx_points, tx_extra,
                                                   g_epoch, verdicts, enc_balances, w.verify_points, issued, tx_status, new_balances,
                                                   new_pendings, new_flags);
        return zk_balances_anonymous_block_device(ctx, n_acct, keys, balances, pendings, acct_flags, n_tx, members, tx_points, tx_extra,
                                                  g_epoch, verdicts, enc_balances, w.verify_points, tx_status, new_balances, new_pendings,
                                                  new_flags);
    };
    if (!n_tx) {
        ZK_TRY(state());
        return zk_check_err_flag(ctx);
    }
    uint32_t cnt[IMP_COUNTERS];
    ZK_CUDA(cudaMemsetAsync(w.cnt, 0, IMP_COUNTERS * sizeof(uint32_t), st));
    ZK_CUDA(cudaMemsetAsync(w.cnt + IMP_BAD, 0xFF, sizeof(uint32_t), st));
    k_imp_an_start<<<grid(n_tx), BT, 0, st>>>(n_tx, (uint32_t)n_acct, conf_pvk && issue_fields, kind, members, w.pos, w.cnt);
    ZK_CUDA(cudaGetLastError());
    // transfers start unapplied; issued holds zero bytes where no applied issue writes
    ZK_CUDA(cudaMemsetAsync(verdicts, 0, n_tx, st));
    ZK_CUDA(cudaMemsetAsync(issued, 0, 64 * n_tx, st));
    ZK_TRY(read_counters(ctx, w.cnt, cnt));
    if (cnt[IMP_BAD] != IMP_NONE) {
        zk_set_error("%s: transaction %u: an index out of range, an unknown kind, or an issue without conf_pvk and issue_fields", fn,
                     cnt[IMP_BAD]);
        return ZK_ERR_INVALID;
    }
    const size_t n_iss = cnt[IMP_ISSUES], n_tr = cnt[IMP_TRANSFERS];
    issues = n_iss > 0;
    if (!issues) {
        // every transaction a transfer: verify the state pass's rows in place, the verdicts straight into the mask
        ZK_TRY(state());
        ZK_TRY(zk_groth16_verify_points_batch_device(ctx, anon_pvk, n_tx, proofs, w.verify_points, zkbal::AN_VERIFY_POINTS, verdicts));
        ZK_TRY(state());
        return zk_check_err_flag(ctx);
    }
    ZK_TRY(zk_bal_prefix_sum(ctx, w.pos, n_tx, w.totals));
    k_imp_an_issue_row<<<grid(IMP_AN_ISSUE_WORDS * n_tx), BT, 0, st>>>(IMP_AN_ISSUE_WORDS * n_tx, kind, w.pos, keys, members, tx_points,
                                                                     issue_fields, tx_extra, g_epoch, proofs, w.rows, w.round_proofs);
    ZK_CUDA(cudaGetLastError());
    ZK_TRY(zk_groth16_verify_points_batch_device(ctx, conf_pvk, n_iss, w.round_proofs, w.rows, IMP_POINTS, w.rv));
    k_imp_an_scatter<<<grid(n_tx), BT, 0, st>>>(n_tx, true, kind, w.pos, w.rv, verdicts);
    ZK_CUDA(cudaGetLastError());
    ZK_TRY(state());
    if (n_tr) {
        k_imp_an_gather<<<grid(IMP_AN_WORDS * n_tx), BT, 0, st>>>(IMP_AN_WORDS * n_tx, kind, w.pos, w.verify_points, proofs, w.rows,
                                                                 w.round_proofs);
        ZK_CUDA(cudaGetLastError());
        ZK_TRY(zk_groth16_verify_points_batch_device(ctx, anon_pvk, n_tr, w.round_proofs, w.rows, zkbal::AN_VERIFY_POINTS, w.rv));
        k_imp_an_scatter<<<grid(n_tx), BT, 0, st>>>(n_tx, false, kind, w.pos, w.rv, verdicts);
        ZK_CUDA(cudaGetLastError());
        ZK_TRY(state());
    }
    return zk_check_err_flag(ctx);
}

extern "C" int zk_import_anonymous_block_device(zk_ctx *ctx, const zk_pvk *anon_pvk, const zk_pvk *conf_pvk, size_t n_accounts,
                                                const uint8_t *d_keys, const uint8_t *d_balances, const uint8_t *d_pendings,
                                                const uint8_t *d_acct_flags, size_t n_tx, const uint8_t *d_kind, const uint32_t *d_members,
                                                const uint8_t *d_tx_points, const uint8_t *d_tx_extra, const uint8_t *d_issue_fields,
                                                const uint8_t *d_g_epoch, const uint8_t *d_proofs, uint8_t *d_verdicts, uint8_t *d_enc_balances,
                                                uint8_t *d_issued, uint8_t *d_tx_status, uint8_t *d_new_balances, uint8_t *d_new_pendings,
                                                uint8_t *d_new_flags) {
    const char *fn = "zk_import_anonymous_block_device";
    ZK_TRY(anon_args(fn, ctx, anon_pvk, n_accounts, d_keys, d_balances, d_pendings, d_acct_flags, n_tx, d_members, d_tx_points, d_tx_extra,
                     d_g_epoch, d_proofs, d_verdicts, d_enc_balances, d_issued, d_tx_status, d_new_balances, d_new_pendings, d_new_flags));
    ZK_TRY(anon_keys(ctx, anon_pvk, conf_pvk));
    if (!n_accounts && !n_tx) return ZK_OK;
    ZK_TRY(zk_use_device(ctx));
    return anon_run(ctx, fn, anon_pvk, conf_pvk, n_accounts, d_keys, d_balances, d_pendings, d_acct_flags, n_tx, d_kind, d_members, d_tx_points,
                    d_tx_extra, d_issue_fields, d_g_epoch, d_proofs, d_verdicts, d_enc_balances, d_issued, d_tx_status, d_new_balances,
                    d_new_pendings, d_new_flags);
}

extern "C" int zk_import_anonymous_block(zk_ctx *ctx, const zk_pvk *anon_pvk, const zk_pvk *conf_pvk, size_t n_accounts, const uint8_t *keys,
                                         const uint8_t *balances, const uint8_t *pendings, const uint8_t *acct_flags, size_t n_tx,
                                         const uint8_t *kind, const uint32_t *members, const uint8_t *tx_points, const uint8_t *tx_extra,
                                         const uint8_t *issue_fields, const uint8_t *g_epoch, const uint8_t *proofs, uint8_t *verdicts,
                                         uint8_t *enc_balances, uint8_t *issued, uint8_t *tx_status, uint8_t *new_balances,
                                         uint8_t *new_pendings, uint8_t *new_flags) {
    const char *fn = "zk_import_anonymous_block";
    ZK_TRY(anon_args(fn, ctx, anon_pvk, n_accounts, keys, balances, pendings, acct_flags, n_tx, members, tx_points, tx_extra, g_epoch, proofs,
                     verdicts, enc_balances, issued, tx_status, new_balances, new_pendings, new_flags));
    ZK_TRY(anon_keys(ctx, anon_pvk, conf_pvk));
    if (!n_accounts && !n_tx) return ZK_OK;
    ZK_TRY(zk_use_device(ctx));
    cudaStream_t st = ctx->stream;
    const size_t na = n_accounts, nk = kind ? n_tx : 0, nf_tx = issue_fields ? n_tx : 0;
    const size_t tp_bytes = 32 * (size_t)IMP_AN_TX_POINTS * n_tx, eb_bytes = 64 * (size_t)IMP_AN_RING * n_tx;
    Carve c;
    for (int pass = 0; pass < 2; pass++) {     // inputs, then outputs
        if (pass) c = Carve{ctx->imp_io.as<uint8_t>(), 0};
        uint8_t *ky = c.take<uint8_t>(32 * na), *b = c.take<uint8_t>(64 * na), *p = c.take<uint8_t>(64 * na), *f = c.take<uint8_t>(na);
        uint32_t *m = c.take<uint32_t>(IMP_AN_RING * n_tx);
        uint8_t *kd = c.take<uint8_t>(nk), *tp = c.take<uint8_t>(tp_bytes), *tx = c.take<uint8_t>(64 * n_tx), *fs = c.take<uint8_t>(96 * nf_tx),
                *ge = c.take<uint8_t>(32), *pf = c.take<uint8_t>(192 * n_tx), *v = c.take<uint8_t>(n_tx), *eb = c.take<uint8_t>(eb_bytes),
                *is = c.take<uint8_t>(64 * n_tx), *ts = c.take<uint8_t>(n_tx), *nb = c.take<uint8_t>(64 * na), *npd = c.take<uint8_t>(64 * na),
                *nf = c.take<uint8_t>(na);
        if (!pass) { ZK_TRY(ctx->imp_io.reserve(c.off)); continue; }
        if (na) {
            ZK_CUDA(cudaMemcpyAsync(ky, keys, 32 * na, cudaMemcpyHostToDevice, st));
            ZK_CUDA(cudaMemcpyAsync(b, balances, 64 * na, cudaMemcpyHostToDevice, st));
            ZK_CUDA(cudaMemcpyAsync(p, pendings, 64 * na, cudaMemcpyHostToDevice, st));
            ZK_CUDA(cudaMemcpyAsync(f, acct_flags, na, cudaMemcpyHostToDevice, st));
        }
        if (n_tx) {
            ZK_CUDA(cudaMemcpyAsync(m, members, 4 * IMP_AN_RING * n_tx, cudaMemcpyHostToDevice, st));
            ZK_CUDA(cudaMemcpyAsync(tp, tx_points, tp_bytes, cudaMemcpyHostToDevice, st));
            ZK_CUDA(cudaMemcpyAsync(tx, tx_extra, 64 * n_tx, cudaMemcpyHostToDevice, st));
            ZK_CUDA(cudaMemcpyAsync(ge, g_epoch, 32, cudaMemcpyHostToDevice, st));
            ZK_CUDA(cudaMemcpyAsync(pf, proofs, 192 * n_tx, cudaMemcpyHostToDevice, st));
        }
        if (nk) ZK_CUDA(cudaMemcpyAsync(kd, kind, nk, cudaMemcpyHostToDevice, st));
        if (nf_tx) ZK_CUDA(cudaMemcpyAsync(fs, issue_fields, 96 * nf_tx, cudaMemcpyHostToDevice, st));
        ZK_TRY(anon_run(ctx, fn, anon_pvk, conf_pvk, na, ky, b, p, f, n_tx, nk ? kd : nullptr, m, tp, tx, nf_tx ? fs : nullptr, ge, pf, v, eb, is,
                        ts, nb, npd, nf));
        if (n_tx) {
            ZK_CUDA(cudaMemcpyAsync(verdicts, v, n_tx, cudaMemcpyDeviceToHost, st));
            ZK_CUDA(cudaMemcpyAsync(enc_balances, eb, eb_bytes, cudaMemcpyDeviceToHost, st));
            ZK_CUDA(cudaMemcpyAsync(issued, is, 64 * n_tx, cudaMemcpyDeviceToHost, st));
            ZK_CUDA(cudaMemcpyAsync(tx_status, ts, n_tx, cudaMemcpyDeviceToHost, st));
        }
        if (na) {
            ZK_CUDA(cudaMemcpyAsync(new_balances, nb, 64 * na, cudaMemcpyDeviceToHost, st));
            ZK_CUDA(cudaMemcpyAsync(new_pendings, npd, 64 * na, cudaMemcpyDeviceToHost, st));
            ZK_CUDA(cudaMemcpyAsync(new_flags, nf, na, cudaMemcpyDeviceToHost, st));
        }
    }
    ZK_CUDA(cudaStreamSynchronize(st));
    return ZK_OK;
}
