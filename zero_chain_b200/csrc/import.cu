// Block imports with their verify / apply rounds on the device (import.cuh): zk_import_confidential_block and
// zk_import_assets_block, and their _device forms.  One engine, run_rounds, parameterised by the state pass (balances.cu's
// zk_balances_confidential_block_device or assets.cu's zk_assets_block_device) and by the chain key (the sender account or
// the sender slot).  Everything stays on the context's stream between the first upload and the last download; the host
// reads a block of four counters before the first round (transfers, and the lowest transaction with a bad index) and after
// each round (failures, transfers left undecided), which is all it needs to launch the next round.
// zk_import_anonymous_block and its _device form (anon_run) take no rounds: a fixed sequence of verifications and state
// passes (import.cuh section 5), with one read of the counter block to size the two verifications.
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
static int read_counters(zk_ctx *ctx, const uint32_t *d_cnt, uint32_t *cnt) {
    ZK_CUDA(cudaMemcpyAsync(cnt, d_cnt, IMP_COUNTERS * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
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
