// Block imports with their verify / apply rounds on the device (import.cuh): zk_import_block, and the single-pallet calls
// zk_import_confidential_block, zk_import_assets_block, zk_import_asset_calls and zk_import_anonymous_block, each with its
// _device form.  One engine (block_run, with the rounds of launch_round / rounds_rest) runs them all: zk_import_block
// with up to three sections, each single-pallet call as the one-section case.  Everything stays on the context's stream
// between the first upload and the last download; the host reads a block of counters only where the next launch's size
// depends on it.
//
// The round buffers live in the context (ctx->imp, ctx->imp_as); the host forms stage their arrays in ctx->io (Stage).
#include "internal.h"
#include "anon_balances.cuh"
#include "assets.cuh"
#include "import.cuh"

#include <functional>
#include <vector>

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
                                                          uint8_t *__restrict__ round_rows, uint8_t *__restrict__ round_proofs, size_t off) {
    IMP_FOR(i, n) imp_gather(i, kind, verdict, pos, rows, proofs, balance_sender, idx, round_rows, round_proofs, off);
}
static __global__ void __launch_bounds__(BT) k_imp_fail(size_t m, const uint32_t *__restrict__ idx, const uint32_t *__restrict__ key_a,
                                                        const uint8_t *__restrict__ rv, uint32_t *first_fail, uint32_t *cnt, size_t off) {
    IMP_FOR(j, m) imp_fail(j, idx, key_a, rv, first_fail, cnt, off);
}
static __global__ void __launch_bounds__(BT) k_imp_decide(size_t m, const uint32_t *__restrict__ idx, const uint32_t *__restrict__ key_a,
                                                          const uint8_t *__restrict__ rv, const uint32_t *__restrict__ first_fail,
                                                          uint8_t *__restrict__ verdict, uint8_t *__restrict__ applied, uint32_t *cnt,
                                                          size_t off) {
    IMP_FOR(j, m) imp_decide(j, idx, key_a, rv, first_fail, verdict, applied, cnt, off);
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
                                                                uint8_t *__restrict__ round_proofs, size_t off) {
    IMP_FOR(i, n) imp_an_issue_row(i, kind, pos, keys, members, tx_points, issue_fields, tx_extra, g_epoch, proofs, rows, round_proofs, off);
}
static __global__ void __launch_bounds__(BT) k_imp_an_scatter(size_t n_tx, bool issues, const uint8_t *__restrict__ kind,
                                                              const uint32_t *__restrict__ pos, const uint8_t *__restrict__ rv,
                                                              uint8_t *__restrict__ verdicts, size_t off) {
    IMP_FOR(k, n_tx) imp_an_scatter(k, issues, kind, pos, rv, verdicts, off);
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
                                                              uint8_t *__restrict__ round_rows, uint8_t *__restrict__ round_proofs,
                                                              size_t off) {
    IMP_FOR(i, n) imp_compact(i, IMP_ROW, true, kind, pos, rows, proofs, round_rows, round_proofs, off);
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

// zk_import_block
static __global__ void __launch_bounds__(BT) k_imp_sig_first(size_t n, const uint8_t *__restrict__ verdicts, uint32_t *first) {
    IMP_FOR(i, n) imp_sig_first(i, verdicts, first);
}
static __global__ void k_imp_sig_code(const uint8_t *__restrict__ verdicts, const uint32_t *first, uint32_t *code) {
    imp_sig_code(verdicts, first, code);
}
static __global__ void __launch_bounds__(BT) k_imp_sig_z(size_t n, const uint8_t *__restrict__ zs, uint32_t *first) {
    IMP_FOR(i, n) imp_sig_z(i, zs, first);
}

static unsigned grid(size_t n) { return (unsigned)(n ? (n + BT - 1) / BT : 1); }

// ---- the engine ---------------------------------------------------------------------------------------------------------
// One engine runs every import: zk_import_block with up to three sections, and each pallet's own call as the one-section
// case.  The 11-point launches are shared: the first (L1) verifies the confidential transfers' first round, every asset
// issue and destroy and every anonymous issue; after it come the asset numbering and slot resolution and the anonymous
// state passes with their 52-point launch; each later launch verifies the undecided transfers of both chain-keyed
// sections, the confidential one's round r with the asset one's round r - 1.  The host reads one block of counters before
// L1 (every section's kinds and indices, and the signatures' batch verdict), one after L1 (the confidential decisions, the
// new slot rows) and one after each later launch.

// the counter block: each section's counters at its own place, read back in one copy
enum BlockCounter {
    BC_CONF = 0, BC_ASSETS = 4, BC_AS_FRONT = 8, BC_ANON = 16,
    BC_SIG_FIRST = 20,           // uint64: the batch check's first rejected entry
    BC_SIG_VERDICT = 22,         // byte 0: the batch verdict
    BC_SIG_LOWEST = 23,          // the lowest extrinsic whose own verdict is not 1
    BC_SIG_CODE = 24,            // and that verdict
    BC_SIG_BAD_Z = 25,           // the lowest extrinsic whose z_i >= r_J
    BC_WORDS = 26
};
static_assert(BC_AS_FRONT + IMP_AS_COUNTERS <= BC_ANON && BC_SIG_FIRST % 2 == 0, "counter block layout");

// the buffers the sections of one launch share
struct Joint {
    uint32_t *cnt, *totals;
    uint8_t *round_rows, *round_proofs, *rv;
};
static void carve(Carve &c, Joint &j, size_t n_rows) {
    j.cnt = c.take<uint32_t>(BC_WORDS); j.totals = c.take<uint32_t>(PREFIX_TOTALS);
    j.round_rows = c.take<uint8_t>(IMP_ROW * n_rows); j.round_proofs = c.take<uint8_t>(192 * n_rows); j.rv = c.take<uint8_t>(n_rows);
}

// the counter block to the host; zk_check_err_flag synchronises the stream and reports a touched account or slot that
// failed to read in a state pass
static int read_counters(zk_ctx *ctx, const uint32_t *d_cnt, uint32_t *cnt) {
    ZK_CUDA(cudaMemcpyAsync(cnt, d_cnt, BC_WORDS * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
    return zk_check_err_flag(ctx);
}

static int verify11(zk_ctx *ctx, const zk_pvk *pvk, size_t n, const uint8_t *proofs, const uint8_t *rows, uint8_t *rv, unsigned *launches) {
    ++*launches;
    return zk_groth16_verify_points_batch_device(ctx, pvk, n, proofs, rows, IMP_POINTS, rv);
}

// One chain-keyed section of the rounds (import.cuh sections 0-4): the confidential transfers, or the asset calls.
// state enqueues the state pass with the mask applied, writing each transfer's balance_sender (and reading tx_points,
// when the section has them); kind == NULL: every transaction is a transfer.  All arrays are device pointers.
struct RoundSec {
    const char *fn = nullptr;
    size_t n_keys = 0, n_tx = 0;
    const uint8_t *kind = nullptr;
    const uint32_t *key_a = nullptr, *key_b = nullptr;
    const uint8_t *rows = nullptr, *proofs = nullptr, *fixed = nullptr;
    uint8_t *verdicts = nullptr;
    std::function<int(const RoundSec &)> state;
    // workspace
    uint8_t *applied = nullptr, *balance_sender = nullptr, *tx_points = nullptr;
    uint32_t *pos = nullptr, *idx = nullptr, *first_fail = nullptr, *cnt = nullptr;
    int cb = 0;                  // its counters' place in the counter block
    size_t m = 0, off = 0;       // undecided transfers; its first row in the current launch
    bool on = false, in_launch = false;
    unsigned rounds = 0;         // the launches it took part in
};

// max_keys: the most chain keys the section can have
static void carve(Carve &c, RoundSec &s, bool tx_points, size_t max_keys) {
    s.applied = c.take<uint8_t>(s.n_tx); s.balance_sender = c.take<uint8_t>(64 * s.n_tx);
    s.tx_points = tx_points ? c.take<uint8_t>(128 * s.n_tx) : nullptr;
    s.pos = c.take<uint32_t>(s.n_tx); s.idx = c.take<uint32_t>(s.n_tx); s.first_fail = c.take<uint32_t>(max_keys);
}

// import.cuh section 0 into verdict: every transfer undecided and applied, the other kinds' verdicts fixed
static int round_start(zk_ctx *ctx, RoundSec &s, const Joint &J, uint8_t *verdict) {
    cudaStream_t st = ctx->stream;
    s.cnt = J.cnt + s.cb;
    ZK_CUDA(cudaMemsetAsync(s.cnt, 0, IMP_COUNTERS * sizeof(uint32_t), st));
    ZK_CUDA(cudaMemsetAsync(s.cnt + IMP_BAD, 0xFF, sizeof(uint32_t), st));
    if (s.n_tx) {
        k_imp_start<<<grid(s.n_tx), BT, 0, st>>>(s.n_tx, (uint32_t)s.n_keys, s.kind, s.key_a, s.key_b, s.fixed, verdict, s.applied, s.cnt);
        if (s.tx_points) k_imp_tx_points<<<grid(32 * s.n_tx), BT, 0, st>>>(32 * s.n_tx, s.rows, s.tx_points);
    }
    ZK_CUDA(cudaGetLastError());
    return ZK_OK;
}
// after the read that follows round_start: the lowest bad transaction, or the section joins the rounds
static int round_join(RoundSec &s, const uint32_t *hc) {
    const uint32_t *h = hc + s.cb;
    if (s.n_tx && h[IMP_BAD] != IMP_NONE) {
        zk_set_error("%s: transaction %u: an index out of range%s", s.fn, h[IMP_BAD], s.kind ? " or an unknown kind" : "");
        return ZK_ERR_INVALID;
    }
    s.m = s.n_tx ? h[IMP_TRANSFERS] : 0;
    s.on = true;
    return ZK_OK;
}

// One launch of the rounds.  Each section that is on runs its state pass; one with undecided transfers compacts them
// behind the rows before it, and extra_rows more rows follow from extra_gather(off).  One verification over them all,
// then each section's decisions and extra_scatter(off) read their verdicts at their own offsets.  *any: a launch ran.
static int launch_round(zk_ctx *ctx, const zk_pvk *pvk, const Joint &J, RoundSec *const *secs, int n, size_t extra_rows,
                        const std::function<int(size_t)> &extra_gather, const std::function<int(size_t)> &extra_scatter,
                        unsigned *launches, bool *any) {
    cudaStream_t st = ctx->stream;
    size_t off = 0;
    for (int i = 0; i < n; i++) {
        RoundSec &s = *secs[i];
        s.in_launch = false;
        if (!s.on) continue;
        ZK_TRY(s.state(s));
        if (!s.m) {                                // nothing undecided: this state pass is the final state
            s.on = false;
            continue;
        }
        s.in_launch = true;
        s.rounds++;
        s.off = off;
        k_imp_flag<<<grid(s.n_tx), BT, 0, st>>>(s.n_tx, s.kind, s.verdicts, s.pos);
        ZK_CUDA(cudaGetLastError());
        ZK_TRY(zk_bal_prefix_sum(ctx, s.pos, s.n_tx, J.totals));
        k_imp_gather<<<grid(IMP_WORDS * s.n_tx), BT, 0, st>>>(IMP_WORDS * s.n_tx, s.kind, s.verdicts, s.pos, s.rows, s.proofs, s.balance_sender,
                                                               s.idx, J.round_rows, J.round_proofs, off);
        ZK_CUDA(cudaGetLastError());
        off += s.m;
    }
    const size_t extra_off = off;
    if (extra_rows) ZK_TRY(extra_gather(extra_off));
    off += extra_rows;
    *any = off > 0;
    if (!off) return ZK_OK;
    ZK_TRY(verify11(ctx, pvk, off, J.round_proofs, J.round_rows, J.rv, launches));
    for (int i = 0; i < n; i++) {
        RoundSec &s = *secs[i];
        if (!s.in_launch) continue;
        ZK_CUDA(cudaMemsetAsync(s.first_fail, 0xFF, s.n_keys * sizeof(uint32_t), st));
        ZK_CUDA(cudaMemsetAsync(s.cnt, 0, 2 * sizeof(uint32_t), st));        // IMP_FAILS, IMP_LEFT
        k_imp_fail<<<grid(s.m), BT, 0, st>>>(s.m, s.idx, s.key_a, J.rv, s.first_fail, s.cnt, s.off);
        k_imp_decide<<<grid(s.m), BT, 0, st>>>(s.m, s.idx, s.key_a, J.rv, s.first_fail, s.verdicts, s.applied, s.cnt, s.off);
        ZK_CUDA(cudaGetLastError());
    }
    if (extra_rows) ZK_TRY(extra_scatter(extra_off));
    return ZK_OK;
}
// after the read that follows a launch: a section without a failure is done (every balance of its round was exact, so
// its state pass is final); otherwise its undecided transfers wait for the next launch
static void round_decided(RoundSec *const *secs, int n, const uint32_t *hc) {
    for (int i = 0; i < n; i++) {
        RoundSec &s = *secs[i];
        if (!s.in_launch) continue;
        const uint32_t *h = hc + s.cb;
        if (!h[IMP_FAILS]) s.on = false;
        else s.m = h[IMP_LEFT];
    }
}
// the launches until every section is done
static int rounds_rest(zk_ctx *ctx, const zk_pvk *pvk, const Joint &J, RoundSec *const *secs, int n, unsigned *launches) {
    uint32_t hc[BC_WORDS];
    for (;;) {
        bool any;
        ZK_TRY(launch_round(ctx, pvk, J, secs, n, 0, nullptr, nullptr, launches, &any));
        if (!any) return zk_check_err_flag(ctx);
        ZK_TRY(read_counters(ctx, J.cnt, hc));
        round_decided(secs, n, hc);
    }
}

// the verifier's own check (MalformedVerifyingKey: a key for other than n_points points), before any work: a call with no
// proofs makes only that check
static int check_key(zk_ctx *ctx, const zk_pvk *pvk, size_t n_points = IMP_POINTS) {
    return zk_groth16_verify_points_batch_device(ctx, pvk, 0, nullptr, nullptr, n_points, nullptr);
}
static int null_arg(const char *fn) {
    zk_set_error("%s: NULL argument", fn);
    return ZK_ERR_INVALID;
}

// ---- the sections' arguments --------------------------------------------------------------------------------------------
// Each holds one call's arguments less ctx and the keys, as device pointers, or as host pointers before staging.
struct ConfIn {
    const char *fn;
    size_t n_accounts;
    const uint8_t *balances, *pendings, *acct_flags;
    size_t n_tx;
    const uint32_t *sender, *recipient;
    const uint8_t *rows, *proofs;
    uint8_t *verdicts, *balance_after, *tx_status, *new_balances, *new_pendings, *new_flags;
    unsigned *rounds;
};
struct AssetIn {
    const char *fn;
    size_t n_slots;
    const uint32_t *slot_ids;
    const uint8_t *slot_keys, *balances, *pendings, *slot_flags;
    uint32_t next_asset_id;
    uint8_t new_slot_flags;
    size_t n_tx;
    const uint8_t *kind;
    const uint32_t *asset_id;
    const uint8_t *rows, *proofs;
    uint8_t *verdicts;
    uint32_t *asset_ids;
    uint8_t *balance_after, *event_ct, *event_flags, *tx_status;
    uint32_t *new_slot_ids;
    uint8_t *new_slot_keys, *new_balances, *new_pendings, *new_flags;
    size_t *n_slots_out;
    unsigned *rounds;
};
struct AnonIn {
    const char *fn;
    size_t n_accounts;
    const uint8_t *keys, *balances, *pendings, *acct_flags;
    size_t n_tx;
    const uint8_t *kind;
    const uint32_t *members;
    const uint8_t *tx_points, *tx_extra, *issue_fields, *g_epoch, *proofs;
    uint8_t *verdicts, *enc_balances, *issued, *tx_status, *new_balances, *new_pendings, *new_flags;
};
struct SigIn {
    size_t n;
    const uint8_t *vks, *sigs, *msgs;
    const uint64_t *msg_off;
    const uint8_t *zs;
};

// NULL arguments and sizes, as each call checks them
static int conf_args(const ConfIn &a) {
    if ((a.n_accounts && (!a.balances || !a.pendings || !a.acct_flags || !a.new_balances || !a.new_pendings || !a.new_flags)) ||
        (a.n_tx && (!a.sender || !a.recipient || !a.rows || !a.proofs || !a.verdicts || !a.balance_after || !a.tx_status)))
        return null_arg(a.fn);
    if (a.n_accounts > zkbal::BAL_MAX || a.n_tx > zkbal::BAL_MAX) {
        zk_set_error("%s: n_accounts = %zu, n_tx = %zu: each must be at most %u", a.fn, a.n_accounts, a.n_tx, zkbal::BAL_MAX);
        return ZK_ERR_INVALID;
    }
    return ZK_OK;
}
static int asset_args(const AssetIn &a) {
    if (!a.n_slots_out || (a.n_slots && (!a.slot_ids || !a.slot_keys || !a.balances || !a.pendings || !a.slot_flags)) ||
        (a.n_tx && (!a.kind || !a.asset_id || !a.rows || !a.proofs || !a.verdicts || !a.asset_ids || !a.balance_after || !a.event_ct ||
                    !a.event_flags || !a.tx_status)) ||
        ((a.n_slots || a.n_tx) && (!a.new_slot_ids || !a.new_slot_keys || !a.new_balances || !a.new_pendings || !a.new_flags)))
        return null_arg(a.fn);
    if (a.n_slots > zkbal::BAL_MAX || a.n_tx > zkbal::AS_MAX_TX) {
        zk_set_error("%s: n_slots = %zu, n_tx = %zu: at most %u slots and %u transactions", a.fn, a.n_slots, a.n_tx, zkbal::BAL_MAX,
                     zkbal::AS_MAX_TX);
        return ZK_ERR_INVALID;
    }
    return ZK_OK;
}
static int anon_args(const AnonIn &a) {
    if ((a.n_accounts && (!a.keys || !a.balances || !a.pendings || !a.acct_flags || !a.new_balances || !a.new_pendings || !a.new_flags)) ||
        (a.n_tx && (!a.members || !a.tx_points || !a.tx_extra || !a.g_epoch || !a.proofs || !a.verdicts || !a.enc_balances || !a.issued ||
                    !a.tx_status)))
        return null_arg(a.fn);
    if (a.n_accounts > zkbal::BAL_MAX || a.n_tx > zkbal::AN_MAX_TX) {
        zk_set_error("%s: n_accounts = %zu, n_tx = %zu: at most %u accounts and %u transactions", a.fn, a.n_accounts, a.n_tx, zkbal::BAL_MAX,
                     zkbal::AN_MAX_TX);
        return ZK_ERR_INVALID;
    }
    return ZK_OK;
}

// ---- the host forms' staging --------------------------------------------------------------------------------------------
// stage(io, h, d): d = h with every array registered in io, which puts its device copy in its place
static void stage(Stage &io, const ConfIn &h, ConfIn &d) {
    const size_t na = h.n_accounts, n = h.n_tx;
    d = h;
    io.in(h.balances, d.balances, 64 * na); io.in(h.pendings, d.pendings, 64 * na); io.in(h.acct_flags, d.acct_flags, na);
    io.in(h.sender, d.sender, n); io.in(h.recipient, d.recipient, n);
    io.in(h.rows, d.rows, IMP_ROW * n); io.in(h.proofs, d.proofs, 192 * n);
    io.out(h.verdicts, d.verdicts, n); io.out(h.balance_after, d.balance_after, 64 * n); io.out(h.tx_status, d.tx_status, n);
    io.out(h.new_balances, d.new_balances, 64 * na); io.out(h.new_pendings, d.new_pendings, 64 * na);
    io.out(h.new_flags, d.new_flags, na);
}
// the grown table has room for a new row at every reference; *n_out of its rows come down
static void stage(Stage &io, const AssetIn &h, AssetIn &d, size_t *n_out) {
    const size_t ns = h.n_slots, n = h.n_tx, nr = h.n_slots + 2 * h.n_tx;
    d = h;
    d.n_slots_out = n_out;
    io.in(h.slot_ids, d.slot_ids, ns); io.in(h.slot_keys, d.slot_keys, 32 * ns); io.in(h.balances, d.balances, 64 * ns);
    io.in(h.pendings, d.pendings, 64 * ns); io.in(h.slot_flags, d.slot_flags, ns);
    io.in(h.kind, d.kind, n); io.in(h.asset_id, d.asset_id, n); io.in(h.rows, d.rows, IMP_ROW * n); io.in(h.proofs, d.proofs, 192 * n);
    io.out(h.verdicts, d.verdicts, n); io.out(h.asset_ids, d.asset_ids, n);
    io.out(h.balance_after, d.balance_after, 64 * n); io.out(h.event_ct, d.event_ct, 128 * n);
    io.out(h.event_flags, d.event_flags, n); io.out(h.tx_status, d.tx_status, n);
    io.out(h.new_slot_ids, d.new_slot_ids, nr, n_out); io.out(h.new_slot_keys, d.new_slot_keys, 32 * nr, n_out, 32);
    io.out(h.new_balances, d.new_balances, 64 * nr, n_out, 64); io.out(h.new_pendings, d.new_pendings, 64 * nr, n_out, 64);
    io.out(h.new_flags, d.new_flags, nr, n_out);
}
static void stage(Stage &io, const AnonIn &h, AnonIn &d) {
    const size_t na = h.n_accounts, n = h.n_tx;
    d = h;
    io.in(h.keys, d.keys, 32 * na); io.in(h.balances, d.balances, 64 * na); io.in(h.pendings, d.pendings, 64 * na);
    io.in(h.acct_flags, d.acct_flags, na); io.in(h.kind, d.kind, n); io.in(h.members, d.members, IMP_AN_RING * n);
    io.in(h.tx_points, d.tx_points, 32 * (size_t)IMP_AN_TX_POINTS * n); io.in(h.tx_extra, d.tx_extra, 64 * n);
    io.in(h.issue_fields, d.issue_fields, 96 * n); io.in(h.g_epoch, d.g_epoch, n ? 32 : 0); io.in(h.proofs, d.proofs, 192 * n);
    io.out(h.verdicts, d.verdicts, n); io.out(h.enc_balances, d.enc_balances, 64 * (size_t)IMP_AN_RING * n);
    io.out(h.issued, d.issued, 64 * n); io.out(h.tx_status, d.tx_status, n);
    io.out(h.new_balances, d.new_balances, 64 * na); io.out(h.new_pendings, d.new_pendings, 64 * na);
    io.out(h.new_flags, d.new_flags, na);
}

// ---- one block --------------------------------------------------------------------------------------------------------
static_assert(IMP_TRANSFER == zkbal::AS_TRANSFER && IMP_ISSUE == zkbal::AS_ISSUE && IMP_DESTROY == zkbal::AS_DESTROY,
              "import.cuh's kinds are assets.cuh's");
static_assert(IMP_AN_RING == zkbal::AN_RING && IMP_AN_ROW == 32 * zkbal::AN_VERIFY_POINTS, "import.cuh's ring layout is anon_balances.cuh's");
static_assert(IMP_AN_TRANSFER == zkbal::AN_TRANSFER && IMP_AN_ISSUE == zkbal::AN_ISSUE, "import.cuh's kinds are anon_balances.cuh's");

// the asset section's passes in front of its rounds (import.cuh section 6), in ctx->imp_as
struct AsWork {
    uint8_t *ref_on, *tx_points, *balances, *pendings, *flags;
    uint32_t *pos, *ipos, *ref_id, *newpos, *table, *slot_a, *slot_b;
};
// n_rows = n_slots + 2 n_tx: the table grown by a new row at every reference at most
static size_t carve(Carve &c, AsWork &w, size_t n_tx, size_t n_rows, size_t cap) {
    w.pos = c.take<uint32_t>(n_tx); w.ipos = c.take<uint32_t>(n_tx); w.ref_id = c.take<uint32_t>(2 * n_tx); w.ref_on = c.take<uint8_t>(2 * n_tx);
    w.newpos = c.take<uint32_t>(2 * n_tx); w.table = c.take<uint32_t>(cap); w.slot_a = c.take<uint32_t>(n_tx); w.slot_b = c.take<uint32_t>(n_tx);
    w.tx_points = c.take<uint8_t>(128 * n_tx);
    w.balances = c.take<uint8_t>(64 * n_rows); w.pendings = c.take<uint8_t>(64 * n_rows); w.flags = c.take<uint8_t>(n_rows);
    return c.off;
}
// the anonymous section's transfer verification (52 points) and its issue flags
struct AnonWork {
    uint8_t *verify_points, *rows, *round_proofs, *rv;
    uint32_t *pos;
};
static void carve(Carve &c, AnonWork &w, size_t n_tx) {
    w.verify_points = c.take<uint8_t>(IMP_AN_ROW * n_tx); w.rows = c.take<uint8_t>(IMP_AN_ROW * n_tx);
    w.round_proofs = c.take<uint8_t>(192 * n_tx); w.rv = c.take<uint8_t>(n_tx); w.pos = c.take<uint32_t>(n_tx);
}

// The schedule of the engine's comment over the sections present (NULL: absent; a section with no rows and no
// transactions is absent).  All arrays are device pointers.  A bad signature returns before any output is written: the
// sections' passes up to the signature check write the workspace only.
static int block_run(zk_ctx *ctx, const zk_pvk *conf_pvk, const zk_pvk *anon_pvk, const SigIn *sg, const ConfIn *ci, const AssetIn *ai,
                     const AnonIn *ni, size_t *first_bad_sig, unsigned *launches) {
    cudaStream_t st = ctx->stream;
    const size_t n_sig = sg ? sg->n : 0, nc = ci ? ci->n_tx : 0, na = ai ? ai->n_tx : 0, nn = ni ? ni->n_tx : 0;
    unsigned n_launch = 0;
    if (launches) *launches = 0;
    if (first_bad_sig) *first_bad_sig = n_sig;

    // the sections' workspace
    Joint J;
    RoundSec C, A;
    AnonWork nw{};
    AsWork aw{};
    uint8_t *sig_v = nullptr;
    size_t ns = ai ? ai->n_slots : 0;                // the asset table's rows, grown after L1
    const size_t n_ref = 2 * na, max_rows = ns + n_ref, cap = ZK_IAS_CAPACITY(max_rows);
    if (ci) {
        C.fn = ci->fn; C.n_keys = ci->n_accounts; C.n_tx = nc; C.key_a = ci->sender; C.key_b = ci->recipient; C.rows = ci->rows;
        C.proofs = ci->proofs; C.verdicts = ci->verdicts; C.cb = BC_CONF;
        C.state = [ctx, ci](const RoundSec &s) -> int {
            // balance_after is written for applied transfers only, and a later round may apply fewer
            if (s.n_tx) ZK_CUDA(cudaMemsetAsync(ci->balance_after, 0, 64 * s.n_tx, ctx->stream));
            return zk_balances_confidential_block_device(ctx, ci->n_accounts, ci->balances, ci->pendings, ci->acct_flags, s.n_tx, ci->sender,
                                                         ci->recipient, s.tx_points, s.applied, s.balance_sender, ci->balance_after,
                                                         ci->tx_status, ci->new_balances, ci->new_pendings, ci->new_flags);
        };
    }
    if (ai) {
        A.fn = ai->fn; A.n_keys = max_rows; A.n_tx = na; A.kind = ai->kind; A.key_a = aw.slot_a; A.key_b = aw.slot_b; A.rows = ai->rows;
        A.proofs = ai->proofs; A.fixed = ai->verdicts; A.verdicts = ai->verdicts; A.cb = BC_ASSETS;
    }
    auto carve_all = [&](Carve &c) {
        carve(c, J, nc + na + nn);
        if (ci) carve(c, C, true, ci->n_accounts);
        if (ai) carve(c, A, false, max_rows);
        if (ni) carve(c, nw, nn);
        sig_v = c.take<uint8_t>(n_sig);
        return c.off;
    };
    Carve sizing;
    ZK_TRY(ctx->imp.reserve(carve_all(sizing)));
    Carve c{ctx->imp.as<uint8_t>(), 0};
    carve_all(c);
    if (ai) {
        Carve as_sizing;
        ZK_TRY(ctx->imp_as.reserve(carve(as_sizing, aw, na, max_rows, cap)));
        Carve ac{ctx->imp_as.as<uint8_t>(), 0};
        carve(ac, aw, na, max_rows, cap);
        A.key_a = aw.slot_a; A.key_b = aw.slot_b;
        A.state = [ctx, ai, &aw, &ns](const RoundSec &s) -> int {
            // balance_after and the events are written for applied transactions only, and a later round may apply fewer
            if (s.n_tx) {
                ZK_CUDA(cudaMemsetAsync(ai->balance_after, 0, 64 * s.n_tx, ctx->stream));
                ZK_CUDA(cudaMemsetAsync(ai->event_ct, 0, 128 * s.n_tx, ctx->stream));
                ZK_CUDA(cudaMemsetAsync(ai->event_flags, 0, s.n_tx, ctx->stream));
            }
            return zk_assets_block_device(ctx, ns, aw.balances, aw.pendings, aw.flags, s.n_tx, ai->kind, aw.slot_a, aw.slot_b, aw.tx_points,
                                          s.applied, s.balance_sender, ai->balance_after, ai->event_ct, ai->event_flags, ai->tx_status,
                                          ai->new_balances, ai->new_pendings, ai->new_flags);
        };
    }
    const ImpAsKeys keys{ai ? ai->slot_ids : nullptr, ai ? ai->slot_keys : nullptr, aw.ref_id, ai ? ai->rows : nullptr, (uint32_t)ns};
    uint32_t *const as_cnt = J.cnt + BC_AS_FRONT, *const an_cnt = J.cnt + BC_ANON;
    uint32_t hc[BC_WORDS];

    // 1. the signatures' batch check, and every section's kinds and indices; nothing but workspace is written
    ZK_CUDA(cudaMemsetAsync(J.cnt, 0, BC_WORDS * sizeof(uint32_t), st));
    if (n_sig) {
        ZK_CUDA(cudaMemsetAsync(J.cnt + BC_SIG_BAD_Z, 0xFF, sizeof(uint32_t), st));
        k_imp_sig_z<<<grid(n_sig), BT, 0, st>>>(n_sig, sg->zs, J.cnt + BC_SIG_BAD_Z);
        ZK_CUDA(cudaGetLastError());
        ZK_TRY(zk_redjubjub_batch_verify_device(ctx, n_sig, sg->vks, sg->sigs, sg->msgs, sg->msg_off, sg->zs,
                                                reinterpret_cast<uint8_t *>(J.cnt + BC_SIG_VERDICT),
                                                reinterpret_cast<uint64_t *>(J.cnt + BC_SIG_FIRST)));
    }
    if (ci) ZK_TRY(round_start(ctx, C, J, J.rv));    // the start verdicts (all undecided) to scratch: verdicts waits for the signatures
    if (ai) {
        ZK_CUDA(cudaMemsetAsync(as_cnt + IMP_AS_BAD, 0xFF, (IMP_AS_COUNTERS - IMP_AS_BAD) * sizeof(uint32_t), st));
        ZK_CUDA(cudaMemsetAsync(aw.table, 0xFF, cap * sizeof(uint32_t), st));
        if (na) k_imp_as_start<<<grid(na), BT, 0, st>>>(na, ai->kind, aw.pos, as_cnt);
        k_imp_as_row_insert<<<grid(ns), BT, 0, st>>>(ns, keys, aw.table, (uint32_t)cap);
        k_imp_as_row_dup<<<grid(ns), BT, 0, st>>>(ns, keys, aw.table, (uint32_t)cap, as_cnt);
        ZK_CUDA(cudaGetLastError());
    }
    if (nn) {
        ZK_CUDA(cudaMemsetAsync(an_cnt + IMP_BAD, 0xFF, sizeof(uint32_t), st));
        k_imp_an_start<<<grid(nn), BT, 0, st>>>(nn, (uint32_t)ni->n_accounts, conf_pvk && ni->issue_fields, ni->kind, ni->members, nw.pos,
                                                an_cnt);
        ZK_CUDA(cudaGetLastError());
    }
    ZK_TRY(read_counters(ctx, J.cnt, hc));
    if (ci) ZK_TRY(round_join(C, hc));
    if (ai) {
        if (hc[BC_AS_FRONT + IMP_AS_BAD] != IMP_NONE) {
            zk_set_error("%s: transaction %u: an unknown kind", ai->fn, hc[BC_AS_FRONT + IMP_AS_BAD]);
            return ZK_ERR_INVALID;
        }
        if (hc[BC_AS_FRONT + IMP_AS_DUP] != IMP_NONE) {
            zk_set_error("%s: slot row %u repeats an earlier row's (asset id, key)", ai->fn, hc[BC_AS_FRONT + IMP_AS_DUP]);
            return ZK_ERR_INVALID;
        }
    }
    if (nn && hc[BC_ANON + IMP_BAD] != IMP_NONE) {
        zk_set_error("%s: transaction %u: an index out of range, an unknown kind, or an issue without conf_pvk and issue_fields", ni->fn,
                     hc[BC_ANON + IMP_BAD]);
        return ZK_ERR_INVALID;
    }
    // every z_i first, as zk_redjubjub_batch_verify checks them; then redjubjub_verify_batched: when the batch check
    // fails, the per-signature verdicts decide
    if (n_sig && hc[BC_SIG_BAD_Z] != IMP_NONE) {
        zk_set_error("zk_import_block: z[%u] >= r_J", hc[BC_SIG_BAD_Z]);
        return ZK_ERR_NOT_CANONICAL;
    }
    if (n_sig && reinterpret_cast<const uint8_t *>(hc + BC_SIG_VERDICT)[0] != 1) {
        ZK_TRY(zk_redjubjub_verify_batch_device(ctx, n_sig, sg->vks, sg->sigs, sg->msgs, sg->msg_off, sig_v));
        ZK_CUDA(cudaMemsetAsync(J.cnt + BC_SIG_LOWEST, 0xFF, sizeof(uint32_t), st));
        k_imp_sig_first<<<grid(n_sig), BT, 0, st>>>(n_sig, sig_v, J.cnt + BC_SIG_LOWEST);
        k_imp_sig_code<<<1, 1, 0, st>>>(sig_v, J.cnt + BC_SIG_LOWEST, J.cnt + BC_SIG_CODE);
        ZK_CUDA(cudaGetLastError());
        ZK_TRY(read_counters(ctx, J.cnt, hc));
        const uint32_t lo = hc[BC_SIG_LOWEST];
        if (lo != IMP_NONE) {
            if (first_bad_sig) *first_bad_sig = lo;
            zk_set_error("zk_import_block: extrinsic %u: bad signature (verdict %u)", lo, hc[BC_SIG_CODE]);
            return ZK_ERR_BAD_SIGNATURE;
        }
    }

    // 2. L1: the confidential transfers' first round, the asset issues and destroys, the anonymous issues
    const size_t m_fixed = na ? hc[BC_AS_FRONT + IMP_AS_FIXED] : 0, n_iss = nn ? hc[BC_ANON + IMP_ISSUES] : 0,
                 n_tr = nn ? hc[BC_ANON + IMP_TRANSFERS] : 0;
    if (nc) ZK_CUDA(cudaMemsetAsync(ci->verdicts, IMP_UNDECIDED, nc, st));
    if (na) {
        ZK_CUDA(cudaMemsetAsync(ai->verdicts, 0, na, st));      // transfers 0 until the rounds start them
        if (m_fixed) ZK_TRY(zk_bal_prefix_sum(ctx, aw.pos, na, J.totals));
    }
    if (nn) {
        // transfers start unapplied; issued holds zero bytes where no applied issue writes
        ZK_CUDA(cudaMemsetAsync(ni->verdicts, 0, nn, st));
        ZK_CUDA(cudaMemsetAsync(ni->issued, 0, 64 * nn, st));
        if (n_iss) ZK_TRY(zk_bal_prefix_sum(ctx, nw.pos, nn, J.totals));
    }
    auto l1_gather = [&](size_t off) -> int {
        if (m_fixed)
            k_imp_as_compact<<<grid(IMP_WORDS * na), BT, 0, st>>>(IMP_WORDS * na, ai->kind, aw.pos, ai->rows, ai->proofs, J.round_rows,
                                                                   J.round_proofs, off);
        if (n_iss)
            k_imp_an_issue_row<<<grid(IMP_AN_ISSUE_WORDS * nn), BT, 0, st>>>(IMP_AN_ISSUE_WORDS * nn, ni->kind, nw.pos, ni->keys, ni->members,
                                                                             ni->tx_points, ni->issue_fields, ni->tx_extra, ni->g_epoch,
                                                                             ni->proofs, J.round_rows, J.round_proofs, off + m_fixed);
        ZK_CUDA(cudaGetLastError());
        return ZK_OK;
    };
    auto l1_scatter = [&](size_t off) -> int {
        if (m_fixed) k_imp_an_scatter<<<grid(na), BT, 0, st>>>(na, true, ai->kind, aw.pos, J.rv, ai->verdicts, off);
        if (n_iss) k_imp_an_scatter<<<grid(nn), BT, 0, st>>>(nn, true, ni->kind, nw.pos, J.rv, ni->verdicts, off + m_fixed);
        ZK_CUDA(cudaGetLastError());
        return ZK_OK;
    };
    RoundSec *const l1[1] = {&C};
    bool any;
    ZK_TRY(launch_round(ctx, conf_pvk, J, l1, ci ? 1 : 0, m_fixed + n_iss, l1_gather, l1_scatter, &n_launch, &any));

    // 3. the anonymous state passes and the 52-point launch (import.cuh section 5)
    if (ni) {
        // the issue verdicts, when there are issues, select the passes of zk_anonymous_calls_block; without issues the
        // state pass is zk_balances_anonymous_block's, as the Python driver runs it
        auto state = [&]() -> int {
            if (n_iss)
                return zk_anonymous_calls_block_device(ctx, ni->n_accounts, ni->keys, ni->balances, ni->pendings, ni->acct_flags, nn, ni->kind,
                                                       ni->members, ni->tx_points, ni->tx_extra, ni->g_epoch, ni->verdicts, ni->enc_balances,
                                                       nw.verify_points, ni->issued, ni->tx_status, ni->new_balances, ni->new_pendings,
                                                       ni->new_flags);
            return zk_balances_anonymous_block_device(ctx, ni->n_accounts, ni->keys, ni->balances, ni->pendings, ni->acct_flags, nn, ni->members,
                                                      ni->tx_points, ni->tx_extra, ni->g_epoch, ni->verdicts, ni->enc_balances, nw.verify_points,
                                                      ni->tx_status, ni->new_balances, ni->new_pendings, ni->new_flags);
        };
        ZK_TRY(state());
        if (nn && !n_iss) {
            // every transaction a transfer: verify the state pass's rows in place, the verdicts straight into the mask
            ++n_launch;
            ZK_TRY(zk_groth16_verify_points_batch_device(ctx, anon_pvk, nn, ni->proofs, nw.verify_points, zkbal::AN_VERIFY_POINTS, ni->verdicts));
            ZK_TRY(state());
        } else if (n_tr) {
            k_imp_an_gather<<<grid(IMP_AN_WORDS * nn), BT, 0, st>>>(IMP_AN_WORDS * nn, ni->kind, nw.pos, nw.verify_points, ni->proofs, nw.rows,
                                                                   nw.round_proofs);
            ZK_CUDA(cudaGetLastError());
            ++n_launch;
            ZK_TRY(zk_groth16_verify_points_batch_device(ctx, anon_pvk, n_tr, nw.round_proofs, nw.rows, zkbal::AN_VERIFY_POINTS, nw.rv));
            k_imp_an_scatter<<<grid(nn), BT, 0, st>>>(nn, false, ni->kind, nw.pos, nw.rv, ni->verdicts, 0);
            ZK_CUDA(cudaGetLastError());
            ZK_TRY(state());
        }
    }

    // 4. the asset ids, references and slots (import.cuh section 6), and the start of the asset rounds
    if (ai) {
        if (na) {
            k_imp_as_issue_flag<<<grid(na), BT, 0, st>>>(na, ai->kind, ai->verdicts, aw.ipos);
            ZK_CUDA(cudaGetLastError());
            ZK_TRY(zk_bal_prefix_sum(ctx, aw.ipos, na, J.totals));
            k_imp_as_refs<<<grid(na), BT, 0, st>>>(na, ai->next_asset_id, ai->kind, ai->asset_id, ai->verdicts, aw.ipos, ai->asset_ids, aw.ref_id,
                                                   aw.ref_on, as_cnt);
            // the references into the hash table; new rows numbered in the order of their first reference
            k_imp_as_ref_insert<<<grid(n_ref), BT, 0, st>>>(n_ref, aw.ref_on, keys, aw.table, (uint32_t)cap);
            k_imp_as_new<<<grid(n_ref), BT, 0, st>>>(n_ref, aw.ref_on, keys, aw.table, (uint32_t)cap, aw.newpos, as_cnt);
            ZK_CUDA(cudaGetLastError());
            ZK_TRY(zk_bal_prefix_sum(ctx, aw.newpos, n_ref, J.totals));
        }
        // the table's rows, then the new ones behind them
        if (ns) {
            ZK_CUDA(cudaMemcpyAsync(aw.balances, ai->balances, 64 * ns, cudaMemcpyDeviceToDevice, st));
            ZK_CUDA(cudaMemcpyAsync(aw.pendings, ai->pendings, 64 * ns, cudaMemcpyDeviceToDevice, st));
            ZK_CUDA(cudaMemcpyAsync(aw.flags, ai->slot_flags, ns, cudaMemcpyDeviceToDevice, st));
            ZK_CUDA(cudaMemcpyAsync(ai->new_slot_ids, ai->slot_ids, 4 * ns, cudaMemcpyDeviceToDevice, st));
            ZK_CUDA(cudaMemcpyAsync(ai->new_slot_keys, ai->slot_keys, 32 * ns, cudaMemcpyDeviceToDevice, st));
        }
        if (na) {
            const uint8_t flags = (uint8_t)(ai->new_slot_flags & ~(zkbal::ACCT_BALANCE | zkbal::ACCT_PENDING));
            k_imp_as_slot<<<grid(n_ref), BT, 0, st>>>(n_ref, aw.ref_on, keys, aw.table, (uint32_t)cap, aw.newpos, flags, aw.slot_a, aw.slot_b,
                                                      ai->new_slot_ids, ai->new_slot_keys, aw.balances, aw.pendings, aw.flags);
            k_imp_as_tx_points<<<grid(32 * na), BT, 0, st>>>(32 * na, ai->kind, ai->rows, aw.tx_points);
            ZK_CUDA(cudaGetLastError());
        }
        // the issue and destroy verdicts fixed in verdicts itself; every slot is a row of the grown table (< max_rows)
        ZK_TRY(round_start(ctx, A, J, ai->verdicts));
    }
    if (C.in_launch || ai) {                       // the anonymous section needs no read
        ZK_TRY(read_counters(ctx, J.cnt, hc));
        round_decided(l1, ci ? 1 : 0, hc);
    }
    if (ai) {
        if (na && hc[BC_AS_FRONT + IMP_AS_OVF] != IMP_NONE) {
            zk_set_error("%s: transaction %u: the issue's asset id would pass 2^32 - 1", ai->fn, hc[BC_AS_FRONT + IMP_AS_OVF]);
            return ZK_ERR_INVALID;
        }
        ns += na ? hc[BC_AS_FRONT + IMP_AS_NEW] : 0;
        if (ns > zkbal::BAL_MAX) {
            zk_set_error("%s: %zu slots after the block's new ones: at most %u", ai->fn, ns, zkbal::BAL_MAX);
            return ZK_ERR_INVALID;
        }
        *ai->n_slots_out = ns;
        A.n_keys = ns;
        ZK_TRY(round_join(A, hc));
    }

    // 5. the later launches: both chain-keyed sections' undecided transfers
    RoundSec *const rest[2] = {ci ? &C : &A, &A};
    ZK_TRY(rounds_rest(ctx, conf_pvk, J, rest, (ci ? 1 : 0) + (ai ? 1 : 0), &n_launch));
    if (ci && ci->rounds) *ci->rounds = C.rounds;
    if (ai && ai->rounds) *ai->rounds = A.rounds;
    if (launches) *launches = n_launch;
    return ZK_OK;
}

// The host forms: every section staged in ctx->io, the engine, the outputs back.  The messages go up from the first
// one, their offsets counted from it.
static int host_run(zk_ctx *ctx, const zk_pvk *conf_pvk, const zk_pvk *anon_pvk, const SigIn *sg, const ConfIn *ci, const AssetIn *ai,
                    const AnonIn *ni, size_t *first_bad_sig, unsigned *launches) {
    SigIn ds{};
    ConfIn dc{};
    AssetIn da{};
    AnonIn dn{};
    size_t n_out = 0;
    std::vector<uint64_t> off;
    Stage io;
    if (sg) {
        ds.n = sg->n;
        for (size_t i = 0; i <= sg->n; i++) off.push_back(sg->msg_off[i] - sg->msg_off[0]);
        io.in(sg->vks, ds.vks, 32 * sg->n); io.in(sg->sigs, ds.sigs, 64 * sg->n); io.in(sg->zs, ds.zs, 32 * sg->n);
        io.in(sg->msgs + sg->msg_off[0], ds.msgs, off[sg->n]); io.in(off.data(), ds.msg_off, sg->n + 1);
    }
    if (ci) stage(io, *ci, dc);
    if (ai) stage(io, *ai, da, &n_out);
    if (ni) stage(io, *ni, dn);
    ZK_TRY(io.up(ctx));
    ZK_TRY(block_run(ctx, conf_pvk, anon_pvk, sg ? &ds : nullptr, ci ? &dc : nullptr, ai ? &da : nullptr, ni ? &dn : nullptr, first_bad_sig,
                     launches));
    ZK_TRY(io.down(ctx));
    ZK_CUDA(cudaStreamSynchronize(ctx->stream));
    if (ai) *ai->n_slots_out = n_out;
    return ZK_OK;
}

// Argument checks, then the engine over the sections that have rows or transactions.  conf_pvk / anon_pvk: NULL where no
// section needs them; each key passed is checked.
static int import_entry(bool device, const char *fn, zk_ctx *ctx, const zk_pvk *conf_pvk, const zk_pvk *anon_pvk, const SigIn *sg,
                        const ConfIn *ci, const AssetIn *ai, const AnonIn *ni, size_t *first_bad_sig, unsigned *launches) {
    if (!ctx) return null_arg(fn);
    if (sg && sg->n) {
        if (!sg->vks || !sg->sigs || !sg->msgs || !sg->msg_off || !sg->zs) return null_arg(fn);
        for (size_t i = 0; i < sg->n && !device; i++)
            if (sg->msg_off[i + 1] < sg->msg_off[i]) {
                zk_set_error("%s: msg_off[%zu] = %llu > msg_off[%zu] = %llu", fn, i, (unsigned long long)sg->msg_off[i], i + 1,
                             (unsigned long long)sg->msg_off[i + 1]);
                return ZK_ERR_INVALID;
            }
    }
    if (ci) ZK_TRY(conf_args(*ci));
    if (ai) ZK_TRY(asset_args(*ai));
    if (ni) ZK_TRY(anon_args(*ni));
    if (ci && ci->n_tx && !conf_pvk) return null_arg(ci->fn);
    if (ai && ai->n_tx && !conf_pvk) return null_arg(ai->fn);
    if (ni && ni->n_tx && !anon_pvk) return null_arg(ni->fn);
    if (anon_pvk) ZK_TRY(check_key(ctx, anon_pvk, zkbal::AN_VERIFY_POINTS));
    if (conf_pvk) ZK_TRY(check_key(ctx, conf_pvk));
    if (ci && ci->rounds) *ci->rounds = 0;
    if (ai && ai->rounds) *ai->rounds = 0;
    if (ai) *ai->n_slots_out = 0;
    if (launches) *launches = 0;
    if (first_bad_sig) *first_bad_sig = sg ? sg->n : 0;
    if (ci && !ci->n_accounts && !ci->n_tx) ci = nullptr;
    if (ai && !ai->n_slots && !ai->n_tx) ai = nullptr;
    if (ni && !ni->n_accounts && !ni->n_tx) ni = nullptr;
    if (sg && !sg->n) sg = nullptr;
    if (!sg && !ci && !ai && !ni) return ZK_OK;
    ZK_TRY(zk_use_device(ctx));
    return (device ? block_run : host_run)(ctx, conf_pvk, anon_pvk, sg, ci, ai, ni, first_bad_sig, launches);
}

// ---- the C ABI ----------------------------------------------------------------------------------------------------------
#define CONF_PARAMS(P)                                                                                                                   \
    size_t n_accounts, const uint8_t *P##balances, const uint8_t *P##pendings, const uint8_t *P##acct_flags, size_t n_tx,                \
        const uint32_t *P##sender, const uint32_t *P##recipient, const uint8_t *P##rows, const uint8_t *P##proofs, uint8_t *P##verdicts, \
        uint8_t *P##balance_after, uint8_t *P##tx_status, uint8_t *P##new_balances, uint8_t *P##new_pendings, uint8_t *P##new_flags,     \
        unsigned *rounds
#define CONF_IN(fn, P)                                                                                                                  \
    ConfIn { fn, n_accounts, P##balances, P##pendings, P##acct_flags, n_tx, P##sender, P##recipient, P##rows, P##proofs, P##verdicts, \
             P##balance_after, P##tx_status, P##new_balances, P##new_pendings, P##new_flags, rounds }

extern "C" int zk_import_confidential_block_device(zk_ctx *ctx, const zk_pvk *pvk, CONF_PARAMS(d_)) {
    const ConfIn c = CONF_IN("zk_import_confidential_block_device", d_);
    if (!pvk) return null_arg(c.fn);
    return import_entry(true, c.fn, ctx, pvk, nullptr, nullptr, &c, nullptr, nullptr, nullptr, nullptr);
}
extern "C" int zk_import_confidential_block(zk_ctx *ctx, const zk_pvk *pvk, CONF_PARAMS()) {
    const ConfIn c = CONF_IN("zk_import_confidential_block", );
    if (!pvk) return null_arg(c.fn);
    return import_entry(false, c.fn, ctx, pvk, nullptr, nullptr, &c, nullptr, nullptr, nullptr, nullptr);
}

// zk_import_assets_block: the caller's slots and issue / destroy verdicts, so only the rounds, as one section
static int assets_run(zk_ctx *ctx, const char *fn, const zk_pvk *pvk, size_t n_slots, const uint8_t *balances, const uint8_t *pendings,
                      const uint8_t *slot_flags, size_t n_tx, const uint8_t *kind, const uint32_t *slot_a, const uint32_t *slot_b,
                      const uint8_t *tx_points, const uint8_t *rows, const uint8_t *proofs, const uint8_t *fixed_verdicts, uint8_t *verdicts,
                      uint8_t *balance_after, uint8_t *event_ct, uint8_t *event_flags, uint8_t *tx_status, uint8_t *new_balances,
                      uint8_t *new_pendings, uint8_t *new_flags, unsigned *rounds) {
    Joint J;
    RoundSec A;
    A.fn = fn; A.n_keys = n_slots; A.n_tx = n_tx; A.kind = kind; A.key_a = slot_a; A.key_b = slot_b; A.rows = rows; A.proofs = proofs;
    A.fixed = fixed_verdicts; A.verdicts = verdicts; A.cb = BC_ASSETS;
    A.state = [&](const RoundSec &s) -> int {
        // balance_after and the events are written for applied transactions only, and a later round may apply fewer
        if (n_tx) {
            ZK_CUDA(cudaMemsetAsync(balance_after, 0, 64 * n_tx, ctx->stream));
            ZK_CUDA(cudaMemsetAsync(event_ct, 0, 128 * n_tx, ctx->stream));
            ZK_CUDA(cudaMemsetAsync(event_flags, 0, n_tx, ctx->stream));
        }
        return zk_assets_block_device(ctx, n_slots, balances, pendings, slot_flags, n_tx, kind, slot_a, slot_b, tx_points, s.applied,
                                      s.balance_sender, balance_after, event_ct, event_flags, tx_status, new_balances, new_pendings, new_flags);
    };
    auto carve_all = [&](Carve &c) {
        carve(c, J, n_tx);
        carve(c, A, false, n_slots);
        return c.off;
    };
    Carve sizing;
    ZK_TRY(ctx->imp.reserve(carve_all(sizing)));
    Carve c{ctx->imp.as<uint8_t>(), 0};
    carve_all(c);
    uint32_t hc[BC_WORDS];
    unsigned launches = 0;
    ZK_TRY(round_start(ctx, A, J, verdicts));
    if (n_tx) ZK_TRY(read_counters(ctx, J.cnt, hc));
    ZK_TRY(round_join(A, hc));
    RoundSec *const secs[1] = {&A};
    ZK_TRY(rounds_rest(ctx, pvk, J, secs, 1, &launches));
    if (rounds) *rounds = A.rounds;
    return ZK_OK;
}

static int assets_block_args(const char *fn, zk_ctx *ctx, const zk_pvk *pvk, size_t n_slots, const void *balances, const void *pendings,
                             const void *slot_flags, size_t n_tx, const void *kind, const void *slot_a, const void *slot_b,
                             const void *tx_points, const void *rows, const void *proofs, const void *fixed_verdicts, const void *verdicts,
                             const void *balance_after, const void *event_ct, const void *event_flags, const void *tx_status,
                             const void *new_balances, const void *new_pendings, const void *new_flags) {
    if (!ctx || !pvk || (n_slots && (!balances || !pendings || !slot_flags || !new_balances || !new_pendings || !new_flags)) ||
        (n_tx && (!kind || !slot_a || !slot_b || !tx_points || !rows || !proofs || !fixed_verdicts || !verdicts || !balance_after ||
                  !event_ct || !event_flags || !tx_status)))
        return null_arg(fn);
    if (n_slots > zkbal::BAL_MAX || n_tx > zkbal::AS_MAX_TX) {
        zk_set_error("%s: n_slots = %zu, n_tx = %zu: at most %u slots and %u transactions", fn, n_slots, n_tx, zkbal::BAL_MAX,
                     zkbal::AS_MAX_TX);
        return ZK_ERR_INVALID;
    }
    return ZK_OK;
}
extern "C" int zk_import_assets_block_device(zk_ctx *ctx, const zk_pvk *pvk, size_t n_slots, const uint8_t *d_balances,
                                             const uint8_t *d_pendings, const uint8_t *d_slot_flags, size_t n_tx, const uint8_t *d_kind,
                                             const uint32_t *d_slot_a, const uint32_t *d_slot_b, const uint8_t *d_tx_points,
                                             const uint8_t *d_rows, const uint8_t *d_proofs, const uint8_t *d_fixed_verdicts,
                                             uint8_t *d_verdicts, uint8_t *d_balance_after, uint8_t *d_event_ct, uint8_t *d_event_flags,
                                             uint8_t *d_tx_status, uint8_t *d_new_balances, uint8_t *d_new_pendings, uint8_t *d_new_flags,
                                             unsigned *rounds) {
    const char *fn = "zk_import_assets_block_device";
    ZK_TRY(assets_block_args(fn, ctx, pvk, n_slots, d_balances, d_pendings, d_slot_flags, n_tx, d_kind, d_slot_a, d_slot_b, d_tx_points, d_rows,
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
    ZK_TRY(assets_block_args(fn, ctx, pvk, n_slots, balances, pendings, slot_flags, n_tx, kind, slot_a, slot_b, tx_points, rows, proofs,
                       fixed_verdicts, verdicts, balance_after, event_ct, event_flags, tx_status, new_balances, new_pendings, new_flags));
    ZK_TRY(check_key(ctx, pvk));
    if (rounds) *rounds = 0;
    if (!n_slots && !n_tx) return ZK_OK;
    ZK_TRY(zk_use_device(ctx));
    const uint8_t *b, *p, *f, *kd, *tp, *rw, *pf, *fx;
    const uint32_t *sa, *sb;
    uint8_t *v, *ba, *ev, *ef, *ts, *nb, *npd, *nf;
    Stage io;
    io.in(balances, b, 64 * n_slots); io.in(pendings, p, 64 * n_slots); io.in(slot_flags, f, n_slots);
    io.in(slot_a, sa, n_tx); io.in(slot_b, sb, n_tx); io.in(kind, kd, n_tx); io.in(tx_points, tp, 128 * n_tx);
    io.in(rows, rw, IMP_ROW * n_tx); io.in(proofs, pf, 192 * n_tx); io.in(fixed_verdicts, fx, n_tx);
    io.out(verdicts, v, n_tx); io.out(balance_after, ba, 64 * n_tx); io.out(event_ct, ev, 128 * n_tx); io.out(event_flags, ef, n_tx);
    io.out(tx_status, ts, n_tx);
    io.out(new_balances, nb, 64 * n_slots); io.out(new_pendings, npd, 64 * n_slots); io.out(new_flags, nf, n_slots);
    ZK_TRY(io.up(ctx));
    ZK_TRY(assets_run(ctx, fn, pvk, n_slots, b, p, f, n_tx, kd, sa, sb, tp, rw, pf, fx, v, ba, ev, ef, ts, nb, npd, nf, rounds));
    ZK_TRY(io.down(ctx));
    ZK_CUDA(cudaStreamSynchronize(ctx->stream));
    return ZK_OK;
}

#define ASSET_PARAMS(P)                                                                                                                 \
    size_t n_slots, const uint32_t *P##slot_ids, const uint8_t *P##slot_keys, const uint8_t *P##balances, const uint8_t *P##pendings,  \
        const uint8_t *P##slot_flags, uint32_t next_asset_id, uint8_t new_slot_flags, size_t n_tx, const uint8_t *P##kind,              \
        const uint32_t *P##asset_id, const uint8_t *P##rows, const uint8_t *P##proofs, uint8_t *P##verdicts, uint32_t *P##asset_ids,   \
        uint8_t *P##balance_after, uint8_t *P##event_ct, uint8_t *P##event_flags, uint8_t *P##tx_status, uint32_t *P##new_slot_ids,    \
        uint8_t *P##new_slot_keys, uint8_t *P##new_balances, uint8_t *P##new_pendings, uint8_t *P##new_flags, size_t *n_slots_out,      \
        unsigned *rounds
#define ASSET_IN(fn, P)                                                                                                                 \
    AssetIn { fn, n_slots, P##slot_ids, P##slot_keys, P##balances, P##pendings, P##slot_flags, next_asset_id, new_slot_flags, n_tx,   \
              P##kind, P##asset_id, P##rows, P##proofs, P##verdicts, P##asset_ids, P##balance_after, P##event_ct, P##event_flags,      \
              P##tx_status, P##new_slot_ids, P##new_slot_keys, P##new_balances, P##new_pendings, P##new_flags, n_slots_out, rounds }

extern "C" int zk_import_asset_calls_device(zk_ctx *ctx, const zk_pvk *pvk, ASSET_PARAMS(d_)) {
    const AssetIn a = ASSET_IN("zk_import_asset_calls_device", d_);
    if (!pvk) return null_arg(a.fn);
    return import_entry(true, a.fn, ctx, pvk, nullptr, nullptr, nullptr, &a, nullptr, nullptr, nullptr);
}
extern "C" int zk_import_asset_calls(zk_ctx *ctx, const zk_pvk *pvk, ASSET_PARAMS()) {
    const AssetIn a = ASSET_IN("zk_import_asset_calls", );
    if (!pvk) return null_arg(a.fn);
    return import_entry(false, a.fn, ctx, pvk, nullptr, nullptr, nullptr, &a, nullptr, nullptr, nullptr);
}

#define ANON_PARAMS(P)                                                                                                                 \
    size_t n_accounts, const uint8_t *P##keys, const uint8_t *P##balances, const uint8_t *P##pendings, const uint8_t *P##acct_flags,  \
        size_t n_tx, const uint8_t *P##kind, const uint32_t *P##members, const uint8_t *P##tx_points, const uint8_t *P##tx_extra,     \
        const uint8_t *P##issue_fields, const uint8_t *P##g_epoch, const uint8_t *P##proofs, uint8_t *P##verdicts,                    \
        uint8_t *P##enc_balances, uint8_t *P##issued, uint8_t *P##tx_status, uint8_t *P##new_balances, uint8_t *P##new_pendings,      \
        uint8_t *P##new_flags
#define ANON_IN(fn, P)                                                                                                                 \
    AnonIn { fn, n_accounts, P##keys, P##balances, P##pendings, P##acct_flags, n_tx, P##kind, P##members, P##tx_points, P##tx_extra, \
             P##issue_fields, P##g_epoch, P##proofs, P##verdicts, P##enc_balances, P##issued, P##tx_status, P##new_balances,         \
             P##new_pendings, P##new_flags }

extern "C" int zk_import_anonymous_block_device(zk_ctx *ctx, const zk_pvk *anon_pvk, const zk_pvk *conf_pvk, ANON_PARAMS(d_)) {
    const AnonIn n = ANON_IN("zk_import_anonymous_block_device", d_);
    if (!anon_pvk) return null_arg(n.fn);
    return import_entry(true, n.fn, ctx, conf_pvk, anon_pvk, nullptr, nullptr, nullptr, &n, nullptr, nullptr);
}
extern "C" int zk_import_anonymous_block(zk_ctx *ctx, const zk_pvk *anon_pvk, const zk_pvk *conf_pvk, ANON_PARAMS()) {
    const AnonIn n = ANON_IN("zk_import_anonymous_block", );
    if (!anon_pvk) return null_arg(n.fn);
    return import_entry(false, n.fn, ctx, conf_pvk, anon_pvk, nullptr, nullptr, nullptr, &n, nullptr, nullptr);
}

// zk_import_block: the parameters of each section carry its prefix (c_, a_, an_), its sizes too
#define BLOCK_PARAMS(P)                                                                                                                \
    zk_ctx *ctx, const zk_pvk *conf_pvk, const zk_pvk *anon_pvk, size_t n_sig, const uint8_t *P##vks, const uint8_t *P##sigs,        \
        const uint8_t *P##msgs, const uint64_t *P##msg_off, const uint8_t *P##zs, size_t c_n_accounts, const uint8_t *P##c_balances,  \
        const uint8_t *P##c_pendings, const uint8_t *P##c_acct_flags, size_t c_n_tx, const uint32_t *P##c_sender,                     \
        const uint32_t *P##c_recipient, const uint8_t *P##c_rows, const uint8_t *P##c_proofs, uint8_t *P##c_verdicts,                 \
        uint8_t *P##c_balance_after, uint8_t *P##c_tx_status, uint8_t *P##c_new_balances, uint8_t *P##c_new_pendings,                 \
        uint8_t *P##c_new_flags, unsigned *c_rounds, size_t a_n_slots, const uint32_t *P##a_slot_ids, const uint8_t *P##a_slot_keys,  \
        const uint8_t *P##a_balances, const uint8_t *P##a_pendings, const uint8_t *P##a_slot_flags, uint32_t a_next_asset_id,         \
        uint8_t a_new_slot_flags, size_t a_n_tx, const uint8_t *P##a_kind, const uint32_t *P##a_asset_id, const uint8_t *P##a_rows,   \
        const uint8_t *P##a_proofs, uint8_t *P##a_verdicts, uint32_t *P##a_asset_ids, uint8_t *P##a_balance_after,                    \
        uint8_t *P##a_event_ct, uint8_t *P##a_event_flags, uint8_t *P##a_tx_status, uint32_t *P##a_new_slot_ids,                      \
        uint8_t *P##a_new_slot_keys, uint8_t *P##a_new_balances, uint8_t *P##a_new_pendings, uint8_t *P##a_new_flags,                 \
        size_t *a_n_slots_out, unsigned *a_rounds, size_t an_n_accounts, const uint8_t *P##an_keys, const uint8_t *P##an_balances,    \
        const uint8_t *P##an_pendings, const uint8_t *P##an_acct_flags, size_t an_n_tx, const uint8_t *P##an_kind,                    \
        const uint32_t *P##an_members, const uint8_t *P##an_tx_points, const uint8_t *P##an_tx_extra, const uint8_t *P##an_issue_fields, \
        const uint8_t *P##an_g_epoch, const uint8_t *P##an_proofs, uint8_t *P##an_verdicts, uint8_t *P##an_enc_balances,              \
        uint8_t *P##an_issued, uint8_t *P##an_tx_status, uint8_t *P##an_new_balances, uint8_t *P##an_new_pendings,                    \
        uint8_t *P##an_new_flags, size_t *first_bad_sig, unsigned *launches
#define BLOCK_RUN(device, fn, P)                                                                                                       \
    do {                                                                                                                              \
        const SigIn s{n_sig, P##vks, P##sigs, P##msgs, P##msg_off, P##zs};                                                            \
        const ConfIn c{fn ": confidential", c_n_accounts, P##c_balances, P##c_pendings, P##c_acct_flags, c_n_tx, P##c_sender,          \
                       P##c_recipient, P##c_rows, P##c_proofs, P##c_verdicts, P##c_balance_after, P##c_tx_status, P##c_new_balances,   \
                       P##c_new_pendings, P##c_new_flags, c_rounds};                                                                  \
        const AssetIn a{fn ": assets", a_n_slots, P##a_slot_ids, P##a_slot_keys, P##a_balances, P##a_pendings, P##a_slot_flags,       \
                        a_next_asset_id, a_new_slot_flags, a_n_tx, P##a_kind, P##a_asset_id, P##a_rows, P##a_proofs, P##a_verdicts,    \
                        P##a_asset_ids, P##a_balance_after, P##a_event_ct, P##a_event_flags, P##a_tx_status, P##a_new_slot_ids,       \
                        P##a_new_slot_keys, P##a_new_balances, P##a_new_pendings, P##a_new_flags, a_n_slots_out, a_rounds};           \
        const AnonIn n{fn ": anonymous", an_n_accounts, P##an_keys, P##an_balances, P##an_pendings, P##an_acct_flags, an_n_tx,        \
                       P##an_kind, P##an_members, P##an_tx_points, P##an_tx_extra, P##an_issue_fields, P##an_g_epoch, P##an_proofs,    \
                       P##an_verdicts, P##an_enc_balances, P##an_issued, P##an_tx_status, P##an_new_balances, P##an_new_pendings,     \
                       P##an_new_flags};                                                                                              \
        return import_entry(device, fn, ctx, conf_pvk, anon_pvk, &s, &c, &a, &n, first_bad_sig, launches);                           \
    } while (0)

extern "C" int zk_import_block_device(BLOCK_PARAMS(d_)) { BLOCK_RUN(true, "zk_import_block_device", d_); }
extern "C" int zk_import_block(BLOCK_PARAMS()) { BLOCK_RUN(false, "zk_import_block", ); }
