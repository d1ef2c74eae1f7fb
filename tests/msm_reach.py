"""Reach model of the device MSM (zero_chain_b200/csrc/msm_driver.cuh): which branches of the sort, the batched-affine
rounds, the bucket accumulation and the bucket reduction a given MSM takes, computed on the host from its scalars.

The MSM tests use it to state, before they run, which branch a case is meant to reach ("bin 0 is staged with a direct
segment", "2 rounds", "k_rowcol_sums").  The constants below are copies of the kernels' constants; test_msm_reach.py reads
each of them out of the CUDA sources and fails when one moves, so a case cannot drift off its branch and keep passing.
Plain Python and numpy, no GPU."""
from dataclasses import dataclass, field

import numpy as np

# copies of the kernels' constants (checked against the sources by test_msm_reach.py)
FINE_STAGE = 25 * 1024            # msm.cuh: entries of k_fine_sort's shared-memory window
FINE_MAX_SEGMENTS = 4             # msm.cuh: a bin of more windows than this is scattered straight to HBM
COARSE_BINS = 512                 # msm.cuh: bins of the coarse level of the two-level sort (the high 9 key bits)
COARSE_CHUNK = 256 * 16           # msm.cuh: COARSE_THREADS * COARSE_PER_THREAD, the least coarse tile length
TASK_LEN_MAX = 64                 # msm_accum.cuh: target upper bound of additions per accumulation task
COMB_SERIAL_MAX = 32              # msm.cuh: buckets with more tasks than this are folded by k_combine_warp
BA_MAX_LEVELS = 8                 # msm_batchaff.cuh: most batched-affine rounds
BA_MIN_ENTRIES = 1 << 22          # internal.h: default ZK_OPT_AFFINE_MIN_ENTRIES
BA_AVG_MIN = 12                   # msm_driver.cuh: one more round while the average bucket length is >= this
ORDER_AVG_MAX = 256               # msm_driver.cuh: tasks are ordered by length when E / NB is below this
ROWCOL_MIN_DOMAINS = 8            # msm_driver.cuh: from this many domains on the reduction runs k_rowcol_sums
ROWCOL_MIN_C = 7                  # msm_driver.cuh: ... for windows of at least this many bits
TWO_LEVEL_MIN_C = 17              # msm_driver.cuh: windows above 16 bits sort in two levels
DIGIT_ZERO = 0xFFFFFFFF           # msm.cuh: code of a zero digit

R = 0x73EDA753299D7D483339D80809A1D80553BDA402FFFE5BFEFFFFFFFF00000001

# the longest task k_pick_task_len can choose
TASK_LEN_LIMIT = TASK_LEN_MAX + 8


def windows(c: int) -> int:
    return 255 // c + 1


def signed_digits(s: int, c: int) -> list:
    """Digit codes of scalar s for c-bit windows, as k_msm_digits writes them: W = 255 // c + 1 windows of signed digits
    d in (-2^(c-1), 2^(c-1)], coded (|d| - 1) | sign << 31, or DIGIT_ZERO."""
    half, full = 1 << (c - 1), 1 << c
    out, carry = [], 0
    for w in range(windows(c)):
        v = ((s >> (w * c)) & (full - 1)) + carry
        if v > half:                     # v = 2^c (all ones plus a carry) is digit 0 with a carry: the code wraps to DIGIT_ZERO
            out.append(((full - v - 1) | 0x80000000) & 0xFFFFFFFF)
            carry = 1
        else:
            out.append(v - 1 if v else DIGIT_ZERO)
            carry = 0
    return out


def digit_value(code: int) -> int:
    if code == DIGIT_ZERO:
        return 0
    m = (code & 0x7FFFFFFF) + 1
    return -m if code >> 31 else m


def recombine(codes, c: int) -> int:
    return sum(digit_value(k) << (c * w) for w, k in enumerate(codes))


def digit_codes(scal, c: int) -> np.ndarray:
    """signed_digits for an (n, 4) uint64 array of canonical scalars at once: uint32 codes, shape (W, n)."""
    s = np.ascontiguousarray(scal, np.uint64).reshape(-1, 4)
    n, W = s.shape[0], windows(c)
    half, full = 1 << (c - 1), 1 << c
    out = np.empty((W, n), np.uint32)
    carry = np.zeros(n, np.int64)
    mask = np.uint64(full - 1)
    for w in range(W):
        bit = w * c
        word, sh = bit // 64, bit % 64
        if word < 4:
            v = s[:, word] >> np.uint64(sh)
            if sh + c > 64 and word + 1 < 4:
                v = v | (s[:, word + 1] << np.uint64(64 - sh))
            v = (v & mask).astype(np.int64)
        else:
            v = np.zeros(n, np.int64)
        v = v + carry
        neg = v > half
        code = np.where(neg, (full - v - 1) | (1 << 31), np.where(v > 0, v - 1, DIGIT_ZERO))
        out[w] = code.astype(np.uint32)
        carry = neg.astype(np.int64)
    return out


def fine_segments(sizes) -> list:
    """Segments of k_fine_sort over one coarse bin of at most FINE_MAX_SEGMENTS * FINE_STAGE entries, as (lo, hi, direct):
    the longest run of buckets from lo whose entries fit the window, or bucket lo alone, scattered straight to HBM, when it
    is larger than the window."""
    off = np.concatenate([[0], np.cumsum(np.asarray(sizes, np.int64))])
    nb, lo, segs = len(sizes), 0, []
    while lo < nb:
        fit = int(np.count_nonzero(off[lo + 1:nb + 1] - off[lo] <= FINE_STAGE))
        hi = lo + (fit if fit > 0 else 1)
        segs.append((lo, hi, fit == 0))
        lo = hi
    return segs


@dataclass
class Reach:
    c: int
    tables: bool
    n_dom: int
    E: int
    NB: int
    levels: int
    ordered: bool
    reduction: str                       # "bit_reduce", "rowcol_stage1" (k_rowcol_stage1 / k_seg_sums) or "rowcol_sums"
    sizes: np.ndarray                    # (n_dom, 2^(c-1)) bucket sizes
    bins: np.ndarray = None              # c > 16: (n_dom, 512) coarse-bin totals
    fine: list = field(default_factory=list)   # c > 16: per domain, per bin "direct", "staged" or "staged+direct"

    @property
    def avg(self) -> int:
        return self.E // self.NB

    def segments(self, dom: int, b: int) -> list:
        low = self.c - 10
        return fine_segments(self.sizes[dom, b << low:(b + 1) << low])

    def heavy(self) -> np.ndarray:
        """(n_dom, 2^(c-1)) mask of the buckets certain to go to k_combine_warp: after the rounds a bucket of m entries
        has ceil(m / 2^levels), and with tasks of at most TASK_LEN_LIMIT entries it has more than COMB_SERIAL_MAX tasks."""
        left = -(-self.sizes // (1 << self.levels))
        return (left + TASK_LEN_LIMIT // 2) // TASK_LEN_LIMIT > COMB_SERIAL_MAX


def reach(scal, c: int, tables: bool = True, batch: int = 1, ba_min_entries: int = BA_MIN_ENTRIES, ba_levels: int = -1) -> Reach:
    """Branches the device MSM of these scalars takes.  scal: (batch * n, 4) canonical scalars, item-major; the options are
    those of zk_ctx_set_opt (ZK_OPT_AFFINE_MIN_ENTRIES, ZK_OPT_AFFINE_LEVELS)."""
    s = np.ascontiguousarray(scal, np.uint64).reshape(batch, -1, 4)
    n, W, nbins = s.shape[1], windows(c), 1 << (c - 1)
    assert tables or batch == 1, "batched MSMs need tables"
    n_dom = batch if tables else W
    sizes = np.zeros((n_dom, nbins), np.int64)
    for k in range(batch):
        codes = digit_codes(s[k], c)
        for w in range(W):
            keys = codes[w][codes[w] != DIGIT_ZERO] & 0x7FFFFFFF
            sizes[k if tables else w] += np.bincount(keys.astype(np.int64), minlength=nbins)
    E, NB = n * W * batch, n_dom * nbins
    levels = 0
    if ba_min_entries >= 0 and E >= ba_min_entries:
        if ba_levels >= 0:
            levels = min(ba_levels, BA_MAX_LEVELS)
        else:
            avg = E // NB
            while avg >= BA_AVG_MIN and levels < BA_MAX_LEVELS:
                levels += 1
                avg >>= 1
    if (n_dom >= ROWCOL_MIN_DOMAINS and c >= ROWCOL_MIN_C) or (tables and c >= TWO_LEVEL_MIN_C):
        reduction = "rowcol_sums" if n_dom >= ROWCOL_MIN_DOMAINS else "rowcol_stage1"
    else:
        reduction = "bit_reduce"
    r = Reach(c, tables, n_dom, E, NB, levels, E // NB < ORDER_AVG_MAX, reduction, sizes)
    if c >= TWO_LEVEL_MIN_C:
        low = c - 10
        r.bins = sizes.reshape(n_dom, COARSE_BINS, 1 << low).sum(axis=2)
        for d in range(n_dom):
            modes = []
            for b in range(COARSE_BINS):
                if r.bins[d, b] > FINE_MAX_SEGMENTS * FINE_STAGE:
                    modes.append("direct")
                elif (sizes[d, b << low:(b + 1) << low] > FINE_STAGE).any():
                    modes.append("staged+direct")
                else:
                    modes.append("staged")
            r.fine.append(modes)
    return r
