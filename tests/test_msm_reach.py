"""The MSM reach model (tests/msm_reach.py) against the CUDA sources it copies: every constant and branch condition the model
uses is read out of the kernels, and the host digit recoding must recombine to the scalar exactly as k_msm_digits does.
CPU only."""
import os
import re

import numpy as np
import pytest

from oracle import pyref as pr
from tests import msm_reach as mr

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "zero_chain_b200", "csrc")


def _src(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def _const(text, name, env=None):
    """value of the C initializer `name = <expr>` (integer suffixes u / l dropped, earlier constants from env)"""
    m = re.search(r"\b%s\s*=\s*([^,;]+)[,;]" % name, text)
    assert m, name
    expr = re.sub(r"\b(0x[0-9a-fA-F]+|\d+)[uUlL]+\b", r"\1", m.group(1).strip())
    return eval(expr, {"__builtins__": {}}, dict(env or {}))


@pytest.mark.parametrize("header,name,copy", [
    ("msm.cuh", "FINE_STAGE", mr.FINE_STAGE),
    ("msm.cuh", "FINE_MAX_SEGMENTS", mr.FINE_MAX_SEGMENTS),
    ("msm.cuh", "COARSE_BINS", mr.COARSE_BINS),
    ("msm.cuh", "COMB_SERIAL_MAX", mr.COMB_SERIAL_MAX),
    ("msm.cuh", "DIGIT_ZERO", mr.DIGIT_ZERO),
    ("msm_accum.cuh", "TASK_LEN_MAX", mr.TASK_LEN_MAX),
    ("msm_batchaff.cuh", "BA_MAX_LEVELS", mr.BA_MAX_LEVELS),
    ("internal.h", "ba_min_entries", mr.BA_MIN_ENTRIES),
])
def test_constant_matches_source(header, name, copy):
    assert _const(_src(header), name) == copy


def test_coarse_chunk_matches_source():
    text = _src("msm.cuh")
    env = {k: _const(text, k) for k in ("COARSE_THREADS", "COARSE_PER_THREAD")}
    assert _const(text, "COARSE_CHUNK", env) == mr.COARSE_CHUNK


@pytest.mark.parametrize("header,fragment", [
    # coarse bins: the high 9 of the c - 1 key bits, windows above 16 bits
    ("msm_driver.cuh", "const bool two_level = c > 16;"),
    ("msm_driver.cuh", "const int low = two_level ? (c - 1) - 9 : 0, sort_bins = two_level ? 512 : nbins;"),
    # k_fine_sort: a whole bin straight to HBM above FINE_MAX_SEGMENTS windows; else segments that fit the window, or one
    # bucket alone when it does not
    ("msm.cuh", "if (total > (uint32_t)FINE_MAX_SEGMENTS * FINE_STAGE) {"),
    ("msm.cuh", "off[threadIdx.x + 1] - base <= (uint32_t)FINE_STAGE);"),
    ("msm.cuh", "const bool direct = fit == 0;"),
    # batched-affine rounds: threshold, forced count, heuristic
    ("msm_driver.cuh", "if (ctx->opts.ba_min_entries >= 0 && (long)E >= ctx->opts.ba_min_entries) {"),
    ("msm_driver.cuh", "levels = (int)(ctx->opts.ba_levels < BA_MAX_LEVELS ? ctx->opts.ba_levels : BA_MAX_LEVELS);"),
    ("msm_driver.cuh", "for (size_t avg = E / NB; avg >= 12 && levels < BA_MAX_LEVELS; avg >>= 1) levels++;"),
    ("msm_batchaff.cuh", "sizes_out[b] = (off_in[b + 1] - off_in[b] + 1) >> 1;"),
    # task order, reduction scheme
    ("msm_driver.cuh", "bool want = E / NB < 256;"),
    ("msm_driver.cuh", "if ((n_dom >= 8 && c >= 7) || (tables && c > 16)) {"),
    ("msm_driver.cuh", "if (n_dom >= 8) {"),
    # tasks per bucket and the heavy-bucket cut
    ("msm.cuh", "if (t > (uint32_t)TASK_LEN_MAX + 8) t = TASK_LEN_MAX + 8;"),
    ("msm.cuh", "uint32_t t = (v + task_len / 2) / task_len;"),
    ("msm.cuh", "if (t1 - t0 > COMB_SERIAL_MAX) {"),
])
def test_branch_condition_matches_source(header, fragment):
    assert fragment in _src(header)


def test_model_thresholds_match_the_conditions():
    assert (mr.BA_AVG_MIN, mr.ORDER_AVG_MAX, mr.ROWCOL_MIN_DOMAINS, mr.ROWCOL_MIN_C, mr.TWO_LEVEL_MIN_C) == (12, 256, 8, 7, 17)
    assert mr.TASK_LEN_LIMIT == mr.TASK_LEN_MAX + 8


def _edge_scalars(c):
    W = mr.windows(c)
    vals = {0, 1, 2, pr.R - 1, pr.R - 2, 1 << (c - 1), (1 << (c - 1)) + 1, (1 << c) - 1, (1 << 254) - 1}
    for w in range(W):
        for d in (-1, 0, 1):
            vals.add((1 << (c * w)) + d)
    # carries through every window: every window all ones, or every window just above half
    vals.add(sum(((1 << c) - 1) << (c * w) for w in range(W)))
    vals.add(sum(((1 << (c - 1)) + 1) << (c * w) for w in range(W)))
    vals.add(sum((1 << (c - 1)) << (c * w) for w in range(W)))
    return sorted(v % pr.R for v in vals if v >= 0)


@pytest.mark.parametrize("c", range(2, 21))
def test_signed_digits_recombine(c):
    half = 1 << (c - 1)
    rng = np.random.default_rng(c)
    vals = _edge_scalars(c) + [int.from_bytes(rng.bytes(32), "little") % pr.R for _ in range(32)]
    for s in vals:
        codes = mr.signed_digits(s, c)
        assert len(codes) == mr.windows(c)
        assert mr.recombine(codes, c) == s, hex(s)
        for k in codes:
            assert k == mr.DIGIT_ZERO or (k & 0x7FFFFFFF) < half          # bucket key in [0, 2^(c-1))
    # the vectorised recoding the model uses for whole MSMs is the same
    limbs = np.array([[(s >> (64 * j)) & (2**64 - 1) for j in range(4)] for s in vals], np.uint64)
    got = mr.digit_codes(limbs, c)
    want = np.array([mr.signed_digits(s, c) for s in vals], np.uint32).T
    assert np.array_equal(got, want)


def test_carry_into_a_full_window_is_a_zero_digit():
    # window all ones plus the carry from below: digit 0 with a carry, coded DIGIT_ZERO (the code wraps)
    c = 5
    codes = mr.signed_digits((1 << 10) - 1, c)
    assert codes[:3] == [0x80000000, mr.DIGIT_ZERO, 0]      # -1, 0, +1: 2^10 - 1 = -1 + 0 * 32 + 1 * 1024


def test_fine_segments():
    S = mr.FINE_STAGE
    assert mr.fine_segments([S]) == [(0, 1, False)]
    assert mr.fine_segments([S, 1]) == [(0, 1, False), (1, 2, False)]
    assert mr.fine_segments([5, S + 1, 0, 7]) == [(0, 1, False), (1, 2, True), (2, 4, False)]
    assert mr.fine_segments([S + 1, S + 2]) == [(0, 1, True), (1, 2, True)]
    assert mr.fine_segments([0, 0]) == [(0, 2, False)]


def test_reach_of_the_production_shape():
    """2^20 terms, 20-bit windows, library defaults: two rounds, ordered tasks, row / column reduction with stage 1"""
    n = 1 << 20
    scal = np.zeros((n, 4), np.uint64)
    scal[:, 0] = np.arange(n, dtype=np.uint64) * 2654435761 % (1 << 32)
    r = mr.reach(scal, 20)
    assert (r.E, r.NB, r.avg) == (13 * n, 1 << 19, 26)
    assert r.levels == 2 and r.ordered and r.reduction == "rowcol_stage1"
    # batched domains take k_rowcol_sums from 8 on
    small = scal[:64 * 9]
    for batch, c, want in ((7, 9, "bit_reduce"), (7, 17, "rowcol_stage1"), (8, 9, "rowcol_sums"), (9, 20, "rowcol_sums")):
        assert mr.reach(small[:64 * batch], c, batch=batch).reduction == want
