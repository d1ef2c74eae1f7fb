"""CPU check of the host forms' staging (Stage, zero_chain_b200/csrc/internal.h), compiled with g++ against a CUDA stub that
works on host memory and records every copy (tests/host_emul/emul_stage.cpp): the carved regions, one copy per non-empty
array and direction, the NULL and zero-count rules, an output whose row count is set after the run, and a buffer that
is reserved once.  The real copies are covered by every host form's GPU test."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
IN, OUT, INOUT = 1, 2, 3
H2D, D2H = 1, 2


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emul_stage") / "libemul_stage.so")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-I", os.path.join(HERE, "host_emul", "cuda_stub"),
                           "-I", os.path.join(ROOT, "zero_chain_b200", "csrc"), "-o", so, os.path.join(HERE, "host_emul", "emul_stage.cpp")])
    lib = C.CDLL(so)
    lib.emu_copies.restype = C.c_size_t
    lib.emu_mallocs.restype = C.c_size_t
    lib.emu_io_base.restype = C.c_uint64
    lib.emu_io_cap.restype = C.c_size_t
    return lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


class Item:
    """one registered array: its host copy (None: a NULL host pointer)"""

    def __init__(self, rng, direction, elem, count, null=False, width=0):
        self.dir, self.elem, self.count, self.width = direction, elem, count, width     # width > 0: rows of width elements
        dt = {1: np.uint8, 4: np.uint32, 8: np.uint64}[elem]
        self.host = None if null else rng.integers(0, 1 << (8 * elem - 1), max(count, 1)).astype(dt)
        self.before = None if null else self.host.copy()

    def ptr(self):
        return self.host.ctypes.data if self.host is not None else None

    def nbytes(self, count=None):
        return self.elem * (self.count if count is None else count)


def copies(emu):
    n = 1024
    kind, dst, src, nb = np.zeros(n, np.int32), np.zeros(n, np.uint64), np.zeros(n, np.uint64), np.zeros(n, np.uint64)
    k = emu.emu_copies(_p(kind), _p(dst), _p(src), _p(nb), C.c_size_t(n))
    assert k <= n
    return [(int(kind[i]), int(dst[i]), int(src[i]), int(nb[i])) for i in range(k)]


def run(emu, items, rows_after=None, run_writes=None):
    """up, the 'run' (run_writes(item, device bytes) per output), down; returns the device pointers and both copy lists"""
    n = len(items)
    rows = np.array([max((it.count // it.width for it in items if it.width), default=0)], np.uint64)
    dev = np.zeros(n, np.uint64)
    host = (C.c_void_p * max(n, 1))(*[it.ptr() for it in items])
    arr = lambda xs, dt: np.array(xs or [0], dt)
    copies(emu)
    assert emu.emu_up(C.c_size_t(n), _p(arr([it.dir for it in items], np.int32)), _p(arr([it.elem for it in items], np.uint64)),
                      _p(arr([it.count for it in items], np.uint64)), host, _p(arr([it.width for it in items], np.uint64)),
                      _p(rows), _p(dev)) == 0
    ups = copies(emu)
    for i, it in enumerate(items):
        if dev[i] and it.dir != IN and run_writes:
            buf = (C.c_uint8 * it.nbytes()).from_address(int(dev[i]))
            run_writes(i, it, buf)
    if rows_after is not None:
        rows[0] = rows_after
    assert emu.emu_down() == 0
    return [int(d) for d in dev], ups, copies(emu), int(rows[0])


def mixed(rng):
    items = []
    for _ in range(int(rng.integers(1, 14))):
        d = int(rng.choice([IN, OUT, INOUT]))
        elem = int(rng.choice([1, 4, 8])) if d == IN else int(rng.choice([1, 4]))
        count = int(rng.choice([0, 1, 3, 64, 1000, 5000]))
        items.append(Item(rng, d, elem, count, null=rng.random() < 0.15))
    return items


def pattern(i, it, buf):
    """the run's output: byte j of output i is (i + 7 j) mod 251"""
    buf[:] = bytes((i + 7 * j) % 251 for j in range(len(buf)))


@pytest.mark.parametrize("seed", range(16))
def test_regions_and_copies(emu, seed):
    rng = np.random.default_rng(7100 + seed)
    items = mixed(rng)
    dev, ups, downs, _ = run(emu, items, run_writes=pattern)
    base, cap = emu.emu_io_base(), emu.emu_io_cap()
    spans = []
    for it, d in zip(items, dev):
        if it.host is None:
            assert d == 0                                       # NULL host: NULL device, no space
            continue
        assert d != 0 and (d - base) % 256 == 0 and base <= d and d + it.nbytes() <= base + cap
        if it.count:
            spans.append((d, d + it.nbytes()))
    spans.sort()
    assert all(a[1] <= b[0] for a, b in zip(spans, spans[1:]))  # no two regions overlap
    # one copy up per non-empty in / in-out array, in registration order, byte for byte; nothing else
    want_up = [(H2D, d, it.ptr(), it.nbytes()) for it, d in zip(items, dev) if it.host is not None and it.count and it.dir != OUT]
    assert ups == want_up
    # one copy down per non-empty out / in-out array; the host arrays hold the run's bytes, the inputs are untouched
    want_down = [(D2H, it.ptr(), d, it.nbytes()) for it, d in zip(items, dev) if it.host is not None and it.count and it.dir != IN]
    assert downs == want_down
    for i, it in enumerate(items):
        if it.host is None or not it.count:
            continue
        got = it.host.view(np.uint8)[:it.nbytes()].tobytes()
        if it.dir == IN:
            assert got == it.before.view(np.uint8)[:it.nbytes()].tobytes()
        else:
            assert got == bytes((i + 7 * j) % 251 for j in range(it.nbytes()))


def test_in_out_arrays_go_up_before_the_run(emu):
    rng = np.random.default_rng(7200)
    items = [Item(rng, INOUT, 1, 300), Item(rng, OUT, 4, 50), Item(rng, INOUT, 4, 20)]
    seen = {}
    dev, ups, downs, _ = run(emu, items, run_writes=lambda i, it, buf: seen.__setitem__(i, bytes(buf)))
    # an in-out array's device copy holds the caller's bytes when the run starts; the run left them, so they come back
    assert seen[0] == items[0].before.tobytes() and seen[2] == items[2].before.tobytes()
    assert items[0].host.tobytes() == items[0].before.tobytes()
    assert [c[0] for c in ups] == [H2D, H2D] and [c[0] for c in downs] == [D2H, D2H, D2H]


def test_zero_count_gets_a_pointer_and_no_copy(emu):
    rng = np.random.default_rng(7300)
    for items in ([Item(rng, IN, 1, 0), Item(rng, OUT, 4, 0), Item(rng, INOUT, 1, 0)],        # nothing to stage at all
                  [Item(rng, IN, 8, 0), Item(rng, IN, 1, 33), Item(rng, OUT, 1, 0, null=True), Item(rng, OUT, 4, 0)]):
        dev, ups, downs, _ = run(emu, items, run_writes=pattern)
        for it, d in zip(items, dev):
            assert (d == 0) == (it.host is None)
        assert all(c[3] for c in ups + downs)
        assert len(ups) == sum(1 for it in items if it.count and it.host is not None and it.dir != OUT)
        assert len(downs) == sum(1 for it in items if it.count and it.host is not None and it.dir != IN)


@pytest.mark.parametrize("rows_after", [0, 1, 17, 40])
def test_late_count_output_comes_down_for_the_count_set_after_the_run(emu, rows_after):
    """a table of 40 rows at most: ids (one uint32 per row), keys (32 bytes), ciphertexts (64 bytes), flags (one byte)"""
    rng = np.random.default_rng(7400 + rows_after)
    table = [Item(rng, OUT, 4, 40, width=1), Item(rng, OUT, 1, 32 * 40, width=32), Item(rng, OUT, 1, 64 * 40, width=64),
             Item(rng, OUT, 1, 40, width=1), Item(rng, OUT, 1, 32 * 40)]
    dev, ups, downs, rows = run(emu, table, rows_after=rows_after, run_writes=pattern)
    assert rows == rows_after and ups == []
    want = [(D2H, it.ptr(), d, it.elem * it.width * rows_after) for it, d in zip(table[:4], dev) if rows_after]
    assert downs == want + [(D2H, table[4].ptr(), dev[4], 32 * 40)]    # one without a row count comes down whole
    for i, it in enumerate(table[:4]):
        n = it.elem * it.width * rows_after
        assert it.host.view(np.uint8)[:n].tobytes() == bytes((i + 7 * j) % 251 for j in range(n))
        assert it.host.view(np.uint8)[n:].tobytes() == it.before.view(np.uint8)[n:].tobytes()    # the rest keeps the caller's bytes


def test_a_smaller_call_reuses_the_buffer(emu):
    rng = np.random.default_rng(7500)
    run(emu, [Item(rng, IN, 1, 200_000), Item(rng, OUT, 4, 10_000)])
    base, cap, mallocs = emu.emu_io_base(), emu.emu_io_cap(), emu.emu_mallocs()
    for _ in range(3):
        dev, _, _, _ = run(emu, [Item(rng, IN, 4, 1000), Item(rng, INOUT, 1, 5000), Item(rng, OUT, 1, 3)])
        assert emu.emu_mallocs() == mallocs and emu.emu_io_base() == base and emu.emu_io_cap() == cap
        assert dev[0] == base
    run(emu, [Item(rng, IN, 1, 2 * cap)])                       # a larger one grows it once
    assert emu.emu_mallocs() == mallocs + 1 and emu.emu_io_cap() >= 2 * cap
