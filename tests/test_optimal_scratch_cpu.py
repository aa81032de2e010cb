"""The optimal encoder (levels 18, 19, 39) on scratch as a device warp finds it, without a GPU.

A warp keeps one OptWork across the units of a launch and never cleans its binary tree, opt[] or match list; its map holds
entries of other epochs and its token statistics whatever the last unit left.  The kernel is exact only if the tree needs no
clearing (every node a walk reads was written in the unit, after its position was searched), no stale opt[] field is read
(only opt[0] is reset per window), the statistics are set up at each unit's first inner block, a map slot of another epoch
counts as empty, and a unit of several inner blocks leaves its big slot's table zero, also when it fails on capacity.  These
tests poison all of it and run sequences of units on one persistent scratch, in the one-lane host build and the 32-lane
emulator, against the reference built with -DLIZARD_RESET_MEM."""
import ctypes
import os
import random

import pytest

import lizard_b200 as lz
from tests import refs
from tests.test_optimal_cpu import _long_runs, _periodic

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LEVELS = [18, 19, 39]
BS = lz.BLOCK_SIZE


@pytest.fixture(scope="module")
def ref():
    L = refs.ref_parity()
    if L is None:
        pytest.skip("oracle/_ref not built")
    return L


@pytest.fixture(scope="module")
def shim():
    L = ctypes.CDLL(os.path.join(ROOT, "lizard_b200", "libhostshim.so"))
    L.lzb_opt_scratch_new.restype = ctypes.c_void_p
    L.lzb_opt_scratch_new.argtypes = [ctypes.c_uint]
    for f in ("lzb_opt_scratch_free", "lzb_opt_scratch_clear_map", "lzb_opt_scratch_big_clean"):
        getattr(L, f).argtypes = [ctypes.c_void_p]
    L.lzb_opt_scratch_poison.argtypes = [ctypes.c_void_p, ctypes.c_uint]
    L.lzb_opt_scratch_poison_map.argtypes = [ctypes.c_void_p, ctypes.c_uint, ctypes.c_uint, ctypes.c_uint, ctypes.c_char_p,
                                             ctypes.c_int]
    L.lzb_opt_compress_on.argtypes = [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_int, ctypes.c_char_p, ctypes.c_int, ctypes.c_int,
                                      ctypes.c_uint, ctypes.c_int]
    L.lzb_emu_lane_order.argtypes = [ctypes.c_int]
    return L


def _on(shim, sc, data, level, cap, epoch, emu):
    dst = ctypes.create_string_buffer(max(cap, 1) + 64)
    n = shim.lzb_opt_compress_on(sc, data, len(data), dst, cap, level, epoch, 1 if emu else 0)
    return dst.raw[:n]


def _units(seed, small):
    rnd = random.Random(seed)
    out = []
    for i in range(12 if not small else 8):
        n = rnd.choice([1500, 2600, 3100] if small else [BS, 5000, 70000, 1000, 300000 if i % 4 == 0 else BS - 1])
        kind = i % 4
        if kind == 0:
            u = lz.datagen(n, rnd.choice([10, 50, 90]), seed + i)
        elif kind == 1:
            u = _periodic(rnd.randint(1, 7), n, seed + i, breaks=max(n // 300, 1))
        elif kind == 2:
            u = _long_runs(seed + i, n)
        else:
            u = bytes(n)
        out.append(u)
    return out


@pytest.mark.parametrize("emu", [False, True])
def test_unit_sequence_on_poisoned_scratch(ref, shim, emu):
    """One warp's scratch over many units and all three levels: the tree, opt[], the match list and the statistics poisoned
    before the first unit and again between units, the map full of other epochs' entries (stale entries of the next unit's
    own buckets among them), capacities that fail among the ones that fit."""
    sc = shim.lzb_opt_scratch_new(11)
    try:
        epoch = 0
        rnd = random.Random(3)
        for i, u in enumerate(_units(7, emu)):
            level = LEVELS[i % 3]
            if emu:
                shim.lzb_emu_lane_order(i % 3)
            bound = ref.Lizard_compressBound(len(u))
            want_full = refs.ref_compress(ref, u, level, bound)
            cap = bound if i % 3 else max(len(want_full) - 1, 1)
            want = refs.ref_compress(ref, u, level, cap)
            if i % 2:
                shim.lzb_opt_scratch_poison(sc, 100 + i)
            if len(u) <= BS:
                epoch += 1
                if i % 4 == 1:                                   # a map full of other epochs' entries
                    shim.lzb_opt_scratch_poison_map(sc, epoch, 18 if level == 18 else 23, i, u, len(u))
            got = _on(shim, sc, u, level, cap, max(epoch, 1), emu)
            assert got == want, (i, level, len(u), cap, len(got), len(want))
            assert shim.lzb_opt_scratch_big_clean(sc) == 1, (i, len(u))
            if rnd.random() < 0.2:
                shim.lzb_opt_scratch_clear_map(sc)
                epoch = 0
    finally:
        if emu:
            shim.lzb_emu_lane_order(0)
        shim.lzb_opt_scratch_free(sc)


def test_big_units_leave_their_slot_zero(ref, shim):
    """Units of several inner blocks on one persistent big slot, some failing on capacity: each one finds the table zero and
    leaves it zero."""
    sc = shim.lzb_opt_scratch_new(5)
    try:
        for i, (n, level) in enumerate([(300000, 19), (BS + 1, 18), (1 << 20, 39), ((4 << 20) + 999, 18), (200000, 39)]):
            u = lz.datagen(n, 40 + 10 * i, i)
            bound = ref.Lizard_compressBound(n)
            cap = bound if i % 2 == 0 else len(refs.ref_compress(ref, u, level, bound)) // 2
            shim.lzb_opt_scratch_poison(sc, i)
            assert _on(shim, sc, u, level, cap, 1, False) == refs.ref_compress(ref, u, level, cap), (i, n, level, cap)
            assert shim.lzb_opt_scratch_big_clean(sc) == 1, (i, n)
    finally:
        shim.lzb_opt_scratch_free(sc)
