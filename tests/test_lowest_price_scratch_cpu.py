"""The lowestPrice encoder (levels 23-25, 43-45) on scratch as a device warp finds it, without a GPU.

A warp keeps one LpWork across the units of a launch and never cleans it between units: the sequence list, chain, streams
and Huffman scratch hold what came before, the map holds entries of other epochs (and, in the workspace the kernel shares
with the other encoder, anything), and a big slot's chain is never cleared.  The kernel is exact only if a map slot of
another epoch counts as empty, the chain needs no clearing, and every unit of several inner blocks leaves its big slot's
table zero, also when it fails on capacity.  These tests run sequences of units on one persistent, poisoned scratch in the
one-lane host build and the 32-lane emulator (all three lane orders), with epochs that follow the kernel's rule up to
kLpEpochMax and past it, and compare every unit with the reference built with -DLIZARD_RESET_MEM.  The map's probe
counters show that the `collide` family builds the long and wrapping probe runs it is made for."""
import ctypes
import os
import random

import pytest

import lizard_b200 as lz
from tests import corpus, refs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LEVELS = corpus.LP_ENCODE_LEVELS
BS = corpus.BS
EPOCH_MAX = (1 << 23) - 1                     # kLpEpochMax, csrc/encode_lp.cuh
LONGEST, PROBES, WRAPS = range(3)             # lzb_lp_probe_stats


def _hash_log(level):
    return 18 if level in (23, 43) else 23


def _mls(level):
    return 4 if level in (25, 45) else 5


@pytest.fixture(scope="module")
def ref():
    L = refs.ref_parity()
    if L is None:
        pytest.skip("oracle/_ref not built")
    return L


@pytest.fixture(scope="module")
def shim():
    L = ctypes.CDLL(os.path.join(ROOT, "lizard_b200", "libhostshim.so"))
    L.lzb_lp_scratch_new.restype = ctypes.c_void_p
    L.lzb_lp_scratch_new.argtypes = [ctypes.c_uint]
    L.lzb_lp_scratch_free.argtypes = [ctypes.c_void_p]
    L.lzb_lp_scratch_poison_map.argtypes = [ctypes.c_void_p, ctypes.c_uint, ctypes.c_uint, ctypes.c_uint, ctypes.c_char_p,
                                            ctypes.c_int, ctypes.c_uint]
    L.lzb_lp_scratch_clear_map.argtypes = [ctypes.c_void_p]
    L.lzb_lp_scratch_big_clean.argtypes = [ctypes.c_void_p]
    L.lzb_lp_compress_on.argtypes = [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_int, ctypes.c_char_p, ctypes.c_int, ctypes.c_int,
                                     ctypes.c_uint, ctypes.c_int]
    L.lzb_emu_lane_order.argtypes = [ctypes.c_int]
    L.lzb_lp_probe_stats.argtypes = [ctypes.POINTER(ctypes.c_ulonglong), ctypes.c_int]
    return L


class Warp:
    """One warp's persistent scratch and epoch, stepped as lizard_encode_lowest_price_kernel steps it: before a unit of one
    inner block, an epoch at kLpEpochMax clears the map and starts over at 1, any other epoch goes up by one."""

    def __init__(self, shim, seed, emu=False):
        self.shim, self.emu, self.epoch, self.poisoned = shim, emu, EPOCH_MAX, None
        self.sc = shim.lzb_lp_scratch_new(seed)

    def close(self):
        self.shim.lzb_lp_scratch_free(self.sc)

    def jump(self, epoch, level, seed, data):
        """Run the next unit, `data`, at `epoch` on a map full of entries of other epochs (0, epoch - 1, epoch + 1,
        kLpEpochMax), among them stale entries of data's own buckets that would change its parse if they were taken for
        current ones.  The unit after it runs at epoch + 2, past the poisoned epoch + 1 (entries of a later epoch than the
        current one cannot be left behind in the kernel: the map is cleared before a warp's first unit and at the wrap)."""
        self.epoch, self.poisoned = epoch - 1, epoch
        self.shim.lzb_lp_scratch_poison_map(self.sc, epoch, _hash_log(level), seed, data, len(data), _mls(level))

    def compress(self, data, level, cap):
        epoch = 0
        if len(data) <= BS:
            if self.epoch == EPOCH_MAX:
                self.shim.lzb_lp_scratch_clear_map(self.sc)
                self.epoch = 0
            self.epoch += 1
            epoch = self.epoch
        dst = ctypes.create_string_buffer(max(cap, 1) + 64)
        n = self.shim.lzb_lp_compress_on(self.sc, data, len(data), dst, cap, level, max(epoch, 1), int(self.emu))
        if epoch and epoch == self.poisoned:
            self.poisoned = None
            if epoch < EPOCH_MAX:
                self.epoch += 1
        return dst.raw[:n]


def _stats(shim):
    out = (ctypes.c_ulonglong * 3)()
    shim.lzb_lp_probe_stats(out, 1)
    return list(out)


def _single_block_units(level):
    """Units of at most one inner block: the shared corpus's, `collide`, and datagen units of assorted sizes."""
    units = [u for us in corpus.lp_corpus().values() for u in us if len(u) <= BS]
    for k, n in enumerate((BS, 70000, 4096, 21, 1000, BS - 1, 0, 300)):
        units.append(lz.datagen(n, (20 * k + level) % 100, level + k))
    return units


# epochs of the sequence, as jumps taken before the unit with that index: epoch 1 on a poisoned map, poisoned maps far up,
# and kLpEpochMax, after which the map is cleared and the units run at 1, 2, ... on what the earlier ones left, until a last
# poisoned map
def _epoch_plan(count):
    return {0: 1, count // 6: 500, count // 3: 1000, count // 2: EPOCH_MAX, 5 * count // 6: 3000}


@pytest.mark.parametrize("lanes", ["host", "emu-forward", "emu-reverse", "emu-shuffled"])
@pytest.mark.parametrize("level", LEVELS)
def test_unit_sequence_on_poisoned_scratch(ref, shim, level, lanes):
    units = _single_block_units(level)
    emu = lanes != "host"
    if emu:
        shim.lzb_emu_lane_order(["emu-forward", "emu-reverse", "emu-shuffled"].index(lanes))
        # 32 coroutines are slow: small units, one datagen unit and the first cluster of `collide` (its keys end at 32 KiB)
        rnd = random.Random(level)
        units = [u for u in units if len(u) < 4096] + [lz.datagen(30000, 50, level),
                                                       corpus.collide_units()[4 * (_mls(level) == 4)][:40000]]
        rnd.shuffle(units)
    rnd = random.Random(100 + level)
    plan = _epoch_plan(len(units))
    w = Warp(shim, seed=level, emu=emu)
    seen_epochs = []
    try:
        for i, u in enumerate(units):
            if i in plan:
                w.jump(plan[i], level, i, u)
            bound = ref.Lizard_compressBound(len(u))
            cap = rnd.choice([bound, bound, max(len(u) - 1, 1), len(u) // 2 + 1])
            want = refs.ref_compress(ref, u, level, cap)
            got = w.compress(u, level, cap)
            seen_epochs.append(w.epoch)
            assert got == want, (lanes, level, i, len(u), cap, w.epoch, len(got), len(want))
    finally:
        w.close()
        shim.lzb_emu_lane_order(0)
    assert EPOCH_MAX in seen_epochs and 1 in seen_epochs[seen_epochs.index(EPOCH_MAX):], seen_epochs   # past the wrap


@pytest.mark.parametrize("level", LEVELS)
def test_big_units_leave_their_slot_zero(ref, shim, level):
    """Units of several inner blocks one after another on one big slot whose chain is garbage: every capacity, failing ones
    included, gives the reference's bytes and leaves the slot's table zero for the next unit.  Units of one inner block in
    between run on the same LpWork."""
    sizes = [BS + 1, BS + 20, BS + 21, 1 << 20, (4 << 20) + 12345]
    w = Warp(shim, seed=7 * level)
    try:
        for k, n in enumerate(sizes):
            u = lz.datagen(n, 30 + 10 * k, level + k)
            full = refs.ref_compress(ref, u, level)
            for cap in (ref.Lizard_compressBound(n), len(full), len(full) - 1, n // 50):
                want = full if cap >= len(full) else refs.ref_compress(ref, u, level, cap)
                got = w.compress(u, level, cap)
                assert got == want, (level, n, cap, len(got), len(want))
                assert shim.lzb_lp_scratch_big_clean(w.sc), ("table not left zero", level, n, cap)
            small = lz.datagen(5000 + k, 50, k)
            assert w.compress(small, level, 9000) == refs.ref_compress(ref, small, level, 9000)
    finally:
        w.close()


@pytest.mark.parametrize("level", LEVELS)
def test_collide_builds_long_and_wrapping_probe_runs(ref, shim, level):
    """At hashLog 23 the `collide` clusters probe past 1000 slots and wrap past the map's last slot; at hashLog 18 (23, 43)
    a bucket is its own home slot and nothing probes.  Every unit still matches the reference."""
    w = Warp(shim, seed=level)
    _stats(shim)
    try:
        for u in corpus.collide_units():
            assert w.compress(u, level, len(u) + 1000) == refs.ref_compress(ref, u, level, len(u) + 1000), level
    finally:
        w.close()
    s = _stats(shim)
    if _hash_log(level) == 18:
        assert s == [0, 0, 0], s
    else:
        assert s[LONGEST] >= 1000 and s[WRAPS] >= 1, s
