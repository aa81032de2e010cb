"""The binary-tree optimal encoder with LZ4 codewords (levels 18, 19 and the Huffman twin 39) without a GPU: the one-lane host
build and the 32-lane warp emulator (all three lane orders) of encode_opt.cuh must write the bytes of the reference built with
-DLIZARD_RESET_MEM.  Also: the reference behaviours the parser restates are reached (parser counters), 19 and 39 parse the
same input differently, the levels that stay unimplemented are still refused, and the new kernel's resources are pinned.
The emulator runs every ballot as 32 context switches, so it only gets units of a few KiB here."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

import lizard_b200 as lz
from tests import refs
from tests.corpus import corpus
from tests.test_encode_resources_cpu import LIB, _cuobjdump
from tests.test_gpu_encode import _cases

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LEVELS = [18, 19, 39]
REFUSED = [12, 26, 27, 28, 29, 32, 33, 46, 47, 48, 49]
BS = lz.BLOCK_SIZE
# csrc/encode_opt.cuh, lzb_opt_stats
(SEARCHED, NEAR_END, SKIPPED, LONG_MATCH, RESCUE, RESCUE_TAKEN, WALK_LONG, WALK_END, WALK_LEAF, WALK_TRIES, GAP_FILL, CAPPED,
 LIT_TIE, MATCH_TIE, RESCALE, SEQUENCES) = range(16)


@pytest.fixture(scope="module")
def ref():
    L = refs.ref_parity()
    if L is None:
        pytest.skip("oracle/_ref not built")
    return L


@pytest.fixture(scope="module")
def shim():
    L = ctypes.CDLL(os.path.join(ROOT, "lizard_b200", "libhostshim.so"))
    for f in ("lzb_host_compress", "lzb_emu_compress"):
        getattr(L, f).argtypes = [ctypes.c_char_p, ctypes.c_int, ctypes.c_char_p, ctypes.c_int, ctypes.c_int]
    L.lzb_emu_lane_order.argtypes = [ctypes.c_int]
    L.lzb_opt_stats.argtypes = [ctypes.POINTER(ctypes.c_ulonglong), ctypes.c_int]
    return L


def _run(fn, data, level, cap):
    dst = ctypes.create_string_buffer(max(cap, 1) + 64)
    n = fn(data, len(data), dst, cap, level)
    return dst.raw[:n]


def _stats(shim):
    out = (ctypes.c_ulonglong * 16)()
    shim.lzb_opt_stats(out, 1)
    return list(out)


def _same(shim, ref, data, level, cap=None, emu=False):
    cap = ref.Lizard_compressBound(len(data)) if cap is None else cap
    want = refs.ref_compress(ref, data, level, cap)
    got = _run(shim.lzb_host_compress, data, level, cap)
    assert got == want, ("host", level, len(data), cap, len(got), len(want))
    if emu:
        for order in (0, 1, 2):
            shim.lzb_emu_lane_order(order)
            got = _run(shim.lzb_emu_compress, data, level, cap)
            assert got == want, ("emu", order, level, len(data), cap, len(got), len(want))
        shim.lzb_emu_lane_order(0)
    return want


def _periodic(period, n, seed, breaks=200):
    """A `period`-byte pattern repeated, broken by random bytes: nodes closer than 8 bytes that the tree walk must rescue."""
    rng = np.random.default_rng(seed)
    a = bytearray((bytes(rng.integers(0, 256, period, dtype=np.uint8)) * (n // period + 1))[:n])
    for i in rng.integers(0, n, breaks):
        a[int(i)] = int(rng.integers(0, 256))
    return bytes(a)


def _long_runs(seed, n=BS):
    """Random bytes with copies of 1500 and 6000 bytes from earlier on: matches beyond sufficientLength and LIZARD_OPT_NUM."""
    rng = np.random.default_rng(seed)
    out = bytearray(rng.integers(0, 256, 9000, dtype=np.uint8).tobytes())
    while len(out) < n:
        k = [1500, 6000, 300][len(out) % 3]
        at = len(out) - int(rng.integers(8, min(len(out), 60000)))
        out += out[at:at + k] + rng.integers(0, 256, int(rng.integers(1, 40)), dtype=np.uint8).tobytes()
    return bytes(out[:n])


def _staggered(seed):
    """Random bytes R, then R with a byte changed every 900 bytes, R with the changes 450 bytes later, and R itself: in the
    last copy every position has a match of up to 900 bytes that reaches past the previous one's end, so one DP window runs
    until LIZARD_OPT_NUM caps the lengths."""
    rng = np.random.default_rng(seed)
    r = rng.integers(0, 256, 20000, dtype=np.uint8)
    a, b = r.copy(), r.copy()
    a[::900] ^= 0x55
    b[450::900] ^= 0x55
    return bytes(np.concatenate([r[:3000], a, b, r]))


@pytest.mark.parametrize("level", LEVELS)
def test_corpus_and_datagen(ref, shim, level):
    units = [u for fam in corpus().values() for u in fam]
    for p in (0, 10, 25, 50, 75, 90, 100):
        units.append(lz.datagen(BS, p, p + level))
    for u in units:
        _same(shim, ref, u, level)
    for i, p in enumerate((0, 50, 100)):                        # the emulator: small units, all three lane orders
        _same(shim, ref, lz.datagen(2500 + 700 * i, p, level), level, emu=True)


@pytest.mark.parametrize("level", LEVELS)
def test_edge_sizes_and_capacities(ref, shim, level):
    for c in _cases():
        want = _same(shim, ref, c, level)
        bound = ref.Lizard_compressBound(len(c))
        for cap in {bound, len(want), max(len(want) - 1, 1), max(len(want) // 2, 1)}:      # cap 0: the reference writes past it
            _same(shim, ref, c, level, cap, emu=len(c) <= 1000 and cap == len(want) - 1)


@pytest.mark.parametrize("level", LEVELS)
def test_units_of_several_inner_blocks(ref, shim, level):
    """Several inner blocks: one window across them, the big-slot table, and (at 39) the rescaled token statistics."""
    _same(shim, ref, lz.datagen(300000, 50, level), level)
    _same(shim, ref, lz.datagen(1 << 20, 70, level), level)


@pytest.mark.parametrize("level", [18, 39])
def test_unit_beyond_4_mib(ref, shim, level):
    _same(shim, ref, lz.datagen((4 << 20) + 70000, 55, level), level)


@pytest.mark.parametrize("level", LEVELS)
def test_long_runs_and_short_periods(ref, shim, level):
    units = [_long_runs(level), bytes(BS), b"\x07" * 9000 + lz.datagen(9000, 50, 1)]
    units += [_periodic(p, 40000, p) for p in range(1, 8)]
    for u in units:
        _same(shim, ref, u, level)
    for p in (1, 3, 7):
        _same(shim, ref, _periodic(p, 1500, p + 10, breaks=20), level, emu=True)
    _same(shim, ref, _long_runs(level + 1, 3000), level, emu=True)


def test_reference_behaviours_are_reached(ref, shim):
    """Every branch the DESIGN notes (3.1b) list for the parser runs on this input set, and the bytes still match."""
    _stats(shim)
    units = [_long_runs(1), _long_runs(2, 300000), bytes(20000), lz.datagen(BS, 50, 3), lz.datagen(300000, 20, 4), _staggered(5)]
    units += [_periodic(p, 30000, p) for p in range(1, 8)]
    for level in LEVELS:
        for u in units:
            _same(shim, ref, u, level)
    s = _stats(shim)
    for k, name in enumerate(("searched", "near_end", "skipped", "long_match", "rescue", "rescue_taken", "walk_long", "walk_end",
                              "walk_leaf", "walk_tries", "gap_fill", "capped", "lit_tie", "match_tie", "rescale", "sequences")):
        assert s[k] > 0, (name, s)


def test_huffman_flag_changes_the_parse(ref, shim):
    """At 39 the token price follows the token statistics, so the parse itself differs from 19 (the parser's own counts are
    taken before any stream is built), and both outputs still match the reference byte for byte."""
    for data in (lz.datagen(300000, 50, 5), _long_runs(6)):
        _stats(shim)
        _same(shim, ref, data, 19)
        plain = _stats(shim)
        _same(shim, ref, data, 39)
        huf = _stats(shim)
        assert plain[SEQUENCES] > 0 and plain[RESCALE] == 0 and huf[RESCALE] + 1 >= len(data) // BS
        assert plain[:RESCALE] != huf[:RESCALE], (plain, huf)


@pytest.mark.parametrize("level", REFUSED)
def test_other_levels_stay_unsupported(shim, level):
    data = lz.datagen(5000, 50, 1)
    assert _run(shim.lzb_host_compress, data, level, 10000) == b""
    assert _run(shim.lzb_emu_compress, data, level, 10000) == b""


def test_kernel_resources():
    """lizard_encode_optimal_kernel at 128 threads under __maxnreg__(96): exactly 96 registers (5 CTAs per SM, 20 KiB of static
    shared memory each) and a 512-byte frame (the entropy stage it inlines), no local memory."""
    exe = _cuobjdump()
    if exe is None:
        pytest.skip("cuobjdump not available")
    out = subprocess.run([exe, "-res-usage", LIB], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, check=True).stdout
    found, name = {}, None
    for line in out.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            name = m.group(1)
            continue
        if name and "REG:" in line:
            found[name] = {k: int(v) for k, v in re.findall(r"(REG|STACK|LOCAL):(\d+)", line)}
            name = None
    k = [n for n in found if "lizard_encode_optimal_kernel" in n]
    assert len(k) == 1
    assert found[k[0]] == {"REG": 96, "STACK": 512, "LOCAL": 0}, found[k[0]]


def test_encode_shape_is_the_kernels():
    L = lz.lib()
    w, t, c, s = ctypes.c_int(), ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    for level in LEVELS:
        assert L.LizardB200_encodeShape(level, ctypes.byref(w), ctypes.byref(t), ctypes.byref(c), ctypes.byref(s)) == 0
        assert (w.value, t.value, c.value, s.value) == (4, 0, 5, 0)
    for level in REFUSED:
        assert L.LizardB200_encodeShape(level, ctypes.byref(w), ctypes.byref(t), ctypes.byref(c), ctypes.byref(s)) != 0
