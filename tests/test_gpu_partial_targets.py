"""Partial decoding on the H100 at its edges: every target of a ~100-token stream at every level 10-49 (exits on every lane
of several 32-token batches, Huffman-coded and plain streams of both codeword flavours mixed in one launch), the stops
around inner-block boundaries with the block-relative target and small capacities, damage in front of and behind the
stopping point, and the device call at every residue mod 16 with guard bytes.  The yardstick is the reference's
Lizard_decompress_safe_partial (built with -DLIZARD_RESET_MEM), compared as tests/test_gpu_partial.py::_check does."""
import ctypes
import functools
import random

import numpy as np
import pytest

import lizard_b200 as lz
from tests import corpus, refs
from tests.test_gpu_corpus import _decode_variant, _layout
from tests.test_gpu_partial import _check
from tests.test_partial_cpu import _damage, _level_inputs, _sweep_boundaries, _token_streams, ref_partial

pytestmark = pytest.mark.gpu
BS = lz.BLOCK_SIZE
GUARD = 0xEE


@pytest.fixture(scope="module")
def ref():
    L = refs.ref_parity()
    if L is None:
        pytest.skip("oracle/_ref not built")
    L.Lizard_decompress_safe_partial.argtypes = [ctypes.c_char_p, ctypes.c_char_p, ctypes.c_int, ctypes.c_int, ctypes.c_int]
    return L


@functools.lru_cache(maxsize=None)
def _every_target(ref, level):
    """The stream of test_partial_cpu.py::test_every_token_boundary with 2000 more bytes of datagen (without them the
    priceFast LIZv1 levels 21, 22, 41 and 42 stop at only 57 places) at `level`, its decoded size n, the targets -1 .. n + 1
    and the reference's result at each with capacity n.  The stream obeys the min-offset rule, so the reference's bytes are
    the input's first `result` bytes (checked here once; the comparisons then need only the results)."""
    data = lz.datagen(6000, 50, 3) + corpus.periodic_units()[0][:1500] + lz.datagen(2000, 40, 5)
    comp = refs.ref_compress(ref, data, level)
    n = len(data)
    assert refs.stream_obeys_min_offset(comp, n)
    targets = list(range(-1, n + 2))
    want = []
    for t in targets:
        r, o = ref_partial(ref, comp, t, n)
        assert r <= n and o == data[:max(r, 0)], (level, t, r)
        want.append(r)
    return data, comp, targets, want


def _differences(data, want, got):
    """Units whose result is not the reference's, or whose bytes are not the input's first `result` bytes."""
    return [(i, r, w) for i, ((r, o), w) in enumerate(zip(got, want)) if r != w or (r > 0 and o != data[:r])]


# ---------------------------------------------------------------------------------------------------------------------
# P1: every target at every level
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("level", range(10, 50))
def test_every_target_at_every_level(ref, level):
    """All n + 3 targets of one stream in one LizardB200_decompress_partial_batch call (one launch, about 9.5k units) under
    decode variants 3, 7 and 23: the reference's result at every target, the same results under every variant, and at
    least 64 places where the reference stops, so that exits fall on every lane of two 32-token batches or more."""
    data, comp, targets, want = _every_target(ref, level)
    n = len(data)
    stops = _sweep_boundaries(ref, comp, n)
    assert len(stops) >= 64, (level, len(stops))
    assert sorted(set(want)) == stops
    L = lz.lib()
    seen = None
    for variant in (3, 7, 23):
        with _decode_variant(variant):
            before = L.LizardB200_launchCount()
            out = lz.decompress_partial_batch([comp] * len(targets), targets, [n] * len(targets))
            assert L.LizardB200_launchCount() - before == 1, (level, variant)
        bad = _differences(data, want, out)
        assert not bad, (level, variant, len(bad), bad[:10])
        if seen is None:
            seen = out
        assert out == seen, (level, variant)


def test_every_eighth_target_of_every_level_in_one_launch(ref):
    """Every eighth target of every level 10-49, about 47k units shuffled together, so that each decode warp takes units of
    different levels, codeword flavours and Huffman states in turn: one launch, and at every unit the result of the
    per-level calls above (the reference's)."""
    rows = []
    for level in range(10, 50):
        data, comp, targets, want = _every_target(ref, level)
        rows += [(level, comp, t, w) for t, w in list(zip(targets, want))[::8]]
    random.Random(8).shuffle(rows)
    assert len(rows) > 45000 and len({lv for lv, _, _, _ in rows[:32]}) > 16
    L = lz.lib()
    before = L.LizardB200_launchCount()
    caps = [len(_every_target(ref, lv)[0]) for lv, _, _, _ in rows]
    out = lz.decompress_partial_batch([c for _, c, _, _ in rows], [t for _, _, t, _ in rows], caps)
    assert L.LizardB200_launchCount() - before == 1
    bad = [(i, lv, t, r, w) for i, ((lv, _, t, w), (r, o)) in enumerate(zip(rows, out))
           if r != w or (r > 0 and o != _every_target(ref, lv)[0][:r])]
    assert not bad, (len(bad), bad[:10])


# ---------------------------------------------------------------------------------------------------------------------
# P2: stops around inner blocks, the block-relative target, capacities
# ---------------------------------------------------------------------------------------------------------------------
LISTED = [-1, 0, 1, 4000, 65536, BS - 1, BS, BS + 1, BS + 20000, 200000, 2 * BS - 1, 2 * BS, 2 * BS + 1, 300000, 3 * BS,
          3 * BS + 1]
CAP_TARGETS = [-1, 0, 1, 50, 4000, BS - 1, BS + 1, 200000]


@pytest.mark.parametrize("level", [10, 21, 30, 41, 45])
def test_stops_around_inner_blocks_and_small_capacities(ref, level):
    """The four-inner-block unit of test_inner_block_boundaries_and_the_block_relative_target and the unit whose first inner
    block is stored raw (test_raw_inner_block_before_a_compressed_one), in one batch: every place the reference stops for
    targets within 300 bytes of an inner-block boundary and one byte either side of it, the listed targets (200000 returns
    262144, a raw first block is copied whole), and capacities 0, 1, 15, 16, 17, n / 2 and n - 1 at a subset of targets."""
    four = lz.datagen(3 * BS + 7000, 50, level)
    raw_first = np.random.default_rng(level).integers(0, 256, BS, dtype=np.uint8).tobytes() + lz.datagen(40000, 50, level)
    units, targets, caps = [], [], []
    for data, bounds in ((four, (BS, 2 * BS, 3 * BS)), (raw_first, (BS,))):
        comp = refs.ref_compress(ref, data, level)
        n = len(data)
        stops = {ref_partial(ref, comp, t, n)[0] for b in bounds for t in range(b - 300, b + 301)}
        near = sorted({s + d for s in stops for d in (-1, 0, 1)} | {t for t in LISTED if t <= n + 1} | {n - 1, n, n + 1})
        for t in near:
            units.append(comp); targets.append(t); caps.append(n)
        for cap in (0, 1, 15, 16, 17, n // 2, n - 1):
            for t in CAP_TARGETS + [n // 2, n - 1, n]:
                units.append(comp); targets.append(t); caps.append(cap)
    assert refs.ref_compress(ref, raw_first, level)[1] == 0x80
    L = lz.lib()
    before = L.LizardB200_launchCount()
    out = lz.decompress_partial_batch(units, targets, caps)
    assert L.LizardB200_launchCount() - before == 1
    assert _check(ref, units, targets, caps, [r for r, _ in out], [o for _, o in out], level) > 20
    n4 = len(four)
    got = {(len(u), t, c): r for u, t, c, (r, _) in zip(units, targets, caps, out)}
    four_len = len(refs.ref_compress(ref, four, level))
    assert got[(four_len, 200000, n4)] == 2 * BS
    assert got[(four_len, BS + 1, n4)] == 2 * BS and got[(four_len, 2 * BS + 1, n4)] == 3 * BS
    raw_len = len(refs.ref_compress(ref, raw_first, level))
    assert [got[(raw_len, t, len(raw_first))] for t in (-1, 0, 1)] == [BS] * 3


# ---------------------------------------------------------------------------------------------------------------------
# P3: damage in front of and behind the stop
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("level", [10, 20, 21, 30, 41])
def test_damage_in_front_of_and_behind_the_stop(ref, level):
    """test_partial_cpu.py::test_damage_in_front_of_and_behind_the_stopping_point in one batch of about 200 units: a unit of
    two inner blocks damaged in the offset and flags streams of one of them, decoded to targets in both.  Both outcomes
    occur: the reference's error for damage in front of the stop, success (as in the reference) with the damage behind it."""
    rnd = random.Random(900 + level)
    data = lz.datagen(BS + 30000, 50, level)
    comp = refs.ref_compress(ref, data, level)
    n = len(data)
    blocks = _token_streams(comp)
    assert len(blocks) == 2, blocks
    units, targets, full = [], [], []
    for k in range(67):
        lo, hi = blocks[k % 2]
        bad = _damage(rnd, comp, lo, hi)
        f = refs.ref_decompress(ref, bad, n)[0]
        for t in (rnd.randrange(-1, 3000), rnd.randrange(0, BS - 100), rnd.randrange(BS, n + 10)):
            units.append(bad); targets.append(t); full.append(f)
    caps = [n] * len(units)
    L = lz.lib()
    before = L.LizardB200_launchCount()
    out = lz.decompress_partial_batch(units, targets, caps)
    assert L.LizardB200_launchCount() - before == 1
    _check(ref, units, targets, caps, [r for r, _ in out], [o for _, o in out], level)
    accepted_behind = sum(1 for (r, _), f in zip(out, full) if f < 0 and r > 0)
    failed_in_front = sum(1 for r, _ in out if r < 0)
    assert accepted_behind > 0 and failed_in_front > 0, (accepted_behind, failed_in_front)


# ---------------------------------------------------------------------------------------------------------------------
# P4: the device call
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("level", [10, 21, 41, 45])
def test_device_call_at_every_target_and_residue(ref, level):
    """The units of test_every_target_at_every_level through LizardB200_decompress_partial_device, with the small units of
    test_partial_cpu.py at a few targets: sources and destinations at every residue mod 16 between guard bytes, targets in
    device memory.  The reference's results and bytes, and no byte outside any unit's [dst, dst + capacity) changed."""
    import torch
    data, comp, targets, want = _every_target(ref, level)
    units, caps = [comp] * len(targets), [len(data)] * len(targets)
    targets, extra = list(targets), []
    for u in _level_inputs(level)[:6]:
        c = refs.ref_compress(ref, u, level)
        for t in (-1, 0, 1, len(u) // 3, len(u) - 1, len(u)):
            units.append(c); targets.append(t); caps.append(len(u))
            extra.append(len(units) - 1)
    rnd = random.Random(level)
    src_off, dst_off, n_src, n_dst = _layout(rnd, [len(c) for c in units], caps, lambda i: i % 16, lambda i: (7 * i + 3) % 16)
    h_src = bytearray(n_src)
    for o, c in zip(src_off, units):
        h_src[o:o + len(c)] = c
    dev = torch.device("cuda", 0)
    L = lz.lib()
    d_src = torch.frombuffer(h_src, dtype=torch.uint8).to(dev)
    d_dst = torch.full((n_dst,), GUARD, dtype=torch.uint8, device=dev)
    t = lambda v, dt: torch.tensor(v, dtype=dt, device=dev)
    t_so, t_sl = t(src_off, torch.int64), t([len(c) for c in units], torch.int32)
    t_do, t_dc, t_tg = t(dst_off, torch.int64), t(caps, torch.int32), t(targets, torch.int32)
    t_res = torch.zeros(len(units), dtype=torch.int32, device=dev)
    before = L.LizardB200_launchCount()
    st = L.LizardB200_decompress_partial_device(d_src.data_ptr(), t_so.data_ptr(), t_sl.data_ptr(), d_dst.data_ptr(),
                                                t_do.data_ptr(), t_dc.data_ptr(), t_tg.data_ptr(), t_res.data_ptr(),
                                                len(units), None)
    assert st == 0, L.LizardB200_lastError()
    torch.cuda.synchronize()
    assert L.LizardB200_launchCount() - before == 1
    out = d_dst.cpu().numpy().tobytes()
    res = t_res.cpu().tolist()
    k = len(want)
    bad = _differences(data, want, [(r, out[o:o + max(r, 0)]) for r, o in zip(res[:k], dst_off[:k])])
    assert not bad, (level, len(bad), bad[:10])
    _check(ref, [units[i] for i in extra], [targets[i] for i in extra], [caps[i] for i in extra], [res[i] for i in extra],
           [out[dst_off[i]:dst_off[i] + caps[i]] for i in extra], (level, "small units"))
    outside = bytearray(out)
    for o, c in zip(dst_off, caps):
        outside[o:o + c] = bytes([GUARD]) * c
    assert outside == bytes([GUARD]) * len(out), (level, "wrote outside a unit's destination")
