"""GPU parity of the lowestPrice kernel (levels 23-25, 43-45) off the datagen path: the shared corpus and the `collide`
family (long, wrapping and racing probe runs in the per-warp map) with edge capacities, the device call at every alignment
and at the sizes around the inner-block and 4 MiB boundaries, warps that take thousands of different units in turn, big
slots reused after failed units, the encoder workspace handed between LP launches, other encoders and streams, the frame
layer and the block call, and the GPU decoding the GPU's LP streams in full and in part.  Every check compares with the
reference built with -DLIZARD_RESET_MEM, bytes and return values."""
import ctypes
import functools
import random
from collections import Counter

import numpy as np
import pytest

import lizard_b200 as lz
from tests import corpus, refs
from tests.test_gpu_corpus import _layout
from tests.test_gpu_partial import _check as _check_partial

pytestmark = pytest.mark.gpu
BS = corpus.BS
LEVELS = corpus.LP_ENCODE_LEVELS


@pytest.fixture(scope="module")
def ref():
    L = refs.ref_parity()
    if L is None:
        pytest.skip("oracle/_ref not built")
    L.Lizard_decompress_safe_partial.argtypes = [ctypes.c_char_p, ctypes.c_char_p, ctypes.c_int, ctypes.c_int, ctypes.c_int]
    return L


@functools.lru_cache(maxsize=None)
def _families():
    return corpus.lp_corpus()


def _units():
    return [u for us in _families().values() for u in us]


def _mismatches(out, want):
    return [(i, r, len(w)) for i, ((r, o), w) in enumerate(zip(out, want)) if r != len(w) or o != w]


def _want(ref, units, level, caps):
    return [refs.ref_compress(ref, u, level, c) for u, c in zip(units, caps)]


# ---------------------------------------------------------------------------------------------------------------------
# 1-3: the corpus, every alignment, the codeword classes
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("level", LEVELS)
def test_corpus_and_collide_with_edge_capacities(ref, level):
    units = _units()
    caps = corpus.edge_capacities(random.Random(900 + level), units, ref.Lizard_compressBound)
    want = _want(ref, units, level, caps)
    bad = _mismatches(lz.compress_batch(units, level, caps), want)
    assert not bad, (level, len(bad), bad[:8])


def _sized_units(level):
    """Datagen units at the sizes around the inner-block and 4 MiB boundaries, the largest above 4 MiB."""
    sizes = [BS - 1, BS, BS + 1, BS + 21, 2 * BS, (4 << 20) - 1, 4 << 20, (4 << 20) + 1, (4 << 20) + 300000]
    return [lz.datagen(n, 40 + 5 * k, level + k) for k, n in enumerate(sizes)]


@pytest.mark.parametrize("level", LEVELS)
def test_device_call_at_every_alignment_with_guards(ref, level):
    """LizardB200_compress_device with every unit's source and destination at a different residue mod 16: the reference's
    bytes and return values, and not one byte written outside [dst, dst + capacity) of a unit."""
    import torch
    L = lz.lib()
    units = _units() + _sized_units(level)
    rnd = random.Random(level)
    caps = corpus.edge_capacities(rnd, units, ref.Lizard_compressBound)
    want = _want(ref, units, level, caps)
    src_off, dst_off, n_src, n_dst = _layout(rnd, [len(u) for u in units], caps, lambda i: (i + level) % 16,
                                             lambda i: (5 * i + 3) % 16)
    h_src = bytearray(n_src)
    for o, u in zip(src_off, units):
        h_src[o:o + len(u)] = u
    dev = torch.device("cuda", 0)
    d_src = torch.frombuffer(h_src, dtype=torch.uint8).to(dev)
    d_dst = torch.full((n_dst,), 0xEE, dtype=torch.uint8, device=dev)
    t = lambda v, dt: torch.tensor(v, dtype=dt, device=dev)
    t_so, t_sl = t(src_off, torch.int64), t([len(u) for u in units], torch.int32)
    t_do, t_dc = t(dst_off, torch.int64), t(caps, torch.int32)
    t_res = torch.zeros(len(units), dtype=torch.int32, device=dev)
    st = L.LizardB200_compress_device(d_src.data_ptr(), t_so.data_ptr(), t_sl.data_ptr(), d_dst.data_ptr(), t_do.data_ptr(),
                                      t_dc.data_ptr(), t_res.data_ptr(), len(units), level, None)
    assert st == 0, L.LizardB200_lastError()
    torch.cuda.synchronize()
    out = bytes(d_dst.cpu().numpy())
    assert t_res.cpu().tolist() == [len(w) for w in want], level
    outside = bytearray(out)
    for i, (o, c, w) in enumerate(zip(dst_off, caps, want)):
        assert out[o:o + len(w)] == w, (level, i, len(units[i]), o % 16)
        outside[o:o + c] = b"\xEE" * c
    assert outside == b"\xEE" * len(out), "wrote outside a unit's destination"


@functools.lru_cache(maxsize=None)
def _gpu_streams(level):
    """The GPU's streams of the corpus and `collide` at the bound."""
    units = _units()
    out = lz.compress_batch(units, level)
    assert all(r > 0 for r, _ in out), level
    return units, [c for _, c in out]


def test_gpu_streams_reach_the_lowest_price_targets(ref):
    """Walked in Python, the GPU's streams at 23-25 decode to the input and contain every class corpus.lp_targets names:
    2-3 byte repeat matches, 24-bit offsets of both token forms, every extension width."""
    seen = Counter()
    for level in corpus.LP_WALKED_LEVELS:
        units, comp = _gpu_streams(level)
        for i, (u, c) in enumerate(zip(units, comp)):
            assert c == refs.ref_compress(ref, u, level), (level, i)
            back, classes = corpus.walk(c)
            assert back == u, (level, i)
            seen.update(classes)
    missing = sorted(t for t in corpus.lp_targets() if seen[t] == 0)
    assert not missing, missing


# ---------------------------------------------------------------------------------------------------------------------
# 4: warps and big slots reused
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("level", [24, 23])
def test_thousands_of_units_reuse_each_warps_map(ref, level):
    """6400 units of 0 to 128 KiB, cut from the shared corpus and datagen, with the whole `collide` units among them: far
    more units than the kernel's at most 1812 resident warps, so every warp encodes several different units on its map
    under new epochs.  (Pieces of `collide` are left out: a unit that holds a cluster takes a warp about ten times as long
    as a datagen unit, DESIGN.md 3.1a.)"""
    rnd = random.Random(level)
    pool = b"".join(u for u in corpus.corpus_units() if len(u) <= BS) + lz.datagen(4 << 20, 50, level)
    units = list(_families()["collide"])
    while len(units) < 6400:
        n = rnd.choice([0, 1, 5, 21, 22, 300, 4096, 9000, 9000, 30000, 70000, BS])
        at = rnd.randrange(0, len(pool) - n)
        units.append(pool[at:at + n])
    rnd.shuffle(units)
    caps = [ref.Lizard_compressBound(len(u)) if i % 4 else max(len(u) // 2, 1) for i, u in enumerate(units)]
    want = _want(ref, units, level, caps)
    before = lz.lib().LizardB200_launchCount()
    out = lz.compress_batch(units, level, caps)
    assert lz.lib().LizardB200_launchCount() - before == 1
    bad = _mismatches(out, want)
    assert not bad, (level, len(bad), [(i, len(units[i]), r, n) for i, r, n in bad[:8]])


@pytest.mark.parametrize("level", [24, 43])
def test_big_slots_reused_after_failed_units(ref, level):
    """64 units of several inner blocks whose capacities alternate between failing early (len // 50) and the bound, among
    single-block units: each of the 8 big slots is taken again after a unit that failed, and must have been left zero."""
    units, caps = [], []
    for i in range(64):
        n = [BS + 21, 300000, 3 * BS + 1, 500000][i % 4]
        u = lz.datagen(n, 30 + i % 60, 1000 + i)
        units.append(u)
        caps.append(n // 50 if i % 2 == 0 else ref.Lizard_compressBound(n))
        small = _families()["collide"][i // 8] if i % 8 == 0 else lz.datagen(20000 + i, 50, i)
        units.append(small)
        caps.append(ref.Lizard_compressBound(len(small)))
    want = _want(ref, units, level, caps)
    assert sum(1 for w, u in zip(want, units) if not w and len(u) > BS) == 32
    bad = _mismatches(lz.compress_batch(units, level, caps), want)
    assert not bad, (level, len(bad), bad[:8])


# ---------------------------------------------------------------------------------------------------------------------
# 5: the encoder workspace handed over
# ---------------------------------------------------------------------------------------------------------------------
def _device_call(units, level, stream):
    """Enqueue LizardB200_compress_device on `stream`; returns what the result check needs (device tensors kept alive)."""
    import torch
    dev = torch.device("cuda", 0)
    caps = [lz.compress_bound(len(u)) for u in units]
    src_off, dst_off, at, ad = [], [], 0, 0
    for u, c in zip(units, caps):
        src_off.append(at); dst_off.append(ad)
        at += len(u) + 16; ad += c + 16
    h = bytearray(at)
    for o, u in zip(src_off, units):
        h[o:o + len(u)] = u
    with torch.cuda.stream(stream):
        d_src = torch.frombuffer(h, dtype=torch.uint8).to(dev, non_blocking=False)
        d_dst = torch.full((ad,), 0xEE, dtype=torch.uint8, device=dev)
        t = lambda v, dt: torch.tensor(v, dtype=dt, device=dev)
        t_so, t_sl, t_do, t_dc = t(src_off, torch.int64), t([len(u) for u in units], torch.int32), t(dst_off, torch.int64), t(caps, torch.int32)
        t_res = torch.zeros(len(units), dtype=torch.int32, device=dev)
    stream.synchronize()                                    # the inputs are in place; the calls below are enqueued back to back
    keep = (d_src, t_so, t_sl, t_do, t_dc)

    def call():
        st = lz.lib().LizardB200_compress_device(d_src.data_ptr(), t_so.data_ptr(), t_sl.data_ptr(), d_dst.data_ptr(),
                                                 t_do.data_ptr(), t_dc.data_ptr(), t_res.data_ptr(), len(units), level,
                                                 ctypes.c_void_p(stream.cuda_stream))
        assert st == 0, lz.lib().LizardB200_lastError()

    def result():
        out, res = bytes(d_dst.cpu().numpy()), t_res.cpu().tolist()
        return [(r, out[o:o + r] if r > 0 else b"") for o, r in zip(dst_off, res)]
    return call, result, keep


def test_workspace_handed_between_lp_other_levels_and_streams(ref):
    """Each step bit for bit: a level-10 batch writes its per-warp scratch over the region the LP pool occupies; an LP batch
    of single-block units (which does not zero the pool); a level-21 batch of 1 MiB units, whose plain hash tables leave
    positions + 2^24 (valid-looking LP table entries) over the pool; an LP batch with units of several inner blocks (which
    must zero the pool first); then an LP device call on one stream and, at once and without a host sync, a level-10
    device call on another, which must wait for the workspace."""
    import torch
    rnd = random.Random(3)
    blocks = [lz.datagen(BS, rnd.choice([10, 50, 90]), k) for k in range(3000)]
    small = [u for u in _units() if len(u) <= BS]
    big = [lz.datagen(n, 50, n) for n in (BS + 1, 600000, 2 << 20)] + small[:20]
    mib = [b"".join(blocks[8 * k:8 * k + 8]) for k in range(256)]
    steps = [(10, blocks), (24, small), (21, mib), (44, big), (21, blocks[:500]), (25, big), (45, small + big)]
    for level, units in steps:
        want = _want(ref, units, level, [ref.Lizard_compressBound(len(u)) for u in units])
        bad = _mismatches(lz.compress_batch(units, level), want)
        assert not bad, (level, len(bad), bad[:8])
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    lp_units = big + _families()["collide"]
    lp_call, lp_result, k1 = _device_call(lp_units, 25, s1)
    f_call, f_result, k2 = _device_call(blocks[:2000], 10, s2)
    lp_call()
    f_call()
    torch.cuda.synchronize()
    for level, units, res in ((25, lp_units, lp_result()), (10, blocks[:2000], f_result())):
        bad = _mismatches(res, _want(ref, units, level, [ref.Lizard_compressBound(len(u)) for u in units]))
        assert not bad, ("device calls on two streams", level, len(bad), bad[:8])


# ---------------------------------------------------------------------------------------------------------------------
# 6: the frame layer and the block call
# ---------------------------------------------------------------------------------------------------------------------
def _frame_data(kind):
    fam = _families()
    if kind == "raw":       # collide / hostile / random blocks: many are stored raw by the frame layer
        rng = np.random.default_rng(1)
        parts = fam["collide"] + fam["hostile"][:2] + [rng.integers(0, 256, BS, dtype=np.uint8).tobytes()] * 2
        return b"".join(parts) + lz.datagen(300000, 50, 2)
    return lz.datagen((9 << 20) + 4321, 50, 5) + b"".join(fam["collide"][:2])


@pytest.mark.parametrize("checksum", [False, True], ids=["plain", "checksum"])
@pytest.mark.parametrize("kind,block_id", [("raw", 1), ("raw", 4), ("big", 5)])
@pytest.mark.parametrize("level", [23, 44])
def test_compress_frame_matches_reference(level, kind, block_id, checksum):
    """LizardF_compressFrame at 23 and 44: blocks the frame stores raw, blockSizeID 5 (16 MiB blocks: a unit of more than
    4 MiB), with and without the content checksum; the reference's frame byte for byte, and it decodes back."""
    R = refs.ref_parity()
    if R is None:
        pytest.skip("oracle/_ref not built")
    theirs, ours = lz.bind_frame_api(R), lz.bind_frame_api(lz.lib())
    data = _frame_data(kind)
    p = lz.make_prefs(level, block_id, True, checksum, 0)
    got = lz.frame_compress(ours, data, p)
    assert got == lz.frame_compress(theirs, data, p), (level, kind, block_id, checksum)
    r, back = lz.frame_decompress(ours, got, len(data))
    assert r == 0 and back == data


@pytest.mark.parametrize("level", [25, 43])
def test_compress_blocks_with_failing_blocks(ref, level):
    """LizardB200_compress_blocks at an LP level, 1 MiB blocks (units of 8 inner blocks) with a dstCapacityEach that random
    blocks overflow: the reference's result (0 for those) and bytes for every block."""
    L = lz.lib()
    mb = 1 << 20
    rng = np.random.default_rng(level)
    blocks = []
    for k in range(10):
        blocks.append(rng.integers(0, 256, mb, dtype=np.uint8).tobytes() if k % 3 == 1 else lz.datagen(mb, 30 + 5 * k, k))
    data = b"".join(blocks) + lz.datagen(12345, 50, 1)
    blocks.append(data[len(blocks) * mb:])
    cap = mb - 1
    n = len(blocks)
    src = np.frombuffer(data, dtype=np.uint8).copy()
    dst = np.zeros(n * mb, dtype=np.uint8)
    res = np.zeros(n, dtype=np.int32)
    st = L.LizardB200_compress_blocks(src.ctypes.data, len(data), mb, dst.ctypes.data, mb, cap, res.ctypes.data, level)
    assert st == 0, L.LizardB200_lastError()
    want = _want(ref, blocks, level, [cap] * n)
    assert res.tolist() == [len(w) for w in want]
    assert sum(1 for w in want if not w) >= 3
    for i, w in enumerate(want):
        assert dst[i * mb:i * mb + len(w)].tobytes() == w, (level, i)


# ---------------------------------------------------------------------------------------------------------------------
# 7: the GPU decodes the GPU's LP streams
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("level", [23, 24, 25])
def test_gpu_decodes_lp_streams_in_full_and_inside_short_repeats(ref, level):
    """The GPU's streams of the corpus and `collide` decode back on the GPU; partial decodes whose targets fall inside (and
    at either end of) 2-3 byte repeat matches, where only lowestPrice puts a match boundary, agree with the reference's
    Lizard_decompress_safe_partial."""
    units, comp = _gpu_streams(level)
    back = lz.decompress_batch(comp, [len(u) for u in units])
    assert all(r == len(u) and o == u for (r, o), u in zip(back, units)), level
    part, targets, caps = [], [], []
    for u, c in zip(units, comp):
        at = []
        corpus.walk(c, at)
        for p in at[:40]:
            for t in (p, p + 1, p + 2):
                part.append(c); targets.append(t); caps.append(len(u))
    assert len(part) >= 300, len(part)
    out = lz.decompress_partial_batch(part, targets, caps)
    compared = _check_partial(ref, part, targets, caps, [r for r, _ in out], [o for _, o in out], level)
    assert compared > 0
    for level2 in ((43, 44, 45) if level == 25 else ()):     # the Huffman twins' streams decode back too
        u2, c2 = _gpu_streams(level2)
        back = lz.decompress_batch(c2, [len(u) for u in u2])
        assert all(r == len(u) and o == u for (r, o), u in zip(back, u2)), level2
