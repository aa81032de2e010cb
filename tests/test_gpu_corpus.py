"""GPU parity on the shared corpus (tests/corpus.py): far offsets, codeword-boundary lengths, Huffman-hostile literals and
periodic data, encoded at every level the GPU implements under three launch shapes (so both hash-table forms run on
purpose), by warps that take many different units in turn, and through the device API at every alignment; decoded at every
level 10-49 by both decoder generations, with and without the Huffman pre-pass, damaged, in a batch of thousands of small
units, and at unaligned device offsets.  The reference built with -DLIZARD_RESET_MEM is the yardstick throughout."""
import contextlib
import ctypes
import functools
import os
import random
from collections import Counter

import pytest

import lizard_b200 as lz
from tests import corpus, refs

pytestmark = pytest.mark.gpu
BS = corpus.BS
DEFAULT_VARIANT = 7                      # api.cu Context::dec_variant
HAS_SMEM_TABLE = {10, 20, 21, 30, 40, 41}     # hashLog <= 14: the levels whose warps can keep a packed shared-memory table
# launch shapes "warps,tables,ctas": the level's measured one; every warp on the plain global table; one warp per CTA, each
# with a shared-memory table where the level has one
SHAPES = (("default", None), ("plain", "14,0,2"), ("packed", "1,1,8"))


@pytest.fixture(scope="module")
def ref():
    L = refs.ref_parity()
    if L is None:
        pytest.skip("oracle/_ref not built")
    return L


@functools.lru_cache(maxsize=None)
def _families():
    return corpus.corpus()


def _units():
    return [u for units in _families().values() for u in units]


@functools.lru_cache(maxsize=None)
def _encode_case(level):
    """The corpus with destination capacities drawn like test_edge_inputs_and_capacities, and the reference's output."""
    L = refs.ref_parity()
    units = _units()
    caps = corpus.edge_capacities(random.Random(500 + level), units, L.Lizard_compressBound)
    return units, caps, [refs.ref_compress(L, u, level, c) for u, c in zip(units, caps)]


@functools.lru_cache(maxsize=None)
def _decode_case(level):
    L = refs.ref_parity()
    units = _units()
    return units, [refs.ref_compress(L, u, level) for u in units]


@contextlib.contextmanager
def _enc_shape(value):
    old = os.environ.get("LIZARDB200_ENC_SHAPE")
    if value is None:
        os.environ.pop("LIZARDB200_ENC_SHAPE", None)
    else:
        os.environ["LIZARDB200_ENC_SHAPE"] = value
    try:
        yield
    finally:
        if old is None:
            os.environ.pop("LIZARDB200_ENC_SHAPE", None)
        else:
            os.environ["LIZARDB200_ENC_SHAPE"] = old


def _shape(level):
    v = [ctypes.c_int() for _ in range(4)]
    assert lz.lib().LizardB200_encodeShape(level, *[ctypes.byref(x) for x in v]) == 0
    return tuple(x.value for x in v[:3])


def _expect_shape(level, value):
    w, t, k = (int(x) for x in value.split(","))
    return (w, t if level in HAS_SMEM_TABLE else 0, k)


@contextlib.contextmanager
def _decode_variant(variant):
    L = lz.lib()
    L.LizardB200_setDecodeVariant.argtypes = [ctypes.c_int]
    assert L.LizardB200_setDecodeVariant(variant) == 0
    try:
        yield
    finally:
        L.LizardB200_setDecodeVariant(DEFAULT_VARIANT)


def _mismatches(out, want):
    return [(i, r, len(w)) for i, ((r, o), w) in enumerate(zip(out, want)) if r != len(w) or o != w]


# ---------------------------------------------------------------------------------------------------------------------
# encode
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("level", corpus.ENCODE_LEVELS)
def test_corpus_encodes_bit_exact_under_every_launch_shape(ref, level):
    units, caps, want = _encode_case(level)
    default = _shape(level)
    for name, value in SHAPES:
        with _enc_shape(value):
            shape = _shape(level)
            assert shape == (default if value is None else _expect_shape(level, value)), (level, name, shape)
            out = lz.compress_batch(units, level, caps)
        bad = _mismatches(out, want)
        assert not bad, (level, name, shape, len(bad), bad[:8])


def _mixed_units(rnd, count):
    """`count` units cut at random places from datagen data and the corpus: lengths 0, 1, 5, 21, 4096, 70000 and 128 KiB,
    plus four multi-inner-block units of 1-4 MiB, in random order."""
    pool = lz.datagen(6 << 20, 50, 9) + b"".join(_units())
    sizes = [0, 1, 5, 21] * 120 + [4096] * 300 + [70000] * 60 + [BS] * 40
    sizes = (sizes * (count // len(sizes) + 1))[:count - 4] + [(1 << 20) + 4321, 2 << 20, 3 << 20, 4 << 20]
    rnd.shuffle(sizes)
    out = []
    for n in sizes:
        at = rnd.randrange(0, len(pool) - n)
        out.append(pool[at:at + n])
    return out


@pytest.mark.parametrize("level", [10, 21, 41, 13])
def test_one_warp_per_sm_encodes_many_different_units_in_turn(ref, level):
    """LIZARDB200_ENC_SHAPE=1,1,1 leaves one encode warp per SM, so each warp runs about eight units of every size in a row
    with the same table, scratch and shared memory: multi-inner-block units (plain 1 MiB table, untagged), single blocks
    (packed table where the level has one) and units of a few bytes."""
    units = _mixed_units(random.Random(level), 1000)
    want = [refs.ref_compress(ref, u, level) for u in units]
    with _enc_shape("1,1,1"):
        assert _shape(level) == _expect_shape(level, "1,1,1")
        out = lz.compress_batch(units, level)
    bad = _mismatches(out, want)
    assert not bad, (level, len(bad), [(i, len(units[i]), r, n) for i, r, n in bad[:8]])


def _layout(rnd, sizes, caps, residue_src, residue_dst):
    """Offsets with the given residues mod 16 and gaps between the units."""
    src_off, dst_off, ps, pd = [], [], 64, 64
    for i, (n, c) in enumerate(zip(sizes, caps)):
        ps += (residue_src(i) - ps) % 16 + 16 * rnd.randrange(0, 3)
        pd += (residue_dst(i) - pd) % 16 + 16 * rnd.randrange(0, 3)
        src_off.append(ps); dst_off.append(pd)
        ps += n; pd += c
    return src_off, dst_off, ps + 64, pd + 64


@pytest.mark.parametrize("level", corpus.ENCODE_LEVELS)
def test_device_api_encodes_at_every_alignment(ref, level):
    """LizardB200_compress_device with every unit's source and destination at a different residue mod 16 (the device-only
    unaligned loads of lanes.cuh): the reference's bytes and return values, and not one byte written outside
    [dst, dst + capacity) of a unit."""
    import torch
    L = lz.lib()
    units, caps, want = _encode_case(level)
    rnd = random.Random(level)
    src_off, dst_off, n_src, n_dst = _layout(rnd, [len(u) for u in units], caps, lambda i: i % 16, lambda i: (5 * i + 3) % 16)
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
    res = t_res.cpu().tolist()
    assert res == [len(w) for w in want], level
    outside = bytearray(out)
    for i, (o, c, w) in enumerate(zip(dst_off, caps, want)):
        assert out[o:o + len(w)] == w, (level, i, o % 16)
        outside[o:o + c] = b"\xEE" * c
    assert outside == b"\xEE" * len(out), "wrote outside a unit's destination"


@pytest.mark.parametrize("lizv1", [False, True], ids=["lz4", "lizv1"])
def test_gpu_streams_reach_every_targeted_class(lizv1):
    """The non-Huffman streams the GPU makes of the corpus, walked in Python: they decode to the input and, per family over
    the walked levels of the flavour, contain every codeword class the family targets (corpus.targets).  Fails, naming the
    classes, if the corpus stops reaching a boundary."""
    levels = [lv for lv in corpus.WALKED_ENCODE_LEVELS if corpus.is_lizv1(lv) == lizv1]
    fams = _families()
    seen = {name: Counter() for name in fams}
    for level in levels:
        for name, units in fams.items():
            for u, (r, c) in zip(units, lz.compress_batch(units, level)):
                assert r > 0, (level, name, len(u))
                back, classes = corpus.walk(c)
                assert back == u, (level, name, len(u))
                seen[name].update(classes)
    missing = {name: corpus.missing(name, lizv1, seen[name]) for name in fams}
    assert not any(missing.values()), (levels, missing)


# ---------------------------------------------------------------------------------------------------------------------
# decode
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("level", range(10, 50))
def test_corpus_decodes_at_every_level_both_generations_and_prepass_states(ref, level):
    """Every level 10-49, the decode-only ones included.  A batch of >= 32 units under variant 7 must run the Huffman
    pre-pass (plan + expand + token kernel: 3 launches); variant 3 and batches of fewer than 32 units must not (1 launch);
    variant 23 is the second-generation kernel behind the same pre-pass."""
    units, comp = _decode_case(level)
    assert len(units) >= 32
    L = lz.lib()
    for variant, n, launches in ((7, len(units), 3), (7, 31, 1), (3, len(units), 1), (23, len(units), 3), (23, 31, 1)):
        with _decode_variant(variant):
            before = L.LizardB200_launchCount()
            out = lz.decompress_batch(comp[:n], [len(u) for u in units[:n]])
            assert L.LizardB200_launchCount() - before == launches, (level, variant, n)
        bad = [(i, r) for i, ((r, o), u) in enumerate(zip(out, units[:n])) if r != len(u) or o != u]
        assert not bad, (level, variant, n, bad[:8])


def _damage(rnd, comp):
    b = bytearray(comp)
    mode = rnd.randrange(4)
    if mode == 0:
        b[rnd.randrange(len(b))] ^= 1 << rnd.randrange(8)
    elif mode == 1:
        b = b[:rnd.randrange(1, len(b))]
    elif mode == 2:
        b[rnd.randrange(min(40, len(b)))] = rnd.randrange(256)
    else:
        for _ in range(3):
            b[rnd.randrange(len(b))] = rnd.randrange(256)
    return bytes(b)


def _check_against_reference(ref, units, caps, out, what):
    """Same return codes as the reference, same bytes where the reference's are defined.  One documented exception
    (DESIGN.md 3.5): behind a raw inner block the reference decodes past the capacity and reports more than `cap`; the
    device refuses such a unit."""
    bad, compared = [], 0
    for i, (u, cap, (r, o)) in enumerate(zip(units, caps, out)):
        rr, ro = refs.ref_decompress(ref, u, cap)
        if rr > cap:
            if r >= 0:
                bad.append((i, len(u), cap, r, rr, "accepted an overrun"))
        elif r != rr:
            bad.append((i, len(u), cap, r, rr))
        elif rr > 0 and refs.stream_obeys_min_offset(u, cap):
            compared += 1
            if o != ro:
                bad.append((i, len(u), cap, "content"))
    assert not bad, (what, len(bad), bad[:10])
    return compared


@pytest.mark.parametrize("level", [20, 21, 22, 26, 29, 40, 41, 42, 45, 49, 10, 30])
def test_damaged_far_and_hostile_streams_match_reference(ref, level):
    """Damaged copies of the far-offset and Huffman-hostile streams: the reference's return codes always, its bytes where
    they are defined (every offset >= 8), with the pre-pass on (variant 7) and on the second generation (23)."""
    rnd = random.Random(700 + level)
    fams = _families()
    _, comp = _decode_case(level)
    first = {name: sum(len(v) for v in list(fams.values())[:k]) for k, name in enumerate(fams)}
    streams = [(comp[first[name] + j], len(u)) for name in ("far", "hostile") for j, u in enumerate(fams[name])]
    bad, caps = [], []
    for c, n in streams:
        for _ in range(12):
            bad.append(_damage(rnd, c))
            caps.append(rnd.choice([n, n, max(n - 1, 0), n + 100]))
    compared = 0
    for variant in (7, 23):
        with _decode_variant(variant):
            out = lz.decompress_batch(bad, caps)
        compared += _check_against_reference(ref, bad, caps, out, (level, variant))
    assert compared > 0


def test_thousands_of_small_units_of_every_level_in_one_batch(ref):
    """5200 small units compressed at every level 10-49, a tenth of them damaged, in one batch: each decode warp takes
    dozens of units in turn, across codeword flavours, Huffman and plain streams, valid and broken ones."""
    rnd = random.Random(5)
    pool = lz.datagen(1 << 20, 50, 4) + b"".join(_units()[:20])
    distinct = []
    for _ in range(640):
        n = rnd.choice([0, 1, 5, 16, 100, 700, 2000, 4096, 9000])
        at = rnd.randrange(0, len(pool) - n)
        raw = pool[at:at + n]
        distinct.append((refs.ref_compress(ref, raw, rnd.randrange(10, 50)), n))
    units, caps = [], []
    for _ in range(5200):
        c, n = rnd.choice(distinct)
        if len(c) > 1 and rnd.random() < 0.1:
            c = _damage(rnd, c)
        units.append(c)
        caps.append(n)
    for variant in (7, 23):
        with _decode_variant(variant):
            out = lz.decompress_batch(units, caps)
        assert _check_against_reference(ref, units, caps, out, variant) > 1000


@pytest.mark.parametrize("variant", [7, 23], ids=["gen1", "gen2"])
def test_device_api_decodes_far_and_threshold_streams_at_unaligned_offsets(ref, variant):
    """LizardB200_decompress_device with the far-offset and codeword-threshold streams at every residue mod 16 of source and
    destination: the original bytes, the sizes as results, nothing touched outside [dst, dst + size)."""
    import torch
    L = lz.lib()
    fams = _families()
    dev = torch.device("cuda", 0)
    for level in (20, 21, 22, 41, 10, 30, 45, 29):
        _, comp = _decode_case(level)
        blocks = fams["far"] + fams["threshold"]
        comp = comp[:len(blocks)]                   # far and threshold are the first two families
        rnd = random.Random(level)
        src_off, dst_off, n_src, n_dst = _layout(rnd, [len(c) for c in comp], [len(b) for b in blocks],
                                                 lambda i: (3 * i + level) % 16, lambda i: (7 * i + 1) % 16)
        h_src = bytearray(n_src)
        for o, c in zip(src_off, comp):
            h_src[o:o + len(c)] = c
        d_src = torch.frombuffer(h_src, dtype=torch.uint8).to(dev)
        d_dst = torch.full((n_dst,), 0xEE, dtype=torch.uint8, device=dev)
        t = lambda v, dt: torch.tensor(v, dtype=dt, device=dev)
        t_so, t_sl = t(src_off, torch.int64), t([len(c) for c in comp], torch.int32)
        t_do, t_dc = t(dst_off, torch.int64), t([len(b) for b in blocks], torch.int32)
        t_res = torch.zeros(len(blocks), dtype=torch.int32, device=dev)
        with _decode_variant(variant):
            st = L.LizardB200_decompress_device(d_src.data_ptr(), t_so.data_ptr(), t_sl.data_ptr(), d_dst.data_ptr(),
                                                t_do.data_ptr(), t_dc.data_ptr(), t_res.data_ptr(), len(blocks), None)
            assert st == 0, L.LizardB200_lastError()
            torch.cuda.synchronize()
        out = bytes(d_dst.cpu().numpy())
        assert t_res.cpu().tolist() == [len(b) for b in blocks], level
        want = bytearray(b"\xEE" * len(out))
        for o, b in zip(dst_off, blocks):
            want[o:o + len(b)] = b
        assert out == bytes(want), level
