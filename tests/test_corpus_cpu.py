"""CPU checks of the shared corpus (tests/corpus.py): the Python walker decodes like the compiled reference, the reference's
streams of the corpus reach every codeword class the families are built for, and the new families give the reference's
bytes through the one-lane host build and the 32-lane emulator of the device code at every level the GPU encodes.  A later
GPU mismatch on this corpus then points either at shared code (these fail too) or at a device-only branch (they pass)."""
import functools
import random
from collections import Counter

import pytest

from tests import corpus, refs
from tests.test_oracle import emu_compress, lz_bound, shim, shim_compress   # noqa: F401  (shim is a fixture)

BS = corpus.BS


@pytest.fixture(scope="module")
def ref():
    L = refs.ref_parity()
    if L is None:
        pytest.skip("oracle/_ref not built (needs /root/reference)")
    return L


@functools.lru_cache(maxsize=None)
def _corpus():
    return corpus.corpus()


@functools.lru_cache(maxsize=None)
def _ref_streams(level):
    L = refs.ref_parity()
    return {name: [refs.ref_compress(L, u, level) for u in units] for name, units in _corpus().items()}


@pytest.mark.parametrize("level", range(10, 30))
def test_walker_decodes_like_the_reference(ref, level):
    """Every non-Huffman level, decode-only ones included: the walker's bytes are the input and the reference's output."""
    for name, units in _corpus().items():
        for u, c in zip(units, _ref_streams(level)[name]):
            out, _ = corpus.walk(c)
            assert out == u, (level, name, len(u))
            r, back = refs.ref_decompress(ref, c, len(u))
            assert r == len(u) and back == out, (level, name, len(u))
    for u in corpus.inputs(5, 25):
        assert corpus.walk(refs.ref_compress(ref, u, level))[0] == u, (level, len(u))


def test_walker_refuses_huffman_streams_and_bad_offsets(ref):
    with pytest.raises(NotImplementedError):
        corpus.walk(refs.ref_compress(ref, _corpus()["hostile"][0], 41))
    bad = bytearray(refs.ref_compress(ref, b"abcdefgh" * 100, 10))
    assert corpus.walk(bytes(bad))[0] == b"abcdefgh" * 100
    i = bad.index(b"abcdefgh\x08\x00") + 8          # eight literals, then the first match's offset (8)
    bad[i:i + 2] = b"\xff\x7f"                          # 32767 bytes back from position 8
    with pytest.raises(ValueError):
        corpus.walk(bytes(bad))


@pytest.mark.parametrize("lizv1", [False, True], ids=["lz4", "lizv1"])
def test_reference_streams_reach_every_targeted_class(ref, lizv1):
    """The corpus is only worth its cost while the reference's streams of it hit the boundaries: per family, summed over the
    walked encode levels of the flavour, every class of corpus.targets() occurs."""
    levels = [lv for lv in corpus.WALKED_ENCODE_LEVELS if corpus.is_lizv1(lv) == lizv1]
    for name in _corpus():
        seen = Counter()
        for level in levels:
            for c in _ref_streams(level)[name]:
                seen.update(corpus.walk(c)[1])
        assert not corpus.missing(name, lizv1, seen), (name, levels, corpus.missing(name, lizv1, seen))


def _emu_subset(units, name, level):
    """What the coroutine emulator (slow) runs: one far block (LIZv1 levels; with a 64 KiB window it is literals), the
    short-boundary block and one 64 KiB+ block of the level's flavour, the Huffman-hostile blocks cut to 8 KiB, the periodic
    units; at the hash-chain levels (the slowest under the emulator) two units of each family, cut to 20000 bytes."""
    lizv1 = corpus.is_lizv1(level)
    if name == "far":
        out = units[:1] if lizv1 else []
    elif name == "threshold":
        out = units[5:7] if lizv1 else units[0:2]
    elif name == "hostile":
        out = [u[:8192] for u in units]
    else:
        out = list(units)
    if level in (13, 14, 15, 16, 17, 34, 35, 36, 37, 38):
        out = [u[:20000] for u in out[:2]]
    return out


@pytest.mark.parametrize("level", corpus.ENCODE_LEVELS)
def test_new_families_one_lane_and_emulated_bit_exact(ref, shim, level):
    rnd = random.Random(300 + level)
    for name, units in _corpus().items():
        caps = corpus.edge_capacities(rnd, units, lz_bound)
        for u, cap in zip(units, caps):
            for c in (cap, lz_bound(len(u))):
                assert shim_compress(shim, u, level, c) == refs.ref_compress(ref, u, level, c), (level, name, len(u), c)
        for u in _emu_subset(units, name, level):
            assert emu_compress(shim, u, level) == refs.ref_compress(ref, u, level), (level, name, len(u))
