"""Lizard_createStream + Lizard_loadDict + Lizard_compress_continue at the hashChain levels (13-17, 34-38) and the priceFast
levels (21, 22, 41, 42) through the device
encoder's code on the CPU: the one-lane host build and the 32-lane warp emulator (lizard_b200/libhostshim.so, TEST-ONLY)
against the compiled reference, byte for byte and with the same return value.  Both layouts count: the dictionary directly
in front of the input (prefix) and a dictionary somewhere else (external)."""
import ctypes
import functools
import os
import random
from collections import Counter

import pytest

from tests import corpus, refs
from tests.test_dict_cpu import _dictionary, _straddler, records

HC_LEVELS = list(range(13, 18)) + list(range(34, 39))
PF_LEVELS = [21, 22, 41, 42]
DICT_LEVELS = HC_LEVELS + PF_LEVELS
DICT_LIMIT = 1 << 24


def _bind_stream(L):
    vp, ci = ctypes.c_void_p, ctypes.c_int
    L.Lizard_createStream.restype = vp
    L.Lizard_createStream.argtypes = [ci]
    L.Lizard_freeStream.argtypes = [vp]
    L.Lizard_loadDict.argtypes = [vp, vp, ci]
    L.Lizard_compress_continue.argtypes = [vp, vp, vp, ci, ci]
    return L


def lz_bound(n):
    return n + 2 + (n // (1 << 17) + 1) * 4


@pytest.fixture(scope="module")
def ref():
    L = refs.ref_parity()
    if L is None:
        pytest.skip("oracle/_ref not built")
    return _bind_stream(L)


@pytest.fixture(scope="module")
def shim():
    p = os.path.join(refs.ROOT, "lizard_b200", "libhostshim.so")
    if not os.path.exists(p):
        pytest.skip("libhostshim.so not built")
    L = ctypes.CDLL(p)
    vp, ci = ctypes.c_void_p, ctypes.c_int
    L.lzb_dict_compress.argtypes = [vp, ci, vp, ci, ci, vp, ci, ci]
    L.lzb_emu_lane_order.argtypes = [ci]
    return L


def _layout(dictionary, data, prefix):
    """(keep-alive, dictionary address, input address): one buffer for the prefix layout, two otherwise."""
    if prefix:
        buf = ctypes.create_string_buffer(dictionary + data, len(dictionary) + len(data) + 16)
        return buf, ctypes.addressof(buf), ctypes.addressof(buf) + len(dictionary)
    d = ctypes.create_string_buffer(dictionary, len(dictionary) + 16)
    s = ctypes.create_string_buffer(data, len(data) + 16)
    return (d, s), ctypes.addressof(d), ctypes.addressof(s)


def ref_run(ref, level, dict_p, dict_n, src_p, n, cap):
    out = ctypes.create_string_buffer(max(cap, 1))
    st = ref.Lizard_createStream(level)
    ref.Lizard_loadDict(st, dict_p, dict_n)
    r = ref.Lizard_compress_continue(st, src_p, out, n, cap)
    ref.Lizard_freeStream(st)
    return r, out.raw[:max(r, 0)]


def dev_run(shim, level, dict_p, dict_n, src_p, n, cap, emu):
    out = ctypes.create_string_buffer(max(cap, 1) + 64)
    ctypes.memset(ctypes.addressof(out) + cap, 0xA5, 64)
    r = shim.lzb_dict_compress(src_p, n, out, cap, level, dict_p, dict_n, emu)
    assert out.raw[cap:cap + 64] == b"\xA5" * 64, "wrote behind the capacity"
    return r, out.raw[:max(r, 0)]


def check(ref, shim, level, dictionary, data, prefix, caps=None, orders=(0, 1, 2), emu=1):
    keep, dict_p, src_p = _layout(dictionary, data, prefix)
    bound = lz_bound(len(data))
    want_full = ref_run(ref, level, dict_p, len(dictionary), src_p, len(data), bound)
    caps = caps if caps is not None else [bound]
    for cap in caps:
        want = want_full if cap == bound else ref_run(ref, level, dict_p, len(dictionary), src_p, len(data), cap)
        got = dev_run(shim, level, dict_p, len(dictionary), src_p, len(data), cap, 0)
        assert got == want, ("host", level, prefix, len(dictionary), len(data), cap, got[0], want[0])
        for o in orders:
            shim.lzb_emu_lane_order(o)
            got = dev_run(shim, level, dict_p, len(dictionary), src_p, len(data), cap, emu)
            assert got == want, ("emu", o, level, prefix, len(dictionary), len(data), cap, got[0], want[0])
    shim.lzb_emu_lane_order(0)
    del keep
    return want_full


@pytest.mark.parametrize("level", DICT_LEVELS)
def test_levels_match_reference(ref, shim, level):
    """Every hashChain and priceFast level, both layouts, inputs that lean on the dictionary (one starts with a match running from the
    dictionary's end into the unit); the dictionary must actually shrink the output."""
    d = _dictionary()
    for prefix in (True, False):
        inputs = (_straddler(d, level), records(6000, 100 + level), d[5000:9000] + records(3000, 200 + level) + d[-2000:])
        for k, data in enumerate(inputs):
            r, comp = check(ref, shim, level, d, data, prefix, orders=(0, 1, 2) if k == 0 else (0,))
            assert 0 < r
        r_dict = check(ref, shim, level, d, records(4000, 7), prefix, orders=(0,))[0]
        r_none = check(ref, shim, level, b"", records(4000, 7), prefix, orders=(0,))[0]
        assert r_dict < r_none


@pytest.mark.parametrize("level", [13, 16, 17, 38, 21, 42])
def test_dictionary_sizes(ref, shim, level):
    """Sizes 0, 1-7, 8, 9, 64 KiB and beyond the 64 KiB window; the prefix layout inserts the 7 positions in front of the unit
    (or the whole dictionary below 8 bytes) at hashChain, the external one never does; priceFast inserts no position of the
    dictionary after Lizard_loadDict in either layout."""
    big = records(200_000, 99)
    for size in (0, 1, 2, 5, 7, 8, 9, 15, 1 << 16, 100_000, 200_000):
        d = big[len(big) - size:]
        for prefix in (True, False):
            data = d[-4:] + records(3000, size) + d[:50] if size else records(3000, 1)
            check(ref, shim, level, d, data, prefix, orders=(0, 2) if size < 100_000 else (0,))


@pytest.mark.parametrize("level", [13, 17, 34, 21, 42])
def test_emulated_dictionary_load(ref, shim, level):
    """The dictionary's table and chain built by the 32-lane replay of Lizard_Insert (same-bucket runs inside one 32-position
    step included: the dictionary repeats with short periods) parse exactly as the reference's."""
    d = records(6000, 21) + b"ab" * 600 + b"xyz" * 500 + bytes(700) + records(3000, 22)
    for prefix in (True, False):
        for data in (_straddler(d, level), d[100:2000] + b"ab" * 50 + records(1500, 23) + d[-300:]):
            check(ref, shim, level, d, data, prefix, orders=(0, 2), emu=3)


@pytest.mark.parametrize("level", [21, 22, 41, 42])
def test_price_fast_repeats_and_matches_into_the_dictionary(ref, shim, level):
    """priceFast: matches that start in the dictionary, and repeat offsets into it (a piece of the dictionary with one byte
    changed every 40: each piece after the first is a repeat of the previous match's offset), in both layouts."""
    shim.lzb_dict_enc_stats.argtypes = [ctypes.POINTER(ctypes.c_ulonglong * 2), ctypes.c_int]
    d = _dictionary()
    piece = bytearray(d[20000:26000])
    for k in range(0, len(piece), 40):
        piece[k] ^= 0x55
    data = records(500, 3) + bytes(piece) + records(2000, 4) + d[-300:] + b"#" + d[-200:]
    for prefix in (True, False):
        st = (ctypes.c_ulonglong * 2)()
        shim.lzb_dict_enc_stats(None, 1)
        check(ref, shim, level, d, data, prefix, orders=(0, 2))
        shim.lzb_dict_enc_stats(ctypes.byref(st), 1)
        assert st[0] > 100 and st[1] > 0, (level, prefix, list(st))


@pytest.mark.parametrize("level", [21, 42])
def test_price_fast_window_inside_a_large_dictionary(ref, shim, level):
    """A 5 MiB dictionary against priceFast's 4 MiB window: pieces from its first MiB lie out of reach, pieces from the last
    ones are found."""
    d = records(5 << 20, 31)
    data = d[100_000:103_000] + records(1000, 5) + d[(3 << 20):(3 << 20) + 3000] + d[-5000:-2000]
    for prefix in (True, False):
        check(ref, shim, level, d, data, prefix, orders=())


def test_dictionary_beyond_16_mib(ref, shim):
    """Lizard_loadDict keeps only the last 2^24 bytes of a larger dictionary."""
    tail = records(1 << 16, 5)
    d = bytes(DICT_LIMIT + 1000 - len(tail)) + tail
    data = tail[-3000:] + records(2000, 6)
    for prefix in (True, False):
        check(ref, shim, 17, d, data, prefix, orders=())


@pytest.mark.parametrize("level", [14, 17, 35, 38, 21, 41])
def test_capacities(ref, shim, level):
    """At the bound, the exact size, one byte less and half: same return value and bytes as the reference."""
    d = _dictionary()
    data = _straddler(d, 3) + records(20000, 4)
    for prefix in (True, False):
        keep, dict_p, src_p = _layout(d, data, prefix)
        exact = ref_run(ref, level, dict_p, len(d), src_p, len(data), len(data) + 64)[0]
        del keep
        check(ref, shim, level, d, data, prefix, caps=[len(data) + 64, exact, exact - 1, exact // 2],
              orders=(0,) if level in (14, 35, 41) else ())


@pytest.mark.parametrize("level", [15, 17, 37, 22, 41])
def test_units_of_several_inner_blocks(ref, shim, level):
    """One window across the dictionary and every inner block of a 300 KB unit."""
    d = _dictionary()
    data = records(150_000, 11) + d[1000:40000] + records(120_000, 12)
    for prefix in (True, False):
        check(ref, shim, level, d, data, prefix, orders=(1,) if level in (15, 41) else ())


def test_source_overlapping_its_dictionary(ref, shim):
    """An input that lies inside its (external) dictionary moves lowLimit to the input's end (lib/lizard_compress.c:568-577)."""
    d = _dictionary()
    buf = ctypes.create_string_buffer(d, len(d))
    base = ctypes.addressof(buf)
    for start, n in ((1000, 5000), (40000, 25000), (len(d) - 3000, 2999), (len(d) - 3000, 2997), (0, 60000)):
        for level in (13, 17, 36, 21, 42):
            bound = n + 2 + 4
            want = ref_run(ref, level, base, len(d), base + start, n, bound)
            assert ctypes.string_at(base, len(d)) == d
            for emu in ((0, 1) if level == 13 else (0,)):
                assert dev_run(shim, level, base, len(d), base + start, n, bound, emu) == want, (start, n, level, emu)


def test_other_levels_have_no_dictionary_path(shim):
    """The shim's dictionary entry point runs the hashChain and priceFast parsers only; every other level returns 0."""
    d = _dictionary()
    data = records(3000, 1)
    keep, dict_p, src_p = _layout(d, data, False)
    for level in [lv for lv in range(10, 50) if lv not in DICT_LEVELS]:
        assert dev_run(shim, level, dict_p, len(d), src_p, len(data), 8000, 0)[0] == 0, level
    del keep


DICT_ENCODE_KERNEL = {"REG": 96, "STACK": 608, "SHARED": 17408, "LOCAL": 0}      # (sm_90a, CUDA 12.9)


def test_dictionary_encode_kernel_resources():
    """lizard_encode_dict_kernel: 96 registers at 4 warps per CTA (5 CTAs per SM), the entropy stage's frame, no local memory
    beyond it.  The existing encode instances keep their SASS (tests/test_dict_cpu.py pins the digests)."""
    import re
    import subprocess
    from tests.test_encode_resources_cpu import _cuobjdump
    exe = _cuobjdump()
    if exe is None:
        pytest.skip("cuobjdump not available")
    lib = os.path.join(refs.ROOT, "lizard_b200", "liblizard_b200.so")
    out = subprocess.run([exe, "-res-usage", lib], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, check=True).stdout
    res, name = None, None
    for line in out.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            name = m.group(1)
        elif name and "lizard_encode_dict_kernel" in name and "REG:" in line:
            res = {k: int(v) for k, v in re.findall(r"(REG|STACK|LOCAL|SHARED):(\d+)", line)}
            name = None
    assert res == DICT_ENCODE_KERNEL, res


# ---- the dictionary corpus (tests/corpus.py dict_corpus) ----------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _dict_corpus():
    return corpus.dict_corpus()


@functools.lru_cache(maxsize=None)
def _ref_dict_streams(level):
    L = refs.ref_parity()
    _bind_stream(L)
    out = []
    for c in _dict_corpus():
        keep, dict_p, src_p = _layout(c.dictionary, c.unit, c.prefix)
        out.append(ref_run(L, level, dict_p, len(c.dictionary), src_p, len(c.unit), lz_bound(len(c.unit)))[1])
        del keep
    return out


@pytest.mark.parametrize("level", corpus.DICT_WALKED_LEVELS)
def test_walker_decodes_reference_dictionary_streams(ref, level):
    """The walker, given the dictionary, decodes the reference's dictionary streams to the input; without it, a stream that
    reaches into the dictionary is refused."""
    refused = 0
    for c, comp in zip(_dict_corpus(), _ref_dict_streams(level)):
        out, classes = corpus.walk(comp, dictionary=c.dictionary)
        assert out == c.unit, (level, c)
        if classes["dict_match"] + classes["dict_straddle"]:
            with pytest.raises(ValueError):
                corpus.walk(comp)
            refused += 1
    assert refused > 10, level


def test_reference_dictionary_streams_reach_every_target(ref):
    """Case by case, the reference's streams hold what each family is built for (corpus.dict_shortfalls: a coded block, the
    straddle of exactly its length, the three 24-byte matches of a poisoned unit, the window's last offset at both window
    sizes, ...), and all of them together every class of corpus.dict_targets()."""
    walked = {level: [corpus.walk(comp, dictionary=c.dictionary)[1] for c, comp in zip(_dict_corpus(), _ref_dict_streams(level))]
              for level in corpus.DICT_WALKED_LEVELS}
    short = corpus.dict_shortfalls(_dict_corpus(), walked)
    short += [(level, i) for level, per_case in walked.items() for i, (c, classes) in enumerate(zip(_dict_corpus(), per_case))
              if c.family == "poisoned" and not corpus.poisoned_parse_ok(classes)]
    assert not short, short[:10]
    seen = Counter()
    for per_case in walked.values():
        for classes in per_case:
            seen.update(classes)
    assert not [t for t in corpus.dict_targets() if seen[t] == 0], dict(seen)


@pytest.mark.parametrize("level", corpus.DICT_WALKED_LEVELS)
def test_poisoned_surroundings_change_the_reference_output(ref, level):
    """The bytes a poisoned case puts around its dictionary matter: the reference given them as part of the dictionary (what
    a kernel reading past the dictionary's end, or extending below its start, would see) writes a different stream.  So a
    device call that writes the reference's bytes with those surroundings in place did not read them."""
    for c in _dict_corpus():
        if c.family != "poisoned":
            continue
        want = _ref_stream(ref, level, c.dictionary, c.unit, c.prefix)
        assert _ref_stream(ref, level, c.before_dict + c.dictionary, c.unit, c.prefix) != want, (level, c, "before")
        if c.after_dict:
            assert _ref_stream(ref, level, c.dictionary + c.after_dict, c.unit, False) != want, (level, c, "after")


def _ref_stream(ref, level, dictionary, unit, prefix):
    keep, dict_p, src_p = _layout(dictionary, unit, prefix)
    r = ref_run(ref, level, dict_p, len(dictionary), src_p, len(unit), lz_bound(len(unit)))
    del keep
    return r


def _emulated(cases, level):
    """What the coroutine emulator (slow) runs: every case but the corpus family's, whose first two it runs cut to 20000
    bytes; at the hashChain levels (the slowest under the emulator) the first two cases of each family, cut to 20000."""
    out, seen = [], Counter()
    for c in cases:
        if c.family == "corpus" or level in HC_LEVELS:
            if seen[c.family] < 2:
                out.append((c, c.unit[:20000]))
            seen[c.family] += 1
        else:
            out.append((c, c.unit))
    return out


@pytest.mark.parametrize("level", DICT_LEVELS)
def test_dict_families_one_lane_and_emulated_bit_exact(ref, shim, level):
    """Every family of the dictionary corpus through the one-lane host build at every level with a dictionary path, at the
    bound and at an edge capacity, and the emulator in lane order 0 (_emulated): the reference's bytes and return value."""
    rnd = random.Random(700 + level)
    cases = _dict_corpus()
    caps = corpus.edge_capacities(rnd, [c.unit for c in cases], lz_bound)
    for c, cap in zip(cases, caps):
        check(ref, shim, level, c.dictionary, c.unit, c.prefix, caps=[lz_bound(len(c.unit)), cap], orders=())
    for c, unit in _emulated(cases, level):
        check(ref, shim, level, c.dictionary, unit, c.prefix, orders=(0,))
