"""Dictionary decoding on the H100 at its edges: reach edges through the batch and device calls, the 2^24 switches of the
reference's in-place and external modes, units that share one dictionary end in a batch (the staging of run_host_batch),
damaged units by the thousand, in-place device calls at every residue mod 16 next to a live dictionary, the streaming
decoder's windows with both an external part and a prefix, and the decode instances on two CUDA streams.  The yardstick is
the reference built with -DLIZARD_RESET_MEM: Lizard_decompress_safe_usingDict and Lizard_decompress_safe_continue at the
same layouts, return codes always, bytes where it succeeds (every stream here obeys the min-offset rule unless damaged;
damaged units compare return codes only)."""
import ctypes
import functools
import random

import numpy as np
import pytest

import lizard_b200 as lz
from tests import corpus, refs
from tests.test_dict_cpu import (PREFIX_MAX, _damage, _dictionary, _level_inputs, _linked_stream, _long_offset_unit,
                                 _shortest_dictionary, records, ref_compress_dict, ref_decode_dict)
from tests.test_gpu_corpus import _decode_variant
from tests.test_partial_cpu import ref_partial

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
GUARD = 0xEE


@pytest.fixture(scope="module")
def ref():
    L = refs.ref_parity()
    if L is None:
        pytest.skip("oracle/_ref not built")
    vp, ci = ctypes.c_void_p, ctypes.c_int
    L.Lizard_createStream.restype = vp
    L.Lizard_createStream.argtypes = [ci]
    L.Lizard_freeStream.argtypes = [vp]
    L.Lizard_loadDict.argtypes = [vp, vp, ci]
    L.Lizard_compress_continue.argtypes = [vp, vp, vp, ci, ci]
    L.Lizard_decompress_safe_usingDict.argtypes = [vp, vp, ci, ci, vp, ci]
    L.Lizard_createStreamDecode.restype = vp
    L.Lizard_freeStreamDecode.argtypes = [vp]
    L.Lizard_setStreamDecode.argtypes = [vp, vp, ci]
    L.Lizard_decompress_safe_continue.argtypes = [vp, vp, vp, ci, ci]
    L.Lizard_decompress_safe_partial.argtypes = [ctypes.c_char_p, ctypes.c_char_p, ci, ci, ci]
    return L


@pytest.fixture(scope="module")
def gpu():
    if not torch.cuda.is_available() or not lz.lib().LizardB200_available():
        pytest.skip("no usable CUDA device")
    return lz.lib()


# ---- host batches ----------------------------------------------------------------------------------------------------
class HostUnits:
    """Units of one LizardB200_decompress_dict_batch call on host buffers.  add() lays a unit's dictionary directly in front
    of its output (prefix) or in a buffer of its own, unless the caller gives the dictionary's address (a shared one)."""

    def __init__(self):
        self.rows, self.held, self.want = [], [], []

    def add(self, comp, cap, dictionary, prefix, want, dict_addr=None, dst=None):
        if dst is None:
            if prefix:
                buf = ctypes.create_string_buffer(dictionary + bytes(cap + 64), len(dictionary) + cap + 64)
                dict_addr, dst = ctypes.addressof(buf), ctypes.addressof(buf) + len(dictionary)
            else:
                buf = ctypes.create_string_buffer(cap + 64)
                dst = ctypes.addressof(buf)
                if dict_addr is None:
                    dbuf = ctypes.create_string_buffer(dictionary, max(len(dictionary), 1))
                    self.held.append(dbuf)
                    dict_addr = ctypes.addressof(dbuf)
            self.held.append(buf)
        self.rows.append((comp, dst, cap, dict_addr, len(dictionary)))
        self.want.append(want)

    def run(self, L, order=None):
        """One call; returns (results, outputs, launches).  order: the unit order of the call (results come back in add order)."""
        order = list(range(len(self.rows))) if order is None else order
        n = len(order)
        src, csz, dst, cap = (ctypes.c_void_p * n)(), (ctypes.c_int * n)(), (ctypes.c_void_p * n)(), (ctypes.c_int * n)()
        dp, ds, res = (ctypes.c_void_p * n)(), (ctypes.c_int * n)(), (ctypes.c_int * n)()
        keep = []
        for j, i in enumerate(order):
            comp, d, c, da, dsz = self.rows[i]
            sb = ctypes.create_string_buffer(comp, max(len(comp), 1))
            keep.append(sb)
            src[j], csz[j], dst[j], cap[j], dp[j], ds[j] = ctypes.addressof(sb), len(comp), d, c, da, dsz
        before = L.LizardB200_launchCount()
        assert L.LizardB200_decompress_dict_batch(src, csz, dst, cap, dp, ds, res, n) == 0, L.LizardB200_lastError()
        launches = L.LizardB200_launchCount() - before
        results = [0] * n
        for j, i in enumerate(order):
            results[i] = res[j]
        outs = [ctypes.string_at(self.rows[i][1], max(results[i], 0)) for i in range(n)]
        return results, outs, launches


def _compare(want, results, outs, caps, what, bytes_too=True):
    """want: the reference's (result, bytes) per unit.  The DESIGN.md 3.5 raw-block overrun: the reference reports more
    than the capacity, the device refuses."""
    bad = []
    for i, ((rr, ro), r, o, cap) in enumerate(zip(want, results, outs, caps)):
        if rr > cap:
            if r >= 0:
                bad.append((i, r, rr, "accepted an overrun"))
        elif r != rr:
            bad.append((i, r, rr))
        elif bytes_too and rr > 0 and o[:rr] != ro:
            bad.append((i, "content"))
    assert not bad, (what, len(bad), bad[:10])


# ---- device calls ----------------------------------------------------------------------------------------------------
def device_call(L, units, dst_residue):
    """LizardB200_decompress_dict_device over one arena that holds every dictionary and output between GUARD bytes.
    units: (comp, cap, dictionary, prefix); prefix lays the dictionary directly in front of the output, otherwise it sits
    elsewhere in the arena (one copy per distinct bytes object).  Returns (results, arena before, arena after, out offsets,
    dict offsets)."""
    dev = torch.device("cuda", 0)
    arena = bytearray(b"\xEE" * 48)
    shared, d_off, o_off = {}, [], []
    for i, (comp, cap, d, prefix) in enumerate(units):
        if not prefix and id(d) not in shared:
            arena += b"\xEE" * (16 + (i % 16))
            shared[id(d)] = len(arena)
            arena += d + b"\xEE" * 16
    for i, (comp, cap, d, prefix) in enumerate(units):
        arena += b"\xEE" * (((dst_residue(i) - len(arena) - (len(d) if prefix else 0)) % 16) + 16)
        if prefix:
            d_off.append(len(arena))
            arena += d
        else:
            d_off.append(shared[id(d)])
        o_off.append(len(arena))
        arena += b"\xEE" * (cap + 24)
    src = b"".join(c for c, _, _, _ in units) + bytes(64)
    s_off = list(np.cumsum([0] + [len(c) for c, _, _, _ in units[:-1]]))
    t = lambda v, dt: torch.tensor(v, dtype=dt, device=dev)
    g_src = torch.frombuffer(bytearray(src), dtype=torch.uint8).to(dev)
    g_arena = torch.frombuffer(bytearray(arena), dtype=torch.uint8).to(dev)
    t_so, t_sl = t(s_off, torch.int64), t([len(c) for c, _, _, _ in units], torch.int32)
    t_oo, t_oc = t(o_off, torch.int64), t([c for _, c, _, _ in units], torch.int32)
    t_do, t_dl = t(d_off, torch.int64), t([len(d) for _, _, d, _ in units], torch.int32)
    t_res = torch.zeros(len(units), dtype=torch.int32, device=dev)
    st = L.LizardB200_decompress_dict_device(g_src.data_ptr(), t_so.data_ptr(), t_sl.data_ptr(), g_arena.data_ptr(),
                                             t_oo.data_ptr(), t_oc.data_ptr(), g_arena.data_ptr(), t_do.data_ptr(),
                                             t_dl.data_ptr(), t_res.data_ptr(), len(units), None)
    assert st == 0, L.LizardB200_lastError()
    torch.cuda.synchronize()
    return t_res.cpu().tolist(), bytes(arena), g_arena.cpu().numpy().tobytes(), o_off, d_off


def _check_device(want, units, res, before, after, o_off, what, bytes_too=True):
    """The reference's results (and bytes), and the arena unchanged outside [dst, dst + result) of the units that succeed
    and outside [dst, dst + capacity) of the others: dictionaries and guard bytes included."""
    caps = [c for _, c, _, _ in units]
    _compare(want, res, [after[o:o + max(r, 0)] for o, r in zip(o_off, res)], caps, what, bytes_too)
    expect = bytearray(before)
    got = bytearray(after)
    for o, c, r in zip(o_off, caps, res):
        if r > 0:
            expect[o:o + r] = got[o:o + r]
        else:
            got[o:o + c] = expect[o:o + c]
    assert got == expect, (what, "wrote outside a unit's output")


# ---------------------------------------------------------------------------------------------------------------------
# D1: reach edges
# ---------------------------------------------------------------------------------------------------------------------
REACH_LEVELS = [13, 17, 20, 21, 35, 41, 45]


def test_reach_edges_in_both_calls(ref, gpu):
    """test_dict_cpu.py::test_reach_edges on the GPU: the dictionary shortened from its front to `need`, need - 1, need / 2
    and 1 bytes, in place and external, at levels 13-45.  All 56 units in one batch under variant 7 (the Huffman pre-pass
    runs ahead of the dictionary kernel: 3 launches) and variant 3 (1 launch), then in one device call.  The reference's
    results and bytes; a dictionary one byte short gives its token error -(index)-1, not -1."""
    L = gpu
    d = _dictionary()
    units, want, short = [], [], []
    for level in REACH_LEVELS:
        data = _level_inputs(level)[2]
        for prefix in (True, False):
            comp = ref_compress_dict(ref, d, data, level, prefix)
            need = _shortest_dictionary(ref, comp, d, len(data), prefix)
            assert 0 < need <= len(d), need
            for k in (need, need - 1, need // 2, 1):
                w = ref_decode_dict(ref, comp, d[len(d) - k:], len(data), prefix)
                if k >= need:
                    assert w == (len(data), data)
                else:
                    assert w[0] < -1, (level, prefix, k, need, w[0])
                    short.append(len(units))
                units.append((comp, len(data), d[len(d) - k:], prefix))
                want.append(w)
    hu = HostUnits()
    for (comp, cap, dd, prefix), w in zip(units, want):
        hu.add(comp, cap, dd, prefix, w)
    for variant, launches in ((7, 3), (3, 1)):
        with _decode_variant(variant):
            res, outs, n = hu.run(L)
        assert n == launches, (variant, n)
        _compare(want, res, outs, [u[1] for u in units], ("batch", variant))
    res, before, after, o_off, _ = device_call(L, units, lambda i: (5 * i + 3) % 16)
    _check_device(want, units, res, before, after, o_off, "device")
    assert all(res[i] < -1 for i in short)


# ---------------------------------------------------------------------------------------------------------------------
# D2: the 2^24 switches
# ---------------------------------------------------------------------------------------------------------------------
SWITCH_SIZES = ((1 << 24) - 2, PREFIX_MAX, 1 << 24, (1 << 24) + 5)


def test_the_2_24_switches(ref, gpu):
    """An offset of 2^24 - 1 at the unit start, and behind a token of 3 literals and an 8-byte match, against dictionaries of
    2^24 - 2 .. 2^24 + 5 bytes in place and external: through Lizard_decompress_safe_usingDict (the batch stages only the
    last 2^24 - 1 bytes) and through the device call (the dictionary on the device directly in front of the output, or
    elsewhere).  Plus a fastLZ4 unit against a 2^17-byte dictionary whose farthest match starts at the edge of the 64 KiB
    window, so that only the dictionary's last 65535 bytes are staged."""
    L = gpu
    big = bytes(random.Random(7).getrandbits(8) for _ in range(1 << 12)) * ((1 << 24) // (1 << 12) + 1)
    streams = [_long_offset_unit(20, PREFIX_MAX), _long_offset_unit(20, PREFIX_MAX, lead=3)]
    dicts = [big[:size] for size in SWITCH_SIZES]
    units, want, seen = [], [], set()
    for comp, n in streams:
        for d in dicts:
            size = len(d)
            for prefix in (True, False):
                w = ref_decode_dict(ref, comp, d, n + 16, prefix)
                seen.add(w[0] > 0)
                got = lz.decompress_using_dict(comp, d, n + 16, prefix)
                assert got == w, (len(comp), size, prefix, got[0], w[0])
                units.append((comp, n + 16, d, prefix))
                want.append(w)
    assert seen == {True, False}
    # the farthest match of a fastLZ4 unit is 65535 back: a dictionary of 2^17 bytes is read at its last 65535 only
    d17 = _dictionary(1 << 17)
    data = d17[-65535:-65535 + 3000] + records(3000, 17) + d17[-2000:]
    for prefix in (True, False):
        comp = ref_compress_dict(ref, d17, data, 17, prefix)
        need = _shortest_dictionary(ref, comp, d17, len(data), prefix)
        assert 65500 < need <= 65535, need
        w = ref_decode_dict(ref, comp, d17, len(data), prefix)
        assert w == (len(data), data)
        assert lz.decompress_using_dict(comp, d17, len(data), prefix) == w
        units.append((comp, len(data), d17, prefix))
        want.append(w)
    res, before, after, o_off, _ = device_call(L, units, lambda i: (3 * i + 1) % 16)
    _check_device(want, units, res, before, after, o_off, "device")


# ---------------------------------------------------------------------------------------------------------------------
# D3: units that share a dictionary end in one batch call
# ---------------------------------------------------------------------------------------------------------------------
def _pieces_of(d, seed, far):
    """A unit of pieces of `d`: one from `far` bytes before its end, one from its last 2 KiB, fresh records between."""
    at = len(d) - far
    return d[at:at + 1500] + records(2500, seed) + d[-2000:] + records(500, seed + 1)


def test_units_sharing_one_dictionary_end(ref, gpu):
    """One batch call whose units use one 1 MiB buffer every way at once: an in-place prefix for one unit and an external
    dictionary for others with the same end; views shortened from the front (same end, smaller size and reach, some below
    the unit's need); views shortened from the back (other ends); fastLZ4 and LIZv1 units on one end (staged 65535 and
    2^24 - 1 bytes); dictSize 0 and -1; a level byte out of range.  Every unit gives the result and bytes of the reference
    called on it alone (dictSize -1 gives -1, include/lizard_b200.h); the same in the reverse unit order."""
    L = gpu
    M = 1 << 20
    B = records(M, 4242)
    cap_max = 12000
    hold = ctypes.create_string_buffer(B + bytes(cap_max + 64), M + cap_max + 64)
    base = ctypes.addressof(hold)
    hu = HostUnits()
    add = lambda comp, cap, d, prefix, dict_addr, dst=None: hu.add(comp, cap, d, prefix,
                                                                   ref_decode_dict(ref, comp, d, cap, prefix)
                                                                   if len(d) else ref_decode_dict(ref, comp, b"", cap, False),
                                                                   dict_addr, dst)
    # fastLZ4 first: its window (65535) is the smallest a unit stages from this end
    for i, level in enumerate((17, 13, 35)):
        data = _pieces_of(B, 10 + i, 60000)
        add(ref_compress_dict(ref, B, data, level, False), len(data), B, False, base)
    data = _pieces_of(B, 20, 900000)
    add(ref_compress_dict(ref, B, data, 21, True), len(data), B, True, base, base + M)          # in place, same end
    for i, level in enumerate((21, 41, 20, 45)):
        data = _pieces_of(B, 30 + i, 700000 + 50000 * i)
        comp = ref_compress_dict(ref, B, data, level, False)
        add(comp, len(data), B, False, base)
        need = _shortest_dictionary(ref, comp, B, len(data), False)
        assert need > 65535, (level, need)
        for k in (need, need - 1, need // 2, 70000):                                            # shortened from the front
            add(comp, len(data), B[M - k:], False, base + M - k)
    for j in (1, 4096, 500000):                                                               # shortened from the back
        dj = B[:M - j]
        for level in (21, 17):
            data = _pieces_of(dj, 40 + j % 7, 60000 if level == 17 else 400000)
            add(ref_compress_dict(ref, dj, data, level, False), len(data), dj, False, base)
    plain = records(5000, 5)
    add(refs.ref_compress(ref, plain, 41), len(plain), b"", False, base)                        # dictSize 0
    comp = bytearray(ref_compress_dict(ref, B, _pieces_of(B, 50, 80000), 21, False))
    comp[0] = 50                                                                               # no such level
    add(bytes(comp), 9000, B, False, base)
    negative = len(hu.rows)
    hu.add(ref_compress_dict(ref, B, plain, 21, False), len(plain), B, False, (-1, b""), base)
    hu.rows[negative] = hu.rows[negative][:4] + (-1,)
    assert sum(1 for w in hu.want if w[0] < 0) >= 8 and sum(1 for w in hu.want if w[0] > 0) >= 15, [w[0] for w in hu.want]
    caps = [r[2] for r in hu.rows]
    assert len(hu.rows) >= 32
    for order in (None, list(range(len(hu.rows)))[::-1]):
        res, outs, launches = hu.run(L, order)
        assert launches == 3                                    # the Huffman pre-pass and the dictionary kernel
        _compare(hu.want, res, outs, caps, "forward" if order is None else "reversed")
        assert ctypes.string_at(base, M) == B


# ---------------------------------------------------------------------------------------------------------------------
# D4: damaged dictionary units
# ---------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _dict_cases():
    return [c for c in corpus.dict_corpus() if c.family in ("straddle", "poisoned")]


def _damaged_units(ref, level, rnd):
    """About 1000 (comp, cap, dictionary, prefix): truncations and flips of the straddler and record units (their first
    token is the dictionary match, so damage falls in front of and behind it), and of the straddle and poisoned cases of
    corpus.dict_corpus()."""
    d = _dictionary()
    base = [(ref_compress_dict(ref, d, data, level, prefix), len(data), d, prefix)
            for prefix in (True, False) for data in _level_inputs(level)[:2]]
    base += [(ref_compress_dict(ref, c.dictionary, c.unit, level, c.prefix), len(c.unit), c.dictionary, c.prefix)
             for c in _dict_cases()[::2]]
    out = []
    while len(out) < 1000:
        for comp, n, dd, prefix in base:
            bad = comp[:rnd.choice([1, 2, len(comp) // 3, len(comp) - 1])] if rnd.random() < 0.25 else _damage(rnd, comp)
            out.append((bad, n, dd, prefix))
    return out


@pytest.mark.parametrize("level", [10, 20, 21, 30, 41])
def test_damaged_units_by_the_thousand(ref, gpu, level):
    """test_dict_cpu.py::test_damaged_streams at scale: about 1000 damaged units per call, through the batch under variants
    3 and 7 and through the device call.  Return codes equal the reference's (bytes are not compared: damage can make
    offsets below 8, DESIGN.md 3.5), and the device call writes nothing outside a unit's output."""
    L = gpu
    units = _damaged_units(ref, level, random.Random(500 + level))
    want = [ref_decode_dict(ref, comp, d, n, prefix) for comp, n, d, prefix in units]
    assert sum(1 for w in want if w[0] < 0) > 100 and sum(1 for w in want if w[0] > 0) > 10
    hu = HostUnits()
    for (comp, n, d, prefix), w in zip(units, want):
        hu.add(comp, n, d, prefix, w)
    for variant in (3, 7):
        with _decode_variant(variant):
            res, outs, _ = hu.run(L)
        _compare(want, res, outs, [u[1] for u in units], (level, variant), bytes_too=False)
    res, before, after, o_off, _ = device_call(L, units, lambda i: (11 * i + 5) % 16)
    _check_device(want, units, res, before, after, o_off, (level, "device"), bytes_too=False)


# ---------------------------------------------------------------------------------------------------------------------
# D5: in-place device calls at every alignment
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("level", [10, 21, 41, 45])
def test_in_place_device_calls_at_every_alignment(ref, gpu, level):
    """The straddle cases of corpus.dict_corpus() (one per codeword threshold length), each dictionary directly in front of
    its output, at every residue mod 16 of the output, guard bytes in front of the dictionary and behind the output: the
    input as result and bytes, and the dictionary and every byte outside [dst, dst + result) unchanged (the pooled sweeps
    store destination-aligned 16 bytes at a time next to a live dictionary)."""
    L = gpu
    cases = [c for c in _dict_cases() if c.family == "straddle"]
    comps = [ref_compress_dict(ref, c.dictionary, c.unit, level, c.prefix) for c in cases]
    units, want = [], []
    for residue in range(16):
        for c, comp in zip(cases, comps):
            units.append((comp, len(c.unit), c.dictionary, True))
            want.append((len(c.unit), c.unit))
    for (comp, n, d, _), w in zip(units[:len(cases)], want):
        assert ref_decode_dict(ref, comp, d, n, True) == w
    res, before, after, o_off, _ = device_call(L, units, lambda i: i // len(cases))
    assert sorted({o % 16 for o in o_off}) == list(range(16))
    _check_device(want, units, res, before, after, o_off, level)


# ---------------------------------------------------------------------------------------------------------------------
# D6: the streaming decoder's windows
# ---------------------------------------------------------------------------------------------------------------------
def _walk(L, size, steps, init=b""):
    """Lizard_setStreamDecode / Lizard_decompress_safe_continue of library L over a buffer of `size` bytes that starts with
    `init`: steps are ("set", offset, size) and ("dec", comp, capacity, offset).  Returns every decode's (result, bytes)."""
    buf = ctypes.create_string_buffer(init, size)
    base = ctypes.addressof(buf)
    sd = L.Lizard_createStreamDecode()
    L.Lizard_setStreamDecode(sd, None, 0)
    out = []
    for step in steps:
        if step[0] == "set":
            L.Lizard_setStreamDecode(sd, base + step[1], step[2])
        else:
            _, comp, cap, at = step
            r = L.Lizard_decompress_safe_continue(sd, comp, base + at, len(comp), cap)
            out.append((r, ctypes.string_at(base + at, max(r, 0))))
    L.Lizard_freeStreamDecode(sd)
    return out


def _windows(steps, results):
    """(external part, prefix) of the window of every decode, as the reference's state machine sets them
    (lib/lizard_decompress.c:322-344)."""
    pre_end, pre_size, ext_size, parts = None, 0, 0, []
    it = iter(results)
    for step in steps:
        if step[0] == "set":
            pre_end, pre_size, ext_size = step[1] + step[2], step[2], 0
            continue
        r = next(it)[0]
        at = step[3]
        if pre_end == at:
            parts.append((ext_size, pre_size))
            if r > 0:
                pre_size += r
                pre_end += r
        else:
            ext_size = pre_size
            parts.append((ext_size, 0))
            if r > 0:
                pre_size, pre_end = r, at + r
    return parts


def _compare_walks(ref, gpu, size, steps, what, init=b"", damaged=None):
    """Both libraries walk the same steps: the same result at every decode, and the same bytes, except at and behind a
    damaged decode (index `damaged`) that the reference accepts: its bytes may come from offsets below 8 (DESIGN.md 3.5)."""
    want = _walk(ref, size, steps, init)
    got = _walk(gpu, size, steps, init)
    rc_only = damaged is not None and want[damaged][0] >= 0
    bad = [(k, g[0], w[0]) for k, (g, w) in enumerate(zip(got, want))
           if g[0] != w[0] or (g[1] != w[1] and not (rc_only and k >= damaged))]
    assert not bad, (what, len(bad), bad[:10])
    return want


def _placed(ref, data, level, piece, offset_of, size):
    """_linked_stream with piece k written at offset_of(k) of a buffer of `size` bytes, as the decoder will place it."""
    buf = ctypes.create_string_buffer(size)
    return _linked_stream(ref, data, level, piece, False, place=lambda k: ctypes.addressof(buf) + offset_of(k))


@pytest.mark.parametrize("level", [10, 21, 41])
def test_continue_with_an_external_part_and_a_prefix(ref, gpu, level):
    """Two buffers of three 16 KiB pieces each, filled in turn: the second and third piece of every buffer decode against a
    window of the other buffer (external part) and the pieces in front of them (prefix), both non-empty; the fastLZ4 window
    (65535 bytes) then takes only the tail of the external part.  A damaged piece in the middle gives the reference's error
    and leaves the state as it was: the intact piece fed next decodes as in the reference."""
    piece, per = 16 << 10, 3
    data = records(piece * per * 4, 700 + level)
    off = lambda k: ((k // per) % 2) * (piece * per + 4096) + (k % per) * piece
    size = 2 * (piece * per + 4096)
    pieces = _placed(ref, data, level, piece, off, size)
    steps = [("dec", comp, n_in, off(k)) for k, (comp, n_in) in enumerate(pieces)]
    want = _compare_walks(ref, gpu, size, steps, level)
    assert b"".join(o for _, o in want) == data
    parts = _windows(steps, want)
    both = [k for k, (e, p) in enumerate(parts) if e > 0 and p > 0]
    assert both == [k for k in range(len(pieces)) if k >= per and k % per], parts
    # a damaged piece in the middle (second piece of a buffer), then the intact one into the same place
    k = per + 1
    rnd = random.Random(level)
    comp = pieces[k][0]
    for j, bad in enumerate((comp[:len(comp) // 2], _damage(rnd, comp), _damage(rnd, comp))):
        damaged = steps[:k] + [("dec", bad, pieces[k][1], off(k))] + steps[k:]
        want = _compare_walks(ref, gpu, size, damaged, (level, "damaged", j), damaged=k)
        assert want[k][0] < 0 or j > 0, want[k][0]
        if want[k][0] < 0:                                      # the state is as it was: the rest decodes the input
            assert b"".join(o for _, o in want[:k] + want[k + 1:]) == data


@pytest.mark.parametrize("level,ring,piece", [(10, 48 << 10, 8 << 10), (30, 48 << 10, 8 << 10), (21, 3 << 19, 1 << 18)])
def test_continue_through_a_ring_buffer(ref, gpu, level, ring, piece):
    """A ring buffer that wraps two and a half times: after a wrap, the piece at the ring's start decodes against the whole
    ring as its external part, and the pieces behind it against what remains of it plus their own prefix."""
    count = 5 * ring // piece // 2
    data = records(count * piece, 800 + level) if ring < (1 << 20) else lz.datagen(count * piece, 50, level)
    off = lambda k: (k * piece) % ring
    pieces = _placed(ref, data, level, piece, off, ring)
    steps = [("dec", comp, n_in, off(k)) for k, (comp, n_in) in enumerate(pieces)]
    want = _compare_walks(ref, gpu, ring, steps, level)
    assert b"".join(o for _, o in want) == data
    assert any(e > 0 and p > 0 for e, p in _windows(steps, want))


@pytest.mark.parametrize("level", [21, 41])
def test_continue_past_2_24(ref, gpu, level):
    """20 MiB decoded contiguously in 1 MiB pieces: the window grows past 2^24 bytes (the offset check goes off) and is
    gathered at its last 2^24 - 1."""
    piece = 1 << 20
    data = lz.datagen(20 * piece, 50, level)
    pieces = _linked_stream(ref, data, level, piece, False)
    steps = [("dec", comp, n_in, k * piece) for k, (comp, n_in) in enumerate(pieces)]
    want = _compare_walks(ref, gpu, len(data) + 64, steps, level)
    assert b"".join(o for _, o in want) == data
    assert max(p for _, p in _windows(steps, want)) > 1 << 24


@pytest.mark.parametrize("level", [10, 21, 41])
def test_continue_behind_a_set_window(ref, gpu, level):
    """Lizard_setStreamDecode to a saved copy of 16 KiB, then two pieces decoded contiguously behind it: prefix mode on a
    window the caller set."""
    saved = records(16 << 10, 60 + level)
    data = records(16 << 10, 61 + level)
    buf = ctypes.create_string_buffer(saved, len(saved) + len(data) + 64)
    base = ctypes.addressof(buf)
    pieces = _linked_stream(ref, data, level, 8 << 10, False, place=lambda k: base + len(saved) + k * (8 << 10),
                            load=(base, len(saved)))
    steps = [("set", 0, len(saved))] + [("dec", comp, n_in, len(saved) + k * (8 << 10)) for k, (comp, n_in) in enumerate(pieces)]
    want = _compare_walks(ref, gpu, len(saved) + len(data) + 64, steps, level, init=saved)
    assert b"".join(o for _, o in want) == data
    assert _windows(steps, want) == [(0, len(saved)), (0, len(saved) + (8 << 10))]


# ---------------------------------------------------------------------------------------------------------------------
# D7: the decode instances on two streams
# ---------------------------------------------------------------------------------------------------------------------
def test_decode_instances_across_two_streams(ref, gpu):
    """Without a host sync: dictionary, partial and plain decode device calls and one LizardB200_compress_device call
    interleaved on two torch.cuda.Streams, each launch's tensors made on its own stream.  The dictionary of stream 1 is
    rewritten on stream 1 between two of its dictionary launches.  Every result is the reference's for the bytes in place at
    its launch: the workspace (decode scratch, pre-pass buffers, counter ring) is handed from stream to stream."""
    L = gpu
    dev = torch.device("cuda", 0)
    d_old, d_new, d_two = records(60000, 71), records(60000, 72), records(60000, 73)
    dict_units = {}
    for name, d in (("one", d_old), ("two", d_two)):
        for level in (17, 21, 41):
            datas = [_pieces_of(d, 100 * level + i, 50000) for i in range(64)]
            dict_units[(name, level)] = [(ref_compress_dict(ref, d, x, level, False), len(x)) for x in datas]
    plain = [lz.datagen(9000 + 37 * i, 50, i) for i in range(256)]
    plain_comp = [refs.ref_compress(ref, u, 41) for u in plain]
    targets = [random.Random(i).randrange(-1, len(u) + 2) for i, u in enumerate(plain)]
    d_arena = torch.frombuffer(bytearray(d_old + bytes(64) + d_two), dtype=torch.uint8).to(dev)
    at = {"one": 0, "two": len(d_old) + 64}
    new_bytes = torch.frombuffer(bytearray(d_new), dtype=torch.uint8).to(dev)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    t = lambda v, dt: torch.tensor(v, dtype=dt, device=dev)
    keep, runs, rewritten = [], [], False

    def dict_launch(s, name, level):
        units = dict_units[(name, level)]
        with torch.cuda.stream(s):
            g_src = torch.frombuffer(bytearray(b"".join(c for c, _ in units)), dtype=torch.uint8).to(dev)
            s_off = list(np.cumsum([0] + [len(c) for c, _ in units[:-1]]))
            o_off = list(np.cumsum([0] + [n + 64 for _, n in units[:-1]]))
            g_out = torch.full((o_off[-1] + units[-1][1] + 64,), GUARD, dtype=torch.uint8, device=dev)
            tabs = (t(s_off, torch.int64), t([len(c) for c, _ in units], torch.int32), t(o_off, torch.int64),
                    t([n for _, n in units], torch.int32), t([at[name]] * len(units), torch.int64),
                    t([len(d_old)] * len(units), torch.int32))
            t_res = torch.zeros(len(units), dtype=torch.int32, device=dev)
        keep.append((g_src, tabs))
        st = L.LizardB200_decompress_dict_device(g_src.data_ptr(), tabs[0].data_ptr(), tabs[1].data_ptr(), g_out.data_ptr(),
                                                 tabs[2].data_ptr(), tabs[3].data_ptr(), d_arena.data_ptr(), tabs[4].data_ptr(),
                                                 tabs[5].data_ptr(), t_res.data_ptr(), len(units), ctypes.c_void_p(s.cuda_stream))
        assert st == 0, L.LizardB200_lastError()
        d = d_new if (name == "one" and rewritten) else {"one": d_old, "two": d_two}[name]
        runs.append((("dict", name, level, rewritten), [(c, n, d) for c, n in units], t_res, g_out, o_off))

    def plain_launch(s, kind):
        units = plain_comp if kind != "compress" else plain
        caps = [len(u) for u in plain] if kind != "compress" else [lz.compress_bound(len(u)) for u in plain]
        with torch.cuda.stream(s):
            g_src = torch.frombuffer(bytearray(b"".join(units)), dtype=torch.uint8).to(dev)
            s_off = list(np.cumsum([0] + [len(c) for c in units[:-1]]))
            o_off = list(np.cumsum([0] + [c + 64 for c in caps[:-1]]))
            g_out = torch.full((o_off[-1] + caps[-1] + 64,), GUARD, dtype=torch.uint8, device=dev)
            tabs = (t(s_off, torch.int64), t([len(c) for c in units], torch.int32), t(o_off, torch.int64), t(caps, torch.int32),
                    t(targets, torch.int32))
            t_res = torch.zeros(len(units), dtype=torch.int32, device=dev)
        keep.append((g_src, tabs))
        a = (g_src.data_ptr(), tabs[0].data_ptr(), tabs[1].data_ptr(), g_out.data_ptr(), tabs[2].data_ptr(), tabs[3].data_ptr())
        if kind == "partial":
            st = L.LizardB200_decompress_partial_device(*a, tabs[4].data_ptr(), t_res.data_ptr(), len(units),
                                                        ctypes.c_void_p(s.cuda_stream))
        elif kind == "plain":
            st = L.LizardB200_decompress_device(*a, t_res.data_ptr(), len(units), ctypes.c_void_p(s.cuda_stream))
        else:
            st = L.LizardB200_compress_device(*a, t_res.data_ptr(), len(units), 10, ctypes.c_void_p(s.cuda_stream))
        assert st == 0, L.LizardB200_lastError()
        runs.append(((kind,), None, t_res, g_out, o_off))

    plan = [(dict_launch, s1, "one", 21), (plain_launch, s2, "partial"), (dict_launch, s2, "two", 41),
            (plain_launch, s1, "plain"), (dict_launch, s1, "one", 41), (plain_launch, s2, "compress"),
            (dict_launch, s2, "two", 17), (dict_launch, s1, "one", 17), ("rewrite",), (dict_launch, s1, "one", 17),
            (plain_launch, s2, "partial"), (dict_launch, s2, "two", 21), (dict_launch, s1, "one", 21),
            (plain_launch, s1, "plain")]
    for step in plan:
        if step[0] == "rewrite":
            with torch.cuda.stream(s1):
                d_arena[:len(d_new)].copy_(new_bytes)
            rewritten = True
        else:
            step[0](*step[1:])
    torch.cuda.synchronize()
    for what, units, t_res, g_out, o_off in runs:
        res, out = t_res.cpu().tolist(), g_out.cpu().numpy().tobytes()
        got = [(r, out[o:o + max(r, 0)]) for r, o in zip(res, o_off)]
        if what[0] == "dict":
            want = [ref_decode_dict(ref, c, d, n, False) for c, n, d in units]
            assert what[3] or all(w[0] > 0 for w in want)
        elif what[0] == "partial":
            want = [ref_partial(ref, c, tg, len(u)) for c, tg, u in zip(plain_comp, targets, plain)]
        elif what[0] == "plain":
            want = [(len(u), u) for u in plain]
        else:
            want = [(len(c), c) for c in (refs.ref_compress(ref, u, 10) for u in plain)]
        bad = [i for i, (g, w) in enumerate(zip(got, want)) if g[0] != w[0] or (w[0] > 0 and g[1] != w[1])]
        assert not bad, (what, len(bad), bad[:10])

