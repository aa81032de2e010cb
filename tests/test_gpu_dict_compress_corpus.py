"""GPU parity of compression against a dictionary off the easy path: the dictionary corpus (tests/corpus.py dict_corpus) with
edge capacities through LizardB200_compress_dict_batch and the device call at every residue mod 16, poisoned bytes around
external dictionaries and units, the codeword classes of the GPU's dictionary streams, units that share a dictionary slot
(prefix and external users, equal ends or sizes, tiny and trimmed dictionaries, many warps waiting on slow loads), the slot
bound in both calls, inputs that overlap or touch their dictionary, the workspace shared by launches on two streams, and the
round trip through the GPU's and the reference's dictionary decoders.  Every check compares with the reference built with
-DLIZARD_RESET_MEM (Lizard_createStream + Lizard_loadDict + Lizard_compress_continue) at the same addresses, bytes and
return value."""
import contextlib
import ctypes
import functools
import random
import re
from collections import Counter, defaultdict

import numpy as np
import pytest

import lizard_b200 as lz
from tests import corpus, refs

pytestmark = pytest.mark.gpu
LEVELS = corpus.DICT_ENCODE_LEVELS
DICT_LIMIT = 1 << 24
GUARD = 0xEE
ERR_MEMORY = -1005                                          # LIZARDB200_ERR_MEMORY


def bound(n):
    return n + 2 + (n // (1 << 17) + 1) * 4


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
    return L


def ref_run(ref, level, dict_p, dict_n, src_p, n, cap):
    out = ctypes.create_string_buffer(max(cap, 1))
    st = ref.Lizard_createStream(level)
    ref.Lizard_loadDict(st, dict_p, dict_n)
    r = ref.Lizard_compress_continue(st, src_p, out, n, cap)
    ref.Lizard_freeStream(st)
    return r, out.raw[:max(r, 0)]


class Arena:
    """Bytes laid out once for the host (a ctypes buffer: the reference and the batch call read it at these addresses) and
    once on the device (the device call reads the same offsets).  Filler is random, so no constant byte hides a read
    outside the dictionary or the unit."""

    def __init__(self, seed):
        self.rng = np.random.default_rng(seed)
        self.h = bytearray()

    def fill(self, n):
        self.h += self.rng.integers(0, 256, n, dtype=np.uint8).tobytes()

    def put(self, body, residue=None, before=b""):
        """Append `before` and `body` so that body starts at `residue` mod 16; returns body's offset."""
        if residue is not None:
            self.fill((residue - len(self.h) - len(before)) % 16)
        self.h += before
        at = len(self.h)
        self.h += body
        return at

    def seal(self):
        self.fill(64)
        self.host = ctypes.create_string_buffer(bytes(self.h), len(self.h))
        self.base = ctypes.addressof(self.host)
        return self

    def device(self):
        import torch
        return torch.frombuffer(bytearray(self.h), dtype=torch.uint8).to("cuda:0")


class Units:
    """Per unit: source offset and size, dictionary offset and size, in one Arena."""

    def __init__(self):
        self.so, self.sl, self.do, self.dl = [], [], [], []

    def add(self, so, sl, do, dl):
        self.so.append(so); self.sl.append(sl); self.do.append(do); self.dl.append(dl)

    def __len__(self):
        return len(self.so)

    def want(self, ref, arena, level, caps):
        b = arena.base
        return [ref_run(ref, level, b + self.do[i], self.dl[i], b + self.so[i], self.sl[i], caps[i]) for i in range(len(self))]


def place_cases(arena, cases, salt):
    """The DictCase list in an Arena: every dictionary and unit at its own residue mod 16, a prefix dictionary right in front
    of its unit, a poisoned case's chosen bytes around them."""
    us = Units()
    for i, c in enumerate(cases):
        rd, ru = (3 * i + salt) % 16, (5 * i + 7 + salt) % 16
        if c.prefix:
            do = arena.put(c.dictionary + c.unit, rd, c.before_dict)
            us.add(do + len(c.dictionary), len(c.unit), do, len(c.dictionary))
        else:
            do = arena.put(c.dictionary, rd, c.before_dict)
            arena.h += c.after_dict
            arena.fill(40)
            so = arena.put(c.unit, ru, c.before_unit)
            us.add(so, len(c.unit), do, len(c.dictionary))
        arena.fill(9)
    return us


def device_call(arena, us, caps, level, d_arena=None, stream=None, keep=None):
    """LizardB200_compress_dict_device over the arena with every destination at its own residue mod 16 between GUARD
    bytes; returns (status, results, destination bytes, destination offsets) after a sync (or the tensors if keep is a
    list: no sync then)."""
    import torch
    dev = torch.device("cuda", 0)
    d_arena = arena.device() if d_arena is None else d_arena
    dst_off, at = [], 64
    for i, c in enumerate(caps):
        at += (7 * i + 1 - at) % 16
        dst_off.append(at)
        at += c + 64
    t = lambda v, dt: torch.tensor(v, dtype=dt, device=dev)
    with torch.cuda.stream(stream) if stream is not None else contextlib.nullcontext():
        # made on the launch's stream, so the fills and copies are ordered before the kernel that reads and writes them
        d_dst = torch.full((at + 64,), GUARD, dtype=torch.uint8, device=dev)
        t_so, t_sl, t_do, t_dc = t(us.so, torch.int64), t(us.sl, torch.int32), t(dst_off, torch.int64), t(caps, torch.int32)
        t_dd, t_dl = t(us.do, torch.int64), t(us.dl, torch.int32)
        t_res = torch.full((len(us),), -7, dtype=torch.int32, device=dev)
    st = lz.lib().LizardB200_compress_dict_device(d_arena.data_ptr(), t_so.data_ptr(), t_sl.data_ptr(), d_dst.data_ptr(),
                                                  t_do.data_ptr(), t_dc.data_ptr(), d_arena.data_ptr(), t_dd.data_ptr(),
                                                  t_dl.data_ptr(), t_res.data_ptr(), len(us), level,
                                                  None if stream is None else ctypes.c_void_p(stream.cuda_stream))
    if keep is not None:
        keep.append((d_arena, t_so, t_sl, t_do, t_dc, t_dd, t_dl))
        return st, t_res, d_dst, dst_off
    torch.cuda.synchronize()
    return st, t_res.cpu().tolist(), d_dst.cpu().numpy().tobytes(), dst_off


def check_device(res, out, dst_off, caps, want, what):
    """Results and bytes are the reference's; nothing outside [dst, dst + cap) of a unit changed."""
    bad = [(i, r, w[0]) for i, (r, w) in enumerate(zip(res, want)) if r != w[0] or out[dst_off[i]:dst_off[i] + max(r, 0)] != w[1]]
    assert not bad, (what, len(bad), bad[:8])
    outside = bytearray(out)
    for o, c in zip(dst_off, caps):
        outside[o:o + c] = bytes([GUARD]) * c
    assert outside == bytes([GUARD]) * len(out), (what, "wrote outside a unit's destination")


def batch_call(arena, us, caps, level):
    """LizardB200_compress_dict_batch on host pointers into the arena: the staging must keep every unit's placement
    relative to its dictionary.  Returns (status, [(result, bytes)])."""
    n, b = len(us), arena.base
    dsts = [ctypes.create_string_buffer(max(c, 1)) for c in caps]
    res = (ctypes.c_int * n)()
    st = lz.lib().LizardB200_compress_dict_batch(
        (ctypes.c_void_p * n)(*[b + o for o in us.so]), (ctypes.c_int * n)(*us.sl),
        (ctypes.c_void_p * n)(*[ctypes.addressof(x) for x in dsts]), (ctypes.c_int * n)(*caps),
        (ctypes.c_void_p * n)(*[b + o if l else None for o, l in zip(us.do, us.dl)]), (ctypes.c_int * n)(*us.dl), res, n, level)
    return st, [(res[i], dsts[i].raw[:max(res[i], 0)]) for i in range(n)]


def check_batch(out, want, what):
    bad = [(i, r, w[0]) for i, ((r, o), w) in enumerate(zip(out, want)) if r != w[0] or o != w[1]]
    assert not bad, (what, len(bad), bad[:8])


# ---------------------------------------------------------------------------------------------------------------------
# 1-3, 8: the corpus (poisoned cases included), the codeword classes, the round trip
# ---------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _cases():
    return corpus.dict_corpus()


@functools.lru_cache(maxsize=None)
def _corpus_arena(level):
    arena = Arena(level)
    us = place_cases(arena, _cases(), level)
    return arena.seal(), us


@functools.lru_cache(maxsize=None)
def _bound_run(ref, level):
    """The device call at the bound (its streams are walked and decoded) and the reference's streams."""
    arena, us = _corpus_arena(level)
    caps = [bound(n) for n in us.sl]
    return caps, us.want(ref, arena, level, caps), device_call(arena, us, caps, level)


@pytest.mark.parametrize("level", LEVELS)
def test_corpus_with_edge_capacities_in_both_calls(ref, level):
    """Every case of the dictionary corpus, both layouts: the batch call and the device call (each with its own edge
    capacities) and the device call at the bound write the reference's bytes.  The poisoned cases' surroundings only
    exist in the device call, where the bytes around the dictionary and the unit are part of the buffer."""
    arena, us = _corpus_arena(level)
    units = [c.unit for c in _cases()]
    for k, call in enumerate(("batch", "device")):
        caps = corpus.edge_capacities(random.Random(1000 * k + level), units, bound)
        want = us.want(ref, arena, level, caps)
        if call == "batch":
            st, out = batch_call(arena, us, caps, level)
            assert st == 0, lz.lib().LizardB200_lastError()
            check_batch(out, want, (level, call))
        else:
            st, res, out, dst_off = device_call(arena, us, caps, level)
            assert st == 0, lz.lib().LizardB200_lastError()
            check_device(res, out, dst_off, caps, want, (level, call))
    caps, want, (st, res, out, dst_off) = _bound_run(ref, level)
    assert st == 0
    check_device(res, out, dst_off, caps, want, (level, "bound"))


def test_gpu_streams_reach_the_dictionary_targets(ref):
    """Walked with their dictionaries, the GPU's streams at 13-17, 21 and 22 decode to the input and hold, case by case, what
    each family is built for (corpus.dict_shortfalls); every poisoned unit's stream at every level holds its three
    dictionary matches of 23-24 bytes and none longer; together they reach every class of corpus.dict_targets().  The
    Huffman twins are checked by bytes (test above)."""
    seen, walked, poisoned = Counter(), {}, []
    for level in corpus.DICT_WALKED_LEVELS:
        caps, want, (st, res, out, dst_off) = _bound_run(ref, level)
        walked[level] = []
        for i, c in enumerate(_cases()):
            comp = out[dst_off[i]:dst_off[i] + res[i]]
            assert res[i] == want[i][0] and comp == want[i][1], (level, i, c)
            back, classes = corpus.walk(comp, dictionary=c.dictionary)
            assert back == c.unit, (level, i, c)
            walked[level].append(classes)
            seen.update(classes)
            if c.family == "poisoned" and not corpus.poisoned_parse_ok(classes):
                poisoned.append((level, i))
    short = corpus.dict_shortfalls(_cases(), walked)
    assert not short and not poisoned, (short[:10], poisoned)
    assert not [t for t in corpus.dict_targets() if seen[t] == 0], dict((t, seen[t]) for t in corpus.dict_targets())


@pytest.mark.parametrize("level", [13, 17, 21, 22, 34, 38, 41, 42])
def test_round_trip_through_both_decoders(ref, level):
    """The GPU's streams read back to the input through decompress_dict_batch, LizardB200_decompress_dict_device (against
    the arena's dictionaries in place on the device) and the reference's Lizard_decompress_safe_usingDict."""
    import torch
    arena, us = _corpus_arena(level)
    caps, want, (st, res, out, dst_off) = _bound_run(ref, level)
    cases = _cases()
    comp = [out[o:o + r] for o, r in zip(dst_off, res)]
    assert all(r > 0 for r in res), level
    back = lz.decompress_dict_batch(comp, [c.dictionary for c in cases], [len(c.unit) for c in cases])
    for i, (c, (r, o)) in enumerate(zip(cases, back)):
        assert r == len(c.unit) and o == c.unit, (level, "batch", i, c)
        dst = ctypes.create_string_buffer(len(c.unit) + 64)
        r = ref.Lizard_decompress_safe_usingDict(comp[i], dst, len(comp[i]), len(c.unit), arena.base + us.do[i], us.dl[i])
        assert r == len(c.unit) and dst.raw[:r] == c.unit, (level, "reference", i, c)
    dev = torch.device("cuda", 0)
    t = lambda v, dt: torch.tensor(v, dtype=dt, device=dev)
    c_off = list(np.cumsum([0] + [len(x) for x in comp[:-1]]))
    d_comp = torch.frombuffer(bytearray(b"".join(comp) + bytes(64)), dtype=torch.uint8).to(dev)
    o_off = list(np.cumsum([0] + [len(c.unit) + 64 for c in cases[:-1]]))
    d_out = torch.zeros(sum(len(c.unit) + 64 for c in cases), dtype=torch.uint8, device=dev)
    d_arena = arena.device()
    t_res = torch.zeros(len(cases), dtype=torch.int32, device=dev)
    # every table a named tensor: a temporary's memory would go back to the allocator before the launch reads it
    t_co, t_cl = t(c_off, torch.int64), t([len(x) for x in comp], torch.int32)
    t_oo, t_oc = t(o_off, torch.int64), t(us.sl, torch.int32)
    t_do, t_dl = t(us.do, torch.int64), t(us.dl, torch.int32)
    st = lz.lib().LizardB200_decompress_dict_device(d_comp.data_ptr(), t_co.data_ptr(), t_cl.data_ptr(), d_out.data_ptr(),
                                                    t_oo.data_ptr(), t_oc.data_ptr(), d_arena.data_ptr(), t_do.data_ptr(),
                                                    t_dl.data_ptr(), t_res.data_ptr(), len(cases), None)
    assert st == 0, lz.lib().LizardB200_lastError()
    torch.cuda.synchronize()
    r_dev, o_dev = t_res.cpu().tolist(), d_out.cpu().numpy().tobytes()
    for i, c in enumerate(cases):
        assert r_dev[i] == len(c.unit) and o_dev[o_off[i]:o_off[i] + r_dev[i]] == c.unit, (level, "device", i, c)


# ---------------------------------------------------------------------------------------------------------------------
# 4: units that share a slot in one device call
# ---------------------------------------------------------------------------------------------------------------------
def _pieces(rng, buf, end, n, reach):
    """n bytes: pieces of buf from the `reach` bytes before `end`, between fresh bytes."""
    out = bytearray()
    while len(out) < n:
        k = int(rng.integers(20, 400))
        at = end - int(rng.integers(k + 1, reach))
        out += buf[max(at, 0):max(at, 0) + k] + rng.integers(0, 256, int(rng.integers(1, 60)), dtype=np.uint8).tobytes()
    return bytes(out[:n])


def _slot_sharing_layout(seed):
    """One arena: a buffer R of 17 MiB + 128 KiB whose windows are the dictionaries, units that reach into them, in both
    layouts (a prefix unit is the part of R right behind its window)."""
    rng = np.random.default_rng(seed)
    top = (17 << 20) + (128 << 10)
    R = rng.integers(0, 256, top, dtype=np.uint8)
    R[: 1 << 20] = np.tile(rng.integers(0, 256, 4099, dtype=np.uint8), (1 << 20) // 4099 + 1)[: 1 << 20]
    R = R.tobytes()
    arena = Arena(seed)
    r0 = arena.put(R, 0)
    arena.fill(100)
    us = Units()
    names = []

    def external(end, size, n, name, reps=1):
        for _ in range(reps):
            u = _pieces(rng, R, end, n, max(min(size, 60000), 1000))
            us.add(arena.put(u, int(rng.integers(16))), n, r0 + end - size, size)
            names.append(name)
            arena.fill(int(rng.integers(1, 50)))

    def prefix(end, size, n, name):
        us.add(r0 + end, n, r0 + end - size, size)
        names.append(name)

    E = 17 << 20
    e1 = 3 << 20                                            # the same (end, size): a prefix unit and external units
    prefix(e1, 50000, 3000, "same key, prefix")
    external(e1, 50000, 4000, "same key, external", reps=3)
    e2 = 5 << 20                                            # the same end, different sizes
    for s in (8, 9, 100, 5000, 65535, 65536, 70000, 1 << 20):
        external(e2, s, 3000, "same end %d" % s)
    prefix(e2, 5000, 2000, "same end, prefix")
    for k in range(6):                                      # the same size, different ends
        external((6 << 20) + 777 * k, 30000, 2500, "same size %d" % k)
    for k in range(16):                                     # tiny dictionaries at many addresses
        t, e = k % 9, (7 << 20) + 1013 * k
        (prefix if k % 3 == 0 else external)(e, t, 1500, "tiny %d" % t)
    for j, s in enumerate((DICT_LIMIT - 1, DICT_LIMIT, DICT_LIMIT + 1, E)):   # over 2^24 with one end: one key after the trim
        external(E, s, 5000, "large %d" % s)
        end = E - 4096 * (j + 1)
        prefix(end, min(s, end), 3000, "large prefix %d" % s)
    for k in range(40):                                     # many warps wait on slow loads
        size = (1 << 20) + k * ((16 << 20) // 40)
        end = min(E, size + 4096 * k)
        external(end, size, 2000, "big %d" % k, reps=3)
    return arena.seal(), us, names


@pytest.mark.parametrize("level", [17, 41])
def test_slot_sharing_in_one_device_call(ref, level):
    """Units that share a slot or only seem to (same end, same size, tiny dictionaries, windows over 2^24 bytes trimmed to
    one key, a prefix unit beside external users of its dictionary) and 40 large dictionaries of 1-17 MiB each used by
    three consecutive units, so warps wait on loads: one device call, the reference's bytes for every unit."""
    arena, us, names = _slot_sharing_layout(level)
    caps = [bound(n) for n in us.sl]
    want = us.want(ref, arena, level, caps)
    st, res, out, dst_off = device_call(arena, us, caps, level)
    assert st == 0, lz.lib().LizardB200_lastError()
    bad = [(names[i], res[i], want[i][0]) for i in range(len(us)) if res[i] != want[i][0]
           or out[dst_off[i]:dst_off[i] + max(res[i], 0)] != want[i][1]]
    assert not bad, (level, len(bad), bad[:8])
    check_device(res, out, dst_off, caps, want, level)
    assert all(r > 0 for r in res)


# ---------------------------------------------------------------------------------------------------------------------
# 5: the slot bound
# ---------------------------------------------------------------------------------------------------------------------
N_BOUND = 5000
BOUND_LEVEL = 13


@functools.lru_cache(maxsize=None)
def _bound_buffer():
    rng = np.random.default_rng(5)
    return ctypes.create_string_buffer(rng.integers(0, 256, 2 << 20, dtype=np.uint8).tobytes(), 2 << 20)   # every _window


def _bound_batch(dict_of_unit):
    """N_BOUND units of 40 bytes at the bound, unit i against the window dict_of_unit(i) = (offset, size) of one buffer."""
    buf = _bound_buffer()
    b = ctypes.addressof(buf)
    n = N_BOUND
    units = [b + 3000 * (i % 120) + 17 for i in range(n)]                # below every dictionary window
    ds = [dict_of_unit(i) for i in range(n)]
    dsts = ctypes.create_string_buffer(64 * n)
    res = (ctypes.c_int * n)()
    st = lz.lib().LizardB200_compress_dict_batch(
        (ctypes.c_void_p * n)(*units), (ctypes.c_int * n)(*[40] * n),
        (ctypes.c_void_p * n)(*[ctypes.addressof(dsts) + 64 * i for i in range(n)]), (ctypes.c_int * n)(*[bound(40)] * n),
        (ctypes.c_void_p * n)(*[b + o if s else None for o, s in ds]), (ctypes.c_int * n)(*[s for _, s in ds]), res, n,
        BOUND_LEVEL)
    return st, units, ds, list(res), dsts


def _window(k):
    """Distinct key k: a window of 8 to 2055 bytes ending at its own address."""
    return 400000 + 131 * k, 8 + (k * 37) % 2048


@functools.lru_cache(maxsize=None)
def _slots():
    st, *_ = _bound_batch(_window)
    assert st == ERR_MEMORY, st
    m = re.search(r"(\d+) distinct dictionaries .* holds (\d+) for (\d+) units", lz.lib().LizardB200_lastError().decode())
    assert m and int(m.group(1)) == N_BOUND and int(m.group(3)) == N_BOUND, lz.lib().LizardB200_lastError()
    return int(m.group(2)), st


def test_batch_call_at_the_slot_bound(ref):
    """S distinct dictionaries (S read from the refusal of a call with N_BOUND of them) and S - 1 plus tiny ones are
    accepted and give the reference's bytes; S + 1, and S plus one tiny dictionary, are refused."""
    S, err = _slots()
    assert 0 < S < N_BOUND
    tiny = lambda i: (500000 + 7 * i, i % 8)
    for name, f, ok in (("S", lambda i: _window(i % S), True),
                        ("S - 1 + tiny", lambda i: _window(i) if i < S - 1 else tiny(i), True),
                        ("S + 1", lambda i: _window(i % (S + 1)), False),
                        ("S + tiny", lambda i: _window(i) if i < S else tiny(i), False)):
        st, units, ds, res, dsts = _bound_batch(f)
        if not ok:
            assert st == err, (name, st)
            continue
        assert st == 0, (name, lz.lib().LizardB200_lastError())
        b = ctypes.addressof(_bound_buffer())
        for i in range(0, N_BOUND, 7):
            want = ref_run(ref, BOUND_LEVEL, b + ds[i][0], ds[i][1], units[i], 40, bound(40))
            assert res[i] == want[0] and dsts.raw[64 * i:64 * i + res[i]] == want[1], (name, i)


def test_device_call_beyond_the_slot_bound(ref):
    """K = S + 117 distinct keys over N_BOUND units in one device call: exactly S keys get a slot, every unit of a key has
    the same outcome, a success is the reference's bytes, a failure is -1 with its destination untouched."""
    S, _ = _slots()
    K = S + 117
    arena = Arena(11)
    buf = arena.put(_bound_buffer().raw, 0)
    us = Units()
    for i in range(N_BOUND):
        o, s = _window(i % K)
        us.add(buf + 3000 * (i % 120) + 17, 40, buf + o, s)
    arena.seal()
    caps = [bound(40)] * N_BOUND
    st, res, out, dst_off = device_call(arena, us, caps, BOUND_LEVEL)
    assert st == 0, lz.lib().LizardB200_lastError()
    by_key = defaultdict(set)
    for i, r in enumerate(res):
        by_key[i % K].add(r > 0)
    assert all(len(v) == 1 for v in by_key.values()), [k for k, v in by_key.items() if len(v) > 1][:8]
    assert sum(1 for v in by_key.values() if True in v) == S
    want = [ref_run(ref, BOUND_LEVEL, arena.base + us.do[i], us.dl[i], arena.base + us.so[i], 40, caps[i]) if r > 0
            else (-1, b"") for i, r in enumerate(res)]
    assert all(r == -1 for r in res if r <= 0)
    assert all(set(out[o:o + c]) == {GUARD} for o, c, r in zip(dst_off, caps, res) if r < 0)
    check_device(res, out, dst_off, caps, want, "beyond the bound")


# ---------------------------------------------------------------------------------------------------------------------
# 6: inputs that overlap or touch their dictionary
# ---------------------------------------------------------------------------------------------------------------------
def _overlap_layout():
    """A buffer of records and, behind them, random bytes to 2^24 + 100000; unit and dictionary windows of it."""
    from tests.test_dict_cpu import records
    rec = records(200000, 77)
    rng = np.random.default_rng(12)
    rest = rng.integers(0, 256, DICT_LIMIT + 100000 - len(rec), dtype=np.uint8).tobytes()
    arena = Arena(13)
    b = arena.put(rec + rest, 0)
    ext = arena.put(rec[120000:126000] + rec[2000:9000], 5)
    arena.seal()
    us, names = Units(), []
    d0, d1 = 20000, 90000                                   # the dictionary [d0, d1)

    def add(name, so, n, do=d0, dl=d1 - d0, base=b):
        us.add(base + so, n, b + do, dl)
        names.append(name)

    add("inside", 30000, 20000)
    add("inside at the end", d1 - 3000, 3000)
    add("starts before, ends inside", d0 - 5000, 25000)
    add("contains", d0 - 1000, d1 - d0 + 2000)
    add("ends at the start", d0 - 6000, 6000)
    add("starts at the end (prefix)", d1, 6000)
    for k in (3, 4, 5):
        add("dictLimit - lowLimit = %d" % k, d1 - 4000, 4000 - k)
    add("external", 0, 13000, base=ext)
    add("external 2", 6000, 7000, base=ext)
    big = DICT_LIMIT + 60000                                # trimmed to [60000, 60000 + 2^24)
    add("in the trimmed part", 30000, 20000, 0, big)
    add("touches the trimmed start", 50000, 10000, 0, big)
    add("straddles the trimmed start", 55000, 20000, 0, big)
    add("prefix of a trimmed dictionary", big, 8000, 0, big)
    return arena, us, names


@pytest.mark.parametrize("level", [13, 17, 36, 22, 41])
def test_overlapping_and_touching_layouts_in_both_calls(ref, level):
    """Inputs inside, around, before and behind their dictionary, lowLimit 3-5 bytes below dictLimit, inputs in the part of
    a dictionary over 2^24 bytes that Lizard_loadDict drops, and external users of the same dictionary, in one batch call
    (which stages an overlapping unit together with its dictionary) and one device call: the reference's bytes."""
    arena, us, names = _overlap_layout()
    caps = [bound(n) for n in us.sl]
    want = us.want(ref, arena, level, caps)
    st, out = batch_call(arena, us, caps, level)
    assert st == 0, lz.lib().LizardB200_lastError()
    bad = [(names[i], r, want[i][0]) for i, (r, o) in enumerate(out) if r != want[i][0] or o != want[i][1]]
    assert not bad, (level, "batch", bad)
    st, res, dout, dst_off = device_call(arena, us, caps, level)
    assert st == 0, lz.lib().LizardB200_lastError()
    bad = [(names[i], r, want[i][0]) for i, r in enumerate(res) if r != want[i][0]]
    assert not bad, (level, "device", bad)
    check_device(res, dout, dst_off, caps, want, (level, "device"))


# ---------------------------------------------------------------------------------------------------------------------
# 7: the workspace across launches
# ---------------------------------------------------------------------------------------------------------------------
def test_workspace_across_launches_on_two_streams(ref):
    """Without a host sync: dictionary launches at 22, 21 (hashLog 18, then 14), 17 and 41 on the same dictionary addresses
    and two streams; the dictionary rewritten by copy_ on the stream between two launches at 17 (the second must load the
    new bytes into a fresh slot); plain launches at 19 (optimal) and 24 (lowestPrice) in between."""
    import torch
    from tests.test_dict_cpu import records
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(21)
    d_old, d_new = records(60000, 31), records(60000, 32)
    units = [(d_old if i % 2 else d_new)[(97 * i) % 50000:][:2000] + records(1500 + 13 * i, 400 + i) for i in range(300)]
    arena = Arena(22)
    do = arena.put(d_old, 3)
    so = [arena.put(u, int(rng.integers(16))) for u in units]
    arena.seal()
    us = Units()
    for o, u in zip(so, units):
        us.add(o, len(u), do, len(d_old))
    d_arena = arena.device()
    new_bytes = torch.frombuffer(bytearray(d_new), dtype=torch.uint8).to(dev)
    caps = [bound(len(u)) for u in units]
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    L = lz.lib()
    keep, runs = [], []
    plan = [("dict", s1, 22), ("dict", s2, 21), ("plain", s1, 19), ("dict", s2, 17), ("plain", s2, 24), ("dict", s1, 41),
            ("dict", s1, 17), ("rewrite", s1, None), ("dict", s1, 17), ("plain", s2, 19), ("dict", s2, 22)]
    t = lambda v, dt: torch.tensor(v, dtype=dt, device=dev)
    rewritten = False
    for kind, s, level in plan:
        if kind == "rewrite":
            with torch.cuda.stream(s):
                d_arena[do:do + len(d_new)].copy_(new_bytes)
            rewritten = True
            continue
        if kind == "dict":
            st, t_res, d_dst, dst_off = device_call(arena, us, caps, level, d_arena, s, keep)
        else:
            dst_off = [64 * ((sum(caps[:i]) + 63) // 64 + i) for i in range(len(units))]
            with torch.cuda.stream(s):                  # ordered before the launch on s
                d_dst = torch.full((dst_off[-1] + caps[-1] + 64,), GUARD, dtype=torch.uint8, device=dev)
                t_res = torch.zeros(len(units), dtype=torch.int32, device=dev)
                t_so, t_sl = t(so, torch.int64), t(us.sl, torch.int32)
                t_do, t_dc = t(dst_off, torch.int64), t(caps, torch.int32)
            keep.append((t_so, t_sl, t_do, t_dc))
            st = L.LizardB200_compress_device(d_arena.data_ptr(), t_so.data_ptr(), t_sl.data_ptr(), d_dst.data_ptr(),
                                              t_do.data_ptr(), t_dc.data_ptr(), t_res.data_ptr(), len(units), level,
                                              ctypes.c_void_p(s.cuda_stream))
        assert st == 0, (kind, level, L.LizardB200_lastError())
        runs.append((kind, level, rewritten, t_res, d_dst, dst_off))
    torch.cuda.synchronize()
    h_new = ctypes.create_string_buffer(d_new, len(d_new) + 16)
    for kind, level, rewritten, t_res, d_dst, dst_off in runs:
        res, out = t_res.cpu().tolist(), d_dst.cpu().numpy().tobytes()
        if kind == "dict":
            dp = ctypes.addressof(h_new) if rewritten else arena.base + do
            want = [ref_run(ref, level, dp, len(d_old), arena.base + o, len(u), c) for o, u, c in zip(so, units, caps)]
            check_device(res, out, dst_off, caps, want, (kind, level, rewritten))
        else:
            for i, (u, c) in enumerate(zip(units, caps)):
                w = refs.ref_compress(ref, u, level, c)
                assert res[i] == len(w) and out[dst_off[i]:dst_off[i] + res[i]] == w, (kind, level, i)
