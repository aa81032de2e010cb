"""GPU parity of compression against a dictionary (hashChain levels 13-17, 34-38, priceFast levels 21, 22, 41, 42): Lizard_loadDict + Lizard_compress_continue,
LizardB200_compress_dict_batch and LizardB200_compress_dict_device write the bytes of the reference built with
-DLIZARD_RESET_MEM (Lizard_createStream + Lizard_loadDict + Lizard_compress_continue at the same addresses), and the GPU's
dictionary decoder reads them back."""
import ctypes

import numpy as np
import pytest

import lizard_b200 as lz
from tests import refs
from tests.test_dict_cpu import _dictionary, _straddler, records

pytestmark = pytest.mark.gpu
DICT_LEVELS = list(range(13, 18)) + list(range(34, 39)) + [21, 22, 41, 42]


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
    return L


def ref_run(ref, level, dict_p, dict_n, src_p, n, cap):
    out = ctypes.create_string_buffer(max(cap, 1))
    st = ref.Lizard_createStream(level)
    ref.Lizard_loadDict(st, dict_p, dict_n)
    r = ref.Lizard_compress_continue(st, src_p, out, n, cap)
    ref.Lizard_freeStream(st)
    return out.raw[:max(r, 0)]


def ref_using_dict(ref, data, d, level, cap=None, prefix=False):
    cap = len(data) + 2 + (len(data) // (1 << 17) + 1) * 4 if cap is None else cap
    if prefix:
        buf = ctypes.create_string_buffer(d + data, len(d) + len(data) + 1)
        return ref_run(ref, level, ctypes.addressof(buf), len(d), ctypes.addressof(buf) + len(d), len(data), cap)
    db = ctypes.create_string_buffer(d, len(d) + 1)
    sb = ctypes.create_string_buffer(data, len(data) + 1)
    return ref_run(ref, level, ctypes.addressof(db), len(d), ctypes.addressof(sb), len(data), cap)


@pytest.mark.parametrize("level", DICT_LEVELS)
def test_drop_in_pair(ref, level):
    """Lizard_loadDict + Lizard_compress_continue in both layouts, dictionary sizes 0 to beyond the window, capacities at the
    exact size and one byte less."""
    big = records(150_000, 77)
    for size in (0, 5, 8, 1 << 16, 150_000):
        d = big[len(big) - size:]
        for prefix in (False, True):
            for data in (_straddler(d, level) if size >= 40 else records(2000, 1), records(9000, level) + d[:3000]):
                want = ref_using_dict(ref, data, d, level, prefix=prefix)
                assert lz.compress_using_dict(data, d, level, prefix=prefix) == want, (level, size, prefix, len(data))
                assert lz.compress_using_dict(data, d, level, len(want), prefix) == want
                short = ref_using_dict(ref, data, d, level, len(want) - 1, prefix)
                assert lz.compress_using_dict(data, d, level, len(want) - 1, prefix) == short


def test_stream_rules(ref):
    """A fresh or reset stream's _continue is Lizard_compress at every GPU level; a later _continue and Lizard_saveDict return 0;
    Lizard_loadDict returns the reference's value; the fast, lowestPrice and optimal parsers have no dictionary path and return
    0 after Lizard_loadDict."""
    L = lz.lib()
    data = records(20000, 3)
    d = _dictionary()
    out = ctypes.create_string_buffer(30000)
    for level in (10, 17, 21, 25, 41):
        st = L.Lizard_createStream(level)
        n = L.Lizard_compress_continue(st, data, out, len(data), 30000)
        assert out.raw[:n] == refs.ref_compress(ref, data, level, 30000), level
        assert L.Lizard_compress_continue(st, data, out, len(data), 30000) == 0
        L.Lizard_resetStream.restype = ctypes.c_void_p
        L.Lizard_resetStream.argtypes = [ctypes.c_void_p, ctypes.c_int]
        st = L.Lizard_resetStream(st, level)
        n = L.Lizard_compress_continue(st, data, out, len(data), 30000)
        assert n > 0 and out.raw[:n] == refs.ref_compress(ref, data, level, 30000), level
        L.Lizard_freeStream(st)
    db = ctypes.create_string_buffer(d, len(d))
    for level in (17, 41, 10, 19, 25):
        st = L.Lizard_createStream(level)
        assert L.Lizard_loadDict(st, db, len(d)) == len(d)
        n = L.Lizard_compress_continue(st, data, out, len(data), 30000)
        if level in (17, 41):
            assert out.raw[:n] == ref_using_dict(ref, data, d, level, 30000)
            assert L.Lizard_compress_continue(st, data, out, len(data), 30000) == 0
        else:
            assert n == 0, level
        assert L.Lizard_saveDict(st, out, 1000) == 0
        L.Lizard_freeStream(st)
    huge = ctypes.create_string_buffer((1 << 24) + 100)
    st = L.Lizard_createStream(17)
    assert L.Lizard_loadDict(st, huge, (1 << 24) + 100) == 1 << 24
    L.Lizard_freeStream(st)
    for level in (10, 25, 19):
        with pytest.raises(lz.LizardB200Error, match="priceFast parsers"):
            lz.compress_dict_batch([data], [d], level)


def _batch_raw(units, dict_ptrs, dict_sizes, src_ptrs, caps, level):
    n = len(units)
    dsts = [ctypes.create_string_buffer(max(c, 1)) for c in caps]
    res = (ctypes.c_int * n)()
    st = lz.lib().LizardB200_compress_dict_batch((ctypes.c_void_p * n)(*src_ptrs), (ctypes.c_int * n)(*[len(u) for u in units]),
                                                 (ctypes.c_void_p * n)(*[ctypes.addressof(b) for b in dsts]),
                                                 (ctypes.c_int * n)(*caps), (ctypes.c_void_p * n)(*dict_ptrs),
                                                 (ctypes.c_int * n)(*dict_sizes), res, n, level)
    assert st == 0, lz.lib().LizardB200_lastError()
    return [(res[i], dsts[i].raw[:max(res[i], 0)]) for i in range(n)]


@pytest.mark.parametrize("level", [13, 17, 36, 21, 41])
def test_5000_unit_batch_is_one_launch(ref, level):
    """No dictionary, one shared dictionary, private dictionaries and prefixes in one call; units at the bound or at half of
    it; the GPU decodes the streams back against their dictionaries."""
    rng = np.random.default_rng(level)
    shared = _dictionary()
    shared_buf = ctypes.create_string_buffer(shared, len(shared) + 16)
    keep, units, dptr, dsize, sptr, dicts = [], [], [], [], [], []
    for i in range(5000):
        kind = i % 5
        n = int(rng.integers(0, 3000))
        u = records(n, 1000 * level + i) if i % 7 else shared[i % 50000:i % 50000 + n]
        if kind == 4:                                             # prefix: a private dictionary right in front of the unit
            d = records(int(rng.integers(1, 6000)), i)
            buf = ctypes.create_string_buffer(d + u, len(d) + len(u) + 16)
            keep.append(buf)
            dptr.append(ctypes.addressof(buf)); dsize.append(len(d)); sptr.append(ctypes.addressof(buf) + len(d))
        else:
            sb = ctypes.create_string_buffer(u, len(u) + 16)
            keep.append(sb)
            sptr.append(ctypes.addressof(sb))
            if kind == 0:
                d = b""
                dptr.append(None); dsize.append(0)
            elif kind in (1, 2) or i % 10 == 8:                  # the workspace holds about 1880 distinct dictionaries
                d = shared
                dptr.append(ctypes.addressof(shared_buf)); dsize.append(len(shared))
            else:
                d = records(int(rng.integers(1, 20000)), 7 * i)
                db = ctypes.create_string_buffer(d, len(d) + 16)
                keep.append(db)
                dptr.append(ctypes.addressof(db)); dsize.append(len(d))
        units.append(u)
        dicts.append(d)
    bound = [len(u) + 6 for u in units]
    caps = [b if i % 3 else max(b // 2, 1) for i, b in enumerate(bound)]
    before = lz.lib().LizardB200_launchCount()
    out = _batch_raw(units, dptr, dsize, sptr, caps, level)
    assert lz.lib().LizardB200_launchCount() - before == 1
    for i, (u, (r, o)) in enumerate(zip(units, out)):
        want = ref_run(ref, level, dptr[i], dsize[i], sptr[i], len(u), caps[i])
        assert r == len(want) and o == want, (level, i, i % 5, len(u), dsize[i], caps[i], r, len(want))
    ok = [i for i, (r, _) in enumerate(out) if r > 0]
    back = lz.decompress_dict_batch([out[i][1] for i in ok], [dicts[i] for i in ok], [len(units[i]) for i in ok])
    for i, (rb, ob) in zip(ok, back):
        assert rb == len(units[i]) and ob == units[i], i


def test_too_many_dictionaries_are_refused():
    """More distinct dictionaries than the workspace has slots for: LIZARDB200_ERR_MEMORY, with the bound in lastError."""
    dicts = [b"%08d" % i for i in range(4000)]
    with pytest.raises(lz.LizardB200Error, match="distinct dictionaries"):
        lz.compress_dict_batch([b"x" * 20] * 4000, dicts, 17)


def _device_layout(units, dicts, prefix):
    """One device buffer for inputs and dictionaries at odd offsets; a prefix unit's dictionary lies right in front of it."""
    h = bytearray(b"\x5C" * 3)
    so, do = [], []
    for u, d, p in zip(units, dicts, prefix):
        if p:
            do.append(len(h)); h += d
            so.append(len(h)); h += u
        else:
            do.append(len(h)); h += d + b"\x33" * 5
            so.append(len(h)); h += u
        h += b"\x77" * 3
    return bytes(h + bytes(16)), so, do


@pytest.mark.parametrize("level", [14, 17, 38, 22, 42])
def test_device_call_unaligned_with_guards(ref, level):
    import torch
    dev = torch.device("cuda", 0)
    d = _dictionary()
    units = [_straddler(d, level), records(1000, 1), records(77777, 2) + d[:5000], records(300000, 3), b"x" * 21, b"",
             records(lz.BLOCK_SIZE - 1, 4)]
    dicts = [d, d[-9000:], d, d, d[:7], d, records(2000, 9)]
    prefix = [False, True, False, True, False, False, True]
    h, so, do = _device_layout(units, dicts, prefix)
    hb = ctypes.create_string_buffer(h, len(h))
    base = ctypes.addressof(hb)
    caps = [len(u) + 2 + (len(u) // (1 << 17) + 1) * 4 for u in units]
    dst_off, at = [], 7
    for c in caps:
        dst_off.append(at)
        at += c + 64 + 3
    d_buf = torch.frombuffer(bytearray(h), dtype=torch.uint8).to(dev)
    d_dst = torch.full((at + 64,), 0xEE, dtype=torch.uint8, device=dev)
    t = lambda v, dt: torch.tensor(v, dtype=dt, device=dev)
    t_so, t_sl = t(so, torch.int64), t([len(u) for u in units], torch.int32)
    t_do, t_dc = t(dst_off, torch.int64), t(caps, torch.int32)
    t_dd, t_dl = t(do, torch.int64), t([len(x) for x in dicts], torch.int32)
    t_res = torch.zeros(len(units), dtype=torch.int32, device=dev)
    st = lz.lib().LizardB200_compress_dict_device(d_buf.data_ptr(), t_so.data_ptr(), t_sl.data_ptr(), d_dst.data_ptr(),
                                                  t_do.data_ptr(), t_dc.data_ptr(), d_buf.data_ptr(), t_dd.data_ptr(),
                                                  t_dl.data_ptr(), t_res.data_ptr(), len(units), level, None)
    assert st == 0
    torch.cuda.synchronize()
    res = t_res.cpu().tolist()
    out = d_dst.cpu().numpy().tobytes()
    for i, (u, o, c, r) in enumerate(zip(units, dst_off, caps, res)):
        want = ref_run(ref, level, base + do[i], len(dicts[i]), base + so[i], len(u), c)
        assert r == len(want) and out[o:o + r] == want, (i, r, len(want))
        assert set(out[o + r:o + c + 64]) <= {0xEE}
    assert set(out[:7]) == {0xEE}


def test_two_streams_share_the_workspace_with_the_other_encoders(ref):
    """A dictionary device call on one stream and, without a host sync, plain level-10 and level-24 device calls on another:
    the workspace is handed over between the launches and every result is the reference's."""
    import torch
    dev = torch.device("cuda", 0)
    d = _dictionary()
    units = [records(4000 + 37 * i, 500 + i) for i in range(600)]
    t = lambda v, dt: torch.tensor(v, dtype=dt, device=dev)
    h = b"".join(units)
    offs = list(np.cumsum([0] + [len(u) for u in units[:-1]]))
    d_src = torch.frombuffer(bytearray(h + bytes(16)), dtype=torch.uint8).to(dev)
    d_dict = torch.frombuffer(bytearray(d + bytes(16)), dtype=torch.uint8).to(dev)
    caps = [len(u) + 6 for u in units]
    t_so, t_sl = t(offs, torch.int64), t([len(u) for u in units], torch.int32)
    t_do, t_dc = t([32768 * i for i in range(len(units))], torch.int64), t(caps, torch.int32)
    t_zo, t_dl = t([0] * len(units), torch.int64), t([len(d)] * len(units), torch.int32)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    L = lz.lib()
    outs = {}
    for name, s, level in (("dict", s1, 17), ("plain10", s2, 10), ("dict2", s1, 41), ("lp", s2, 24), ("dict3", s2, 22)):
        dst = torch.zeros(32768 * len(units), dtype=torch.uint8, device=dev)
        res = torch.zeros(len(units), dtype=torch.int32, device=dev)
        if name.startswith("dict"):
            st = L.LizardB200_compress_dict_device(d_src.data_ptr(), t_so.data_ptr(), t_sl.data_ptr(), dst.data_ptr(),
                                                   t_do.data_ptr(), t_dc.data_ptr(), d_dict.data_ptr(), t_zo.data_ptr(),
                                                   t_dl.data_ptr(), res.data_ptr(), len(units), level, ctypes.c_void_p(s.cuda_stream))
        else:
            st = L.LizardB200_compress_device(d_src.data_ptr(), t_so.data_ptr(), t_sl.data_ptr(), dst.data_ptr(), t_do.data_ptr(),
                                              t_dc.data_ptr(), res.data_ptr(), len(units), level, ctypes.c_void_p(s.cuda_stream))
        assert st == 0
        outs[name] = (level, dst, res)
    torch.cuda.synchronize()
    db = ctypes.create_string_buffer(d, len(d))
    for name, (level, dst, res) in outs.items():
        r = res.cpu().tolist()
        o = dst.cpu().numpy().tobytes()
        for i, u in enumerate(units):
            if name.startswith("dict"):
                sb = ctypes.create_string_buffer(u, len(u) + 1)
                want = ref_run(ref, level, ctypes.addressof(db), len(d), ctypes.addressof(sb), len(u), caps[i])
            else:
                want = refs.ref_compress(ref, u, level, caps[i])
            assert r[i] == len(want) and o[32768 * i:32768 * i + r[i]] == want, (name, i)
