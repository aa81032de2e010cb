"""GPU: decoding against dictionaries.  The drop-in Lizard_decompress_safe_usingDict in its three modes, the streaming
decoder (Lizard_setStreamDecode / Lizard_decompress_safe_continue) over a linked stream, LizardB200_decompress_dict_batch
(one launch for thousands of units that mix no dictionary, shared and private dictionaries and in-place prefixes),
LizardB200_decompress_dict_device at unaligned offsets with guard bytes, and the reference's frame layer decoding linked
frames through our library (oracle/_ref/relinked_dict).  Every stream is written by the compiled reference."""
import ctypes
import os
import random
import subprocess

import pytest

import lizard_b200 as lz
from tests import refs
from tests.test_dict_cpu import (_linked_stream, _straddler, records, ref_compress_dict, ref_decode_dict)

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
RELINKED = os.path.join(refs.REF_DIR, "relinked_dict")


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


@pytest.fixture(scope="module")
def gpu():
    if not torch.cuda.is_available() or not lz.lib().LizardB200_available():
        pytest.skip("no usable CUDA device")
    return lz.lib()


def _dict(seed=12345, size=1 << 16):
    return records(size, seed)


@pytest.mark.parametrize("level", [10, 17, 21, 41, 45])
def test_drop_in_three_modes(ref, gpu, level):
    """No dictionary, in place, external: return codes and bytes of the reference, a shortened dictionary gives its token
    error, and a negative dictSize returns -1."""
    d = _dict()
    for data in (_straddler(d, level), records(20000, level) + d[-3000:]):
        assert lz.decompress_using_dict(refs.ref_compress(ref, data, level), b"", len(data)) == (len(data), data)
        for prefix in (True, False):
            comp = ref_compress_dict(ref, d, data, level, prefix)
            assert lz.decompress_using_dict(comp, d, len(data), prefix) == (len(data), data)
            for k in (1, 4000, len(d) - 9):
                want = ref_decode_dict(ref, comp, d[k:], len(data), prefix)
                r, out = lz.decompress_using_dict(comp, d[k:], len(data), prefix)
                assert r == want[0] and (r <= 0 or out == want[1]), (prefix, k, r, want[0])
            assert lz.decompress_using_dict(comp, d, len(data) - 1, prefix)[0] == ref_decode_dict(ref, comp, d, len(data) - 1, prefix)[0]
    L = gpu
    buf = ctypes.create_string_buffer(64)
    assert L.Lizard_decompress_safe_usingDict(comp, buf, len(comp), 64, buf, -5) == -1


@pytest.mark.parametrize("level", [10, 21, 41])
def test_continue_over_a_linked_stream(ref, gpu, level):
    """4 MiB that the reference compressed in 64 KiB linked pieces, decoded with Lizard_decompress_safe_continue into one
    buffer (prefix in place) and, compressed from two alternating buffers, into two alternating buffers (external
    dictionary).  Lizard_setStreamDecode to a saved copy of the last piece continues the second stream half way."""
    L = gpu
    piece = 64 << 10
    data = records(4 << 20, 40 + level)
    for double in (False, True):
        pieces = _linked_stream(ref, data, level, piece, double)
        sd = L.Lizard_createStreamDecode()
        assert L.Lizard_setStreamDecode(sd, None, 0) == 1
        total = ctypes.create_string_buffer(len(data))
        bufs = [ctypes.create_string_buffer(piece) for _ in range(2)]
        saved = ctypes.create_string_buffer(piece)
        out = bytearray()
        for k, (comp, n_in) in enumerate(pieces):
            dst = ctypes.addressof(bufs[k % 2]) if double else ctypes.addressof(total) + len(out)
            if double and k == len(pieces) // 2:
                ctypes.memmove(saved, bytes(out[-piece:]), piece)
                L.Lizard_setStreamDecode(sd, saved, piece)
            r = L.Lizard_decompress_safe_continue(sd, comp, dst, len(comp), n_in)
            assert r == n_in, (double, k, r)
            out += ctypes.string_at(dst, r)
        L.Lizard_freeStreamDecode(sd)
        assert bytes(out) == data, double


def test_batch_of_5000_mixed_units_is_one_launch(ref, gpu):
    """5000 units over levels 10-49: no dictionary, one shared dictionary, eight private ones, and in-place prefixes.  One
    launch of the dictionary kernel, plus the two Huffman pre-pass launches when the decode variant enables them."""
    L = gpu
    rnd = random.Random(5)
    shared = _dict(1)
    privates = [_dict(100 + i, 8192 + 1000 * i) for i in range(8)]
    kinds = ["none", "shared", "private", "prefix"]
    protos = []                                                 # (kind, dictionary, level, data, comp)
    for i in range(160):
        level = 10 + i % 40
        kind = kinds[i % 4]
        d = {"none": b"", "shared": shared, "private": privates[i % 8], "prefix": privates[(i + 3) % 8]}[kind]
        data = (_straddler(d, i) if d else records(3000, i))[: rnd.randrange(800, 3000)]
        comp = refs.ref_compress(ref, data, level) if not d else ref_compress_dict(ref, d, data, level, kind == "prefix")
        protos.append((kind, d, level, data, comp))
    n = 5000
    held, dict_bufs = [], {}
    src, csz, dst, cap, dp, ds = ((ctypes.c_void_p * n)(), (ctypes.c_int * n)(), (ctypes.c_void_p * n)(), (ctypes.c_int * n)(),
                                  (ctypes.c_void_p * n)(), (ctypes.c_int * n)())
    res = (ctypes.c_int * n)()
    plan = []
    for i in range(n):
        kind, d, level, data, comp = protos[i % len(protos)]
        sb = ctypes.create_string_buffer(comp, len(comp))
        if kind == "prefix":
            ob = ctypes.create_string_buffer(d + bytes(len(data) + 16), len(d) + len(data) + 16)
            dst[i] = ctypes.addressof(ob) + len(d)
            dp[i] = ctypes.addressof(ob)
        else:
            ob = ctypes.create_string_buffer(len(data) + 16)
            dst[i] = ctypes.addressof(ob)
            if d:
                if id(d) not in dict_bufs:
                    dict_bufs[id(d)] = ctypes.create_string_buffer(d, len(d))
                dp[i] = ctypes.addressof(dict_bufs[id(d)])
        held += [sb, ob]
        src[i] = ctypes.addressof(sb)
        csz[i], cap[i], ds[i] = len(comp), len(data), len(d)
        plan.append((kind, data))
    for variant, extra in ((7, 2), (3, 0), (31, 2)):
        assert L.LizardB200_setDecodeVariant(variant) == 0
        before = L.LizardB200_launchCount()
        assert L.LizardB200_decompress_dict_batch(src, csz, dst, cap, dp, ds, res, n) == 0
        assert L.LizardB200_launchCount() - before == 1 + extra
        for i, (kind, data) in enumerate(plan):
            assert res[i] == len(data) and ctypes.string_at(dst[i], res[i]) == data, (variant, i, kind, res[i])
    L.LizardB200_setDecodeVariant(7)
    # the Python binding: external dictionaries, one buffer per distinct bytes object
    units = [p[4] for p in protos if p[0] != "prefix"]
    got = lz.decompress_dict_batch(units, [p[1] for p in protos if p[0] != "prefix"], [len(p[3]) for p in protos if p[0] != "prefix"])
    assert [o for _, o in got] == [p[3] for p in protos if p[0] != "prefix"]


def test_device_call_at_unaligned_offsets_with_guards(ref, gpu):
    """Units, outputs and dictionaries at odd offsets of device allocations with guard bytes around every output and
    dictionary; one dictionary sits directly in front of its unit's output in the same allocation (in-place mode).  Only
    [dst, dst + result) changes, dictionaries stay as they were."""
    L = gpu
    dev = torch.device("cuda")
    shared = _dict(2)
    units = []
    for i, level in enumerate([10, 17, 21, 41, 45, 13, 26, 38]):
        data = _straddler(shared, 50 + i)
        units.append((level, data, ref_compress_dict(ref, shared, data, level, i == 3)))
    n = len(units)
    src_host = bytearray()
    s_off, s_len, o_off, o_cap, d_off, d_len = [], [], [], [], [], []
    arena = bytearray(b"\x77" * 5)                           # dictionaries and outputs share one allocation
    shared_at = len(arena)
    arena += shared + b"\x77" * 11
    for i, (level, data, comp) in enumerate(units):
        src_host += b"\x00" * (3 + i)
        s_off.append(len(src_host)); s_len.append(len(comp)); src_host += comp
        arena += b"\x5a" * (9 + i)
        if i == 3:                                              # in place: a copy of the dictionary right in front of the output
            d_off.append(len(arena)); arena += shared
        else:
            d_off.append(shared_at)
        d_len.append(len(shared))
        o_off.append(len(arena)); o_cap.append(len(data)); arena += b"\x5a" * (len(data) + 13 + i)
    t = lambda v, dt: torch.tensor(v, dtype=dt, device=dev)
    # every array a named tensor: a temporary's memory could go to the next allocation before the kernel reads it
    g_src, g_arena, res = t(list(src_host), torch.uint8), t(list(arena), torch.uint8), t([0] * n, torch.int32)
    g_s_off, g_s_len, g_o_off, g_o_cap = t(s_off, torch.int64), t(s_len, torch.int32), t(o_off, torch.int64), t(o_cap, torch.int32)
    g_d_off, g_d_len = t(d_off, torch.int64), t(d_len, torch.int32)
    st = L.LizardB200_decompress_dict_device(g_src.data_ptr(), g_s_off.data_ptr(), g_s_len.data_ptr(),
                                             g_arena.data_ptr(), g_o_off.data_ptr(), g_o_cap.data_ptr(),
                                             g_arena.data_ptr(), g_d_off.data_ptr(), g_d_len.data_ptr(),
                                             res.data_ptr(), n, None)
    assert st == 0
    torch.cuda.synchronize()
    want = bytearray(arena)
    for i, (level, data, comp) in enumerate(units):
        want[o_off[i]:o_off[i] + len(data)] = data
    assert res.cpu().tolist() == [len(u[1]) for u in units]
    assert bytes(g_arena.cpu().tolist()) == bytes(want)


@pytest.mark.parametrize("level", [10, 21, 41])
def test_reference_frame_layer_decodes_linked_frames(tmp_path, ref, gpu, level):
    """Linked-block frames that the pure reference wrote (4 MiB, 128 KiB blocks, a zeroed LizardF_preferences_t apart from
    the block size and level), decoded by the reference's frame layer over our library: whole (each block straight into the
    output, the previous blocks an in-place prefix) and in 4000-byte destination chunks (each block through the frame layer's
    temporary buffer, an external dictionary)."""
    if not os.path.exists(RELINKED):
        pytest.skip("oracle/_ref/relinked_dict not built")
    lz.bind_frame_api(ref)
    data = records(4 << 20, 70 + level)
    frame = lz.frame_compress(ref, data, lz.make_prefs(level, 1, False, True, 0))
    src = os.path.join(str(tmp_path), "in.liz")
    with open(src, "wb") as f:
        f.write(frame)
    for chunk in (len(data), 4000):
        out = os.path.join(str(tmp_path), "out.bin")
        r = subprocess.run([RELINKED, src, out, str(chunk)], capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, (chunk, r.stdout, r.stderr)
        assert open(out, "rb").read() == data, chunk
