"""GPU parity of the optimal levels (18, 19, 39): every compress entry point writes the bytes of the reference built with
-DLIZARD_RESET_MEM, in one launch, and the GPU decoder reads them back, in full and in part."""
import ctypes

import numpy as np
import pytest

import lizard_b200 as lz
from tests import refs
from tests.corpus import corpus
from tests.test_gpu_encode import _cases
from tests.test_optimal_cpu import _long_runs, _periodic

pytestmark = pytest.mark.gpu
BS = lz.BLOCK_SIZE
LEVELS = [18, 19, 39]


@pytest.fixture(scope="module")
def ref():
    L = refs.ref_parity()
    if L is None:
        pytest.skip("oracle/_ref not built")
    return L


@pytest.fixture(scope="module")
def data4m():
    return lz.datagen(4 << 20, 50, 4)


@pytest.mark.parametrize("level", LEVELS)
def test_drop_in_symbol_and_round_trip(ref, data4m, level):
    for data in (data4m[:BS], data4m[:300000], data4m[:5000], b"", data4m[:1]):
        got = lz.compress(data, level)
        assert got == refs.ref_compress(ref, data, level), (level, len(data))
        if data:
            r, back = lz.decompress(got, len(data))
            assert r == len(data) and back == data


@pytest.mark.parametrize("level", [19, 39])
def test_whole_4mib_call(ref, data4m, level):
    got = lz.compress(data4m, level)
    assert got == refs.ref_compress(ref, data4m, level)
    r, back = lz.decompress(got, len(data4m))
    assert r == len(data4m) and back == data4m


@pytest.mark.parametrize("level", [18, 39])
def test_5000_unit_batch_is_one_launch(ref, level):
    rng = np.random.default_rng(level)
    sizes = rng.integers(0, 9000, 5000)
    big = lz.datagen(int(sizes.sum()) + 1, 50, level)
    units, at = [], 0
    for s in sizes:
        units.append(big[at:at + int(s)])
        at += int(s)
    caps = [ref.Lizard_compressBound(len(u)) if i % 3 else max(len(u) // 2, 1) for i, u in enumerate(units)]
    before = lz.lib().LizardB200_launchCount()
    out = lz.compress_batch(units, level, caps)
    assert lz.lib().LizardB200_launchCount() - before == 1
    for u, cap, (r, o) in zip(units, caps, out):
        want = refs.ref_compress(ref, u, level, cap)
        assert r == len(want) and o == want
    back = lz.decompress_batch([o for r, o in out if r > 0], [len(u) for u, (r, o) in zip(units, out) if r > 0])
    assert all(rb == len(u) and ob == u for (rb, ob), u in zip(back, [u for u, (r, o) in zip(units, out) if r > 0]))


@pytest.mark.parametrize("level", [19, 39])
def test_mixed_unit_sizes_contend_for_big_slots(ref, level):
    """Units of one inner block run on the per-warp map, larger ones queue for the few big slots."""
    units = []
    for i in range(120):
        n = [BS, 300000, BS // 3, 1 << 20, 200000][i % 5]
        units.append(lz.datagen(n, 40 + i % 50, i))
    out = lz.compress_batch(units, level, [ref.Lizard_compressBound(len(u)) for u in units])
    for i, (u, (r, o)) in enumerate(zip(units, out)):
        assert o == refs.ref_compress(ref, u, level), (level, i, len(u))


@pytest.mark.parametrize("level", [18, 39])
def test_device_call_unaligned_with_guards(ref, level):
    import torch
    dev = torch.device("cuda", 0)
    units = [lz.datagen(n, 50, n) for n in (BS, 1000, 77777, 300000, 21, 0, BS - 1)]
    src_off, at = [], 3
    for u in units:
        src_off.append(at)
        at += len(u) + 5
    h_src = bytearray(at + 8)
    for u, o in zip(units, src_off):
        h_src[o:o + len(u)] = u
    caps = [ref.Lizard_compressBound(len(u)) for u in units]
    dst_off, at = [], 7
    for c in caps:
        dst_off.append(at)
        at += c + 64 + 3
    d_src = torch.frombuffer(h_src, dtype=torch.uint8).to(dev)
    d_dst = torch.full((at + 64,), 0xEE, dtype=torch.uint8, device=dev)
    t = lambda v, dt: torch.tensor(v, dtype=dt, device=dev)
    t_so, t_sl = t(src_off, torch.int64), t([len(u) for u in units], torch.int32)
    t_do, t_dc = t(dst_off, torch.int64), t(caps, torch.int32)
    t_res = torch.zeros(len(units), dtype=torch.int32, device=dev)
    st = lz.lib().LizardB200_compress_device(d_src.data_ptr(), t_so.data_ptr(), t_sl.data_ptr(), d_dst.data_ptr(), t_do.data_ptr(),
                                             t_dc.data_ptr(), t_res.data_ptr(), len(units), level, None)
    assert st == 0
    torch.cuda.synchronize()
    res = t_res.cpu().tolist()
    out = d_dst.cpu().numpy().tobytes()
    for u, o, c, r in zip(units, dst_off, caps, res):
        want = refs.ref_compress(ref, u, level, c)
        assert r == len(want) and out[o:o + r] == want
        assert set(out[o + r:o + c + 64]) <= {0xEE}
    assert set(out[:7]) == {0xEE}


@pytest.mark.parametrize("level", [19, 39])
@pytest.mark.parametrize("block_id", [1, 4])
def test_compress_frame_bit_exact(level, block_id):
    R = refs.ref_parity()
    if R is None:
        pytest.skip("oracle/_ref not built")
    ref, ours = lz.bind_frame_api(R), lz.bind_frame_api(lz.lib())
    data = lz.datagen(9 * BS + 12345 if block_id == 1 else (9 << 20) + 999, 50, level)
    p = lz.make_prefs(level, block_id, True, True, 0)
    got = lz.frame_compress(ours, data, p)
    assert got == lz.frame_compress(ref, data, p)
    r, back = lz.frame_decompress(ours, got, len(data))
    assert r == 0 and back == data


@pytest.mark.parametrize("level", LEVELS)
def test_corpus_with_edge_capacities(ref, level):
    """The shared corpus, runs and short periods in one batch, each unit at its bound, its exact size, one byte less and half."""
    base = [u for fam in corpus().values() for u in fam] + list(_cases()) + [_long_runs(level), _periodic(3, 50000, level)]
    units, caps = [], []
    for u in base:
        bound = ref.Lizard_compressBound(len(u))
        n = len(refs.ref_compress(ref, u, level, bound))
        for cap in sorted({bound, n, max(n - 1, 1), max(n // 2, 1)}):
            units.append(u)
            caps.append(cap)
    out = lz.compress_batch(units, level, caps)
    for i, (u, cap, (r, o)) in enumerate(zip(units, caps, out)):
        want = refs.ref_compress(ref, u, level, cap)
        assert r == len(want) and o == want, (level, i, len(u), cap)


@pytest.mark.parametrize("level", [18, 39])
def test_compress_blocks(ref, level):
    L = lz.lib()
    for bs, n in ((BS, 9 * BS + 777), (300000, 1000000)):
        data = lz.datagen(n, 60, level + bs)
        nblk = (n + bs - 1) // bs
        stride = ref.Lizard_compressBound(bs)
        dst = ctypes.create_string_buffer(nblk * stride)
        sizes = (ctypes.c_int * nblk)()
        st = L.LizardB200_compress_blocks(data, n, bs, dst, stride, stride, sizes, level)
        assert st == 0, L.LizardB200_lastError()
        for i in range(nblk):
            blk = data[i * bs:(i + 1) * bs]
            assert dst.raw[i * stride:i * stride + sizes[i]] == refs.ref_compress(ref, blk, level, stride), (level, bs, i)


def test_workspace_shared_with_other_encoders_and_streams(ref):
    """The optimal kernel, the other encode kernels and the lowestPrice kernel take turns on one workspace, on two streams
    without a host sync in between: every launch finds the scratch as the previous one left it and still writes the
    reference's bytes."""
    import torch
    dev = torch.device("cuda", 0)
    units = [lz.datagen(n, 50, n) for n in (BS, 5000, 300000, 77777, BS - 3)]
    caps = [ref.Lizard_compressBound(len(u)) for u in units]
    src_off, at = [], 0
    for u in units:
        src_off.append(at)
        at += len(u)
    d_src = torch.frombuffer(bytearray(b"".join(units)), dtype=torch.uint8).to(dev)
    dst_off, at = [], 0
    for c in caps:
        dst_off.append(at)
        at += c
    t = lambda v, dt: torch.tensor(v, dtype=dt, device=dev)
    t_so, t_sl = t(src_off, torch.int64), t([len(u) for u in units], torch.int32)
    t_do, t_dc = t(dst_off, torch.int64), t(caps, torch.int32)
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    runs = []
    for i, level in enumerate([19, 10, 39, 25, 18, 41, 19, 45, 39]):
        d_dst = torch.zeros(at, dtype=torch.uint8, device=dev)
        t_res = torch.zeros(len(units), dtype=torch.int32, device=dev)
        s = streams[i % 2]
        st = lz.lib().LizardB200_compress_device(d_src.data_ptr(), t_so.data_ptr(), t_sl.data_ptr(), d_dst.data_ptr(),
                                                 t_do.data_ptr(), t_dc.data_ptr(), t_res.data_ptr(), len(units), level,
                                                 ctypes.c_void_p(s.cuda_stream))
        assert st == 0
        runs.append((level, d_dst, t_res))
    torch.cuda.synchronize()
    for level, d_dst, t_res in runs:
        out = d_dst.cpu().numpy().tobytes()
        for u, o, c, r in zip(units, dst_off, caps, t_res.cpu().tolist()):
            want = refs.ref_compress(ref, u, level, c)
            assert r == len(want) and out[o:o + r] == want, (level, len(u))


@pytest.mark.parametrize("level", [19, 39])
def test_gpu_decodes_the_output_in_full_and_in_part(ref, level):
    units = [lz.datagen(n, p, n) for n, p in ((BS, 50), (300000, 70), (5000, 20))] + [_long_runs(level), _periodic(5, 40000, 1)]
    out = lz.compress_batch(units, level, [ref.Lizard_compressBound(len(u)) for u in units])
    comp = [o for r, o in out]
    back = lz.decompress_batch(comp, [len(u) for u in units])
    assert all(r == len(u) and o == u for (r, o), u in zip(back, units))
    for frac in (1, 3, 7):
        targets = [len(u) * frac // 8 for u in units]
        part = lz.decompress_partial_batch(comp, targets, [len(u) for u in units])
        for (r, o), u, tg in zip(part, units, targets):
            assert r >= tg and o[:tg] == u[:tg], (level, len(u), tg, r)
