"""LizardB200_compressFramesAsync on the GPU (DESIGN.md 3.4c): tables and results in device memory, enqueue-only.

- Every admitted frame gets LizardB200_compressFrames's result and bytes (and the reference's frame where the reference
  writes one): every GPU level, block size IDs 1-7 with and without the checksum and the content size, empty and 1-byte
  frames at their bound and in the 25-32-byte range of the content-size quirk, linked preferences on single- and multi-block
  frames, refused levels; guard bytes around every range untouched.
- Admission: bounds of blocks or staging bytes that fit a prefix exactly, or miss it by one, admit exactly that prefix (also
  inside the second and third planning tile of a 3000-frame call); the rest get ERROR_allocation_failed, their ranges untouched.
- The call returns while the stream is still busy; a graph captured after a warm call compresses new contents and sizes on
  replay, and a graph that compresses and then decompresses (LizardB200_decompressFramesAsync) gives the input back; the launch
  count does not depend on the frames; two streams share the workspace; integer addresses; a capture that would grow the
  workspace is refused; stageBytes = SIZE_MAX; null tables; one 1 GiB frame."""
import ctypes

import numpy as np
import pytest

import lizard_b200 as lz
from tests.test_frame_compress_async_cpu import begin, block_size, one_shot
from tests.test_frame_device_cpu import _data
from tests.test_gpu_frame_device import (ERROR_LIMIT, GPU_LEVELS, GUARD, Arena, _inputs, check_guards, expect, first_diff,
                                         host_compress, out_arena, ours, ref, run_compress)   # noqa: F401 (fixtures)

pytestmark = pytest.mark.gpu
BS = lz.BLOCK_SIZE
ALLOC_FAILED = (1 << 64) - 9
SIZE_MAX = (1 << 64) - 1


def _torch():
    import torch
    return torch


def _tab(torch, v):
    return torch.tensor(v, dtype=torch.int64, device="cuda:0")


def _one_shot(p, n):
    q = one_shot(p.frameInfo.blockSizeID, p.frameInfo.blockMode, p.frameInfo.contentChecksumFlag, p.frameInfo.contentSize, n)
    q.compressionLevel = p.compressionLevel
    return q


def demand(ours, n, cap, p):
    """(blocks, staging bytes) an n-byte frame with cap bytes of room asks for: nothing if it fails LizardF_compressFrame's
    checks or is empty; else its blocks and their lengths rounded up to 16."""
    q = _one_shot(p, n)
    if n == 0 or cap < ours.LizardF_compressFrameBound(n, ctypes.byref(q)) or ours.LizardF_isError(begin(ours, q)[0]):
        return 0, 0
    bs = block_size(q.frameInfo.blockSizeID)
    nb = -(-n // bs)
    return nb, (nb - 1) * bs + ((n - (nb - 1) * bs + 15) // 16) * 16


def bounds(ours, units, caps, p):
    d = [demand(ours, len(u), c, p) for u, c in zip(units, caps)]
    return sum(b for b, _ in d), sum(s for _, s in d)


def run_async(ours, units, caps, p, max_blocks=None, stage=None, stream=None):
    """The units laid out as run_compress lays them out, through the async call; (results, output bytes, offsets)."""
    torch = _torch()
    mb, st = bounds(ours, units, caps, p)
    max_blocks = mb if max_blocks is None else max_blocks
    stage = st if stage is None else stage
    src = Arena(7)
    for u in units:
        src.put(u)
    d_src = src.device()
    dst = out_arena(caps)
    d_dst = dst.device()
    res = torch.full((len(units),), 0x7777, dtype=torch.int64, device="cuda:0")
    lz.compress_frames_async(d_src, _tab(torch, src.off), _tab(torch, [len(u) for u in units]), d_dst, _tab(torch, dst.off),
                             _tab(torch, caps), res, p, max_blocks, stage, stream)
    torch.cuda.synchronize()
    return [int(x) % (1 << 64) for x in res.cpu().tolist()], bytes(d_dst.cpu().numpy().tobytes()), dst.off


def same_as_sync(ours, units, caps, p, admitted=None, ref=None, **kw):
    """Admitted frames (all unless `admitted` says) get compressFrames's result and bytes, the others allocation_failed and
    nothing in their range; with `ref`, a frame the reference also writes equals it."""
    want, want_out, off = run_compress(units, caps, p)
    got, out, off2 = run_async(ours, units, caps, p, **kw)
    assert off == off2
    sizes = []
    for k, (u, c, w, r, o) in enumerate(zip(units, caps, want, got, off)):
        if admitted is not None and not admitted[k]:
            expect(r == ALLOC_FAILED, k, len(u), r, lz.frame_error(r))
            sizes.append(0)
            continue
        expect(r == w, k, len(u), c, r, w, lz.frame_error(r), lz.frame_error(w))
        if r < ERROR_LIMIT:
            expect(out[o:o + r] == want_out[o:o + r], k, len(u), first_diff(out[o:o + r], want_out[o:o + r]))
            if ref is not None:
                rr, rf = host_compress(ref, u, p, c)
                expect(ref.LizardF_isError(rr) or rr > c or rf == out[o:o + r], "reference", k, len(u))
        sizes.append(r if r < ERROR_LIMIT else 0)
    check_guards(out, off, caps, sizes)
    return got


# ---- same results and bytes as LizardB200_compressFrames -------------------------------------------------------------------
@pytest.mark.parametrize("level", GPU_LEVELS)
def test_every_gpu_level(ref, ours, level):
    units = _inputs(level)
    for checksum, csize in ((True, 1), (False, 0)):
        p = lz.make_prefs(level, 1, True, checksum, csize)
        caps = [ours.LizardF_compressFrameBound(len(u), ctypes.byref(p)) + 7 for u in units]
        res = same_as_sync(ours, units, caps, p, ref=ref)
        assert all(r < ERROR_LIMIT for r in res)


@pytest.mark.parametrize("bsid", [1, 2, 3, 4, 5, 6, 7])
def test_block_sizes(ours, bsid):
    units = [lz.datagen(n, 50, n) for n in (0, 1, 15, 200 << 10, (1 << 20) + 3, (4 << 20) + 1)]
    if bsid >= 5:
        units.append(_data((17 << 20) + 99, bsid))
    for checksum in (False, True):
        for csize in (0, 1):
            p = lz.make_prefs(10, bsid, True, checksum, csize)
            caps = [ours.LizardF_compressFrameBound(len(u), ctypes.byref(p)) for u in units]
            same_as_sync(ours, units, caps, p)


def test_empty_and_one_byte_frames(ours):
    """At the bound and through the range where a 1-byte input's record outgrows it (ERROR_dstMaxSize_tooSmall)."""
    for checksum in (False, True):
        for csize in (0, 1):
            p = lz.make_prefs(21, 1, True, checksum, csize)
            units, caps = [], []
            for u in (b"", b"x"):
                bound = ours.LizardF_compressFrameBound(len(u), ctypes.byref(p))
                for c in sorted({bound - 1, bound, bound + 1} | set(range(24, 34))):
                    units.append(u); caps.append(c)
            res = same_as_sync(ours, units, caps, p)
            if csize:
                assert any(lz.frame_error(r) == "ERROR_dstMaxSize_tooSmall" for u, r in zip(units, res) if u)


def test_linked_preferences(ours):
    units = [b"", b"x", lz.datagen(BS, 50, 1), lz.datagen(BS + 1, 50, 2), _data(3 * BS + 7, 3), lz.datagen(5000, 50, 4)]
    p = lz.make_prefs(10, 1, False, True, 1)
    caps = [ours.LizardF_compressFrameBound(len(u), ctypes.byref(p)) for u in units]
    res = same_as_sync(ours, units, caps, p)
    assert lz.frame_error(res[3]) == lz.frame_error(res[4]) == "ERROR_blockMode_invalid"
    assert res[2] < ERROR_LIMIT and res[5] < ERROR_LIMIT


def test_refused_levels(ours):
    units = _inputs(3)
    for level in (12, 26, 33, 49):
        p = lz.make_prefs(level, 1, True, True, 0)
        caps = [ours.LizardF_compressFrameBound(len(u), ctypes.byref(p)) for u in units]
        res = same_as_sync(ours, units, caps, p, max_blocks=64, stage=64 * BS)
        assert all(lz.frame_error(r) == "ERROR_compressionLevel_invalid" for r in res), level


# ---- admission ---------------------------------------------------------------------------------------------------------------
def check_admission(ours, units, caps, p, cuts, extra=()):
    """For each frame index k in `cuts`: bounds that end exactly at frame k's blocks or staging bytes, and one below."""
    per = [demand(ours, len(u), c, p) for u, c in zip(units, caps)]
    cum_b, cum_s = np.cumsum([b for b, _ in per]), np.cumsum([s for _, s in per])
    cases = list(extra)
    for k in cuts:
        cases += [(int(cum_b[k]), int(cum_s[-1])), (int(cum_b[k]) - 1, int(cum_s[-1])),
                  (int(cum_b[-1]), int(cum_s[k])), (int(cum_b[-1]), int(cum_s[k]) - 1)]
    for mb, st in cases:
        adm = [bool(b <= mb and s <= st) for b, s in zip(cum_b, cum_s)]
        assert adm == sorted(adm, reverse=True)
        same_as_sync(ours, units, caps, p, admitted=adm, max_blocks=mb, stage=st)


def _admission_frames(ours, p):
    units, caps = [], []
    for k in range(14):
        u = _data((k % 4) * BS + 100 * k + 1, k)                       # 1-4 blocks
        units.append(u); caps.append(ours.LizardF_compressFrameBound(len(u), ctypes.byref(_one_shot(p, len(u)))))
        if k % 4 == 1:
            units.append(b""); caps.append(100)                        # takes nothing
        if k % 5 == 2:
            units.append(u); caps.append(caps[-1] - 1)                 # below its bound: takes nothing
    return units, caps


def test_admission_prefix(ours):
    p = lz.make_prefs(21, 1, True, True, 1)
    units, caps = _admission_frames(ours, p)
    tb, ts = bounds(ours, units, caps, p)
    check_admission(ours, units, caps, p, (0, 3, 7, len(units) - 2), [(0, ts), (tb, 0), (0, 0)])


def test_admission_cut_in_a_later_planning_tile(ours):
    """3000 frames span three planning tiles of 1024: bounds that end inside the second and the third tile."""
    p = lz.make_prefs(10, 1, True, False, 0)
    rng = np.random.default_rng(21)
    pool = [b"", b"x", lz.datagen(700, 50, 1), lz.datagen(3000, 60, 2), _data(BS + 900, 3), lz.datagen(20000, 40, 4),
            rng.integers(0, 256, 5000, dtype=np.uint8).tobytes()]
    pcaps = [ours.LizardF_compressFrameBound(len(u), ctypes.byref(_one_shot(p, len(u)))) for u in pool]
    pool.append(pool[5]); pcaps.append(pcaps[5] - 1)                  # below its bound
    pick = [int(x) for x in rng.integers(0, len(pool), 3000)]
    units, caps = [pool[k] for k in pick], [pcaps[k] for k in pick]
    check_admission(ours, units, caps, p, (1100, 1500, 2047, 2048, 2600))


def test_five_thousand_mixed_frames(ours):
    rng = np.random.default_rng(5)
    sizes = [int(x) for x in rng.integers(0, 40000, 5000)]
    units = [lz.datagen(n, 50, i)[:n] for i, n in enumerate(sizes)]
    p = lz.make_prefs(10, 1, True, True, 1)
    caps = [ours.LizardF_compressFrameBound(n, ctypes.byref(p)) - (1 if i % 97 == 5 else 0) for i, n in enumerate(sizes)]
    res = same_as_sync(ours, units, caps, p)
    assert sum(r >= ERROR_LIMIT for r in res) > 40


# ---- enqueue-only, graphs, launches, streams -----------------------------------------------------------------------------------
def _tables(torch, ours, units, p, slot=None):
    """Device tables for units at fixed source slots (slot[k] bytes each, default the unit's size) and room for the largest."""
    slot = slot or [len(u) for u in units]
    src = Arena(11)
    for u, s in zip(units, slot):
        src.put(u + bytes([GUARD]) * (s - len(u)))
    caps = [ours.LizardF_compressFrameBound(s, ctypes.byref(p)) for s in slot]
    dst = out_arena(caps, 5)
    t = dict(src=src.device(), dst=dst.device(), src_off=_tab(torch, src.off), size=_tab(torch, [len(u) for u in units]),
             dst_off=_tab(torch, dst.off), cap=_tab(torch, caps), res=torch.zeros(len(units), dtype=torch.int64, device="cuda:0"))
    return t, src.off, dst.off, caps


def _call(t, p, mb, st, stream=None):
    lz.compress_frames_async(t["src"], t["src_off"], t["size"], t["dst"], t["dst_off"], t["cap"], t["res"], p, mb, st, stream)


def _check_tables(t, units, caps, p, dst_off):
    torch = _torch()
    torch.cuda.synchronize()
    want, want_out, woff = run_compress(units, caps, p)
    res = [int(x) % (1 << 64) for x in t["res"].cpu().tolist()]
    out = bytes(t["dst"].cpu().numpy().tobytes())
    for k, (w, r, o, wo) in enumerate(zip(want, res, dst_off, woff)):
        expect(r == w and w < ERROR_LIMIT and out[o:o + r] == want_out[wo:wo + w], k, r, w)


def test_returns_before_the_work_is_done(ours):
    torch = _torch()
    units = [_data(2 * BS + 1000 * k, k) for k in range(16)]
    p = lz.make_prefs(10, 1, True, True, 1)
    t, _, dst_off, caps = _tables(torch, ours, units, p)
    mb, st = bounds(ours, units, caps, p)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        _call(t, p, mb, st)                                             # warm-up: grows the workspace
        s.synchronize()
        t["res"].zero_(); s.synchronize()
        torch.cuda._sleep(1 << 30)                                      # about a second of GPU time ahead of the call
        _call(t, p, mb, st)
        busy = not s.query()
    assert busy, "the call waited for the stream"
    _check_tables(t, units, caps, p, dst_off)


def _replay_sets(k0):
    a = [_data(BS * (1 + k % 3) + 333 * k, k0 + k) for k in range(10)]
    b = [lz.datagen(BS * (k % 3) + 77 * k + 1, 40, k0 + 50 + k) for k in range(10)]
    return a, b


def test_cuda_graph_replays_new_contents(ours):
    torch = _torch()
    a, b = _replay_sets(0)
    slot = [max(len(x), len(y)) for x, y in zip(a, b)]
    p = lz.make_prefs(41, 1, True, True, 1)
    t, src_off, dst_off, caps = _tables(torch, ours, a, p, slot)
    mb = sum(-(-s // BS) for s in slot)
    st = mb * BS
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        _call(t, p, mb, st)                                             # warm-up of the same shape
    s.synchronize()
    _check_tables(t, a, caps, p, dst_off)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        _call(t, p, mb, st)
    for units in (b, a, b):
        host = bytearray(t["src"].cpu().numpy().tobytes())
        for u, o in zip(units, src_off):
            host[o:o + len(u)] = u
        t["src"].copy_(torch.frombuffer(host, dtype=torch.uint8))
        t["size"].copy_(_tab(torch, [len(u) for u in units]))
        t["res"].zero_()
        t["dst"].fill_(GUARD)
        torch.cuda.synchronize()
        g.replay()
        _check_tables(t, units, caps, p, dst_off)


def test_cuda_graph_compresses_then_decompresses(ours):
    """One captured graph: compress the units, then decompress the frames with their sizes read from the compress results."""
    torch = _torch()
    a, b = _replay_sets(7)
    slot = [max(len(x), len(y)) for x, y in zip(a, b)]
    p = lz.make_prefs(10, 1, True, True, 1)
    t, src_off, _, caps = _tables(torch, ours, a, p, slot)
    mb = sum(-(-s // BS) for s in slot)
    back = out_arena(slot, 13)
    d_back = back.device()
    back_off, back_cap = _tab(torch, back.off), _tab(torch, slot)
    res2 = torch.zeros(len(a), dtype=torch.int64, device="cuda:0")

    def both():
        _call(t, p, mb, mb * BS)
        lz.decompress_frames_async(t["dst"], t["dst_off"], t["res"], d_back, back_off, back_cap, res2, mb, mb * BS)

    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        both()                                                          # warm-up of the same shape
    s.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        both()
    for units in (b, a):
        host = bytearray(t["src"].cpu().numpy().tobytes())
        for u, o in zip(units, src_off):
            host[o:o + len(u)] = u
        t["src"].copy_(torch.frombuffer(host, dtype=torch.uint8))
        t["size"].copy_(_tab(torch, [len(u) for u in units]))
        res2.zero_()
        d_back.fill_(GUARD)
        torch.cuda.synchronize()
        g.replay()
        torch.cuda.synchronize()
        got = [int(x) for x in res2.cpu().tolist()]
        out = bytes(d_back.cpu().numpy().tobytes())
        for k, (u, o) in enumerate(zip(units, back.off)):
            expect(got[k] == len(u) and out[o:o + len(u)] == u, k, got[k], len(u))


def test_launches_do_not_depend_on_the_frames(ours):
    rng = np.random.default_rng(5)
    sizes = [int(x) for x in rng.integers(1, 40000, 5000)]
    units = [lz.datagen(n, 50, i)[:n] for i, n in enumerate(sizes)]
    p = lz.make_prefs(10, 1, True, True, 0)
    caps = [ours.LizardF_compressFrameBound(n, ctypes.byref(p)) for n in sizes]
    mb, st = bounds(ours, units, caps, p)
    counts = []
    for us, cs in (([units[1]], [caps[1]]), (units, caps), ([units[1]], [caps[1]])):
        before = ours.LizardB200_launchCount()
        res, _, _ = run_async(ours, us, cs, p, mb, st)
        counts.append(ours.LizardB200_launchCount() - before)
        assert res[1 if len(us) > 1 else 0] < ERROR_LIMIT
    assert counts[0] == counts[1] == counts[2], counts


def test_two_streams_share_the_workspace(ours):
    torch = _torch()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    ua = [_data(2 * BS + i * 1000, i) for i in range(20)]
    ub = [lz.datagen(BS // 2 + i, 50, 100 + i) for i in range(30)]
    p = lz.make_prefs(41, 1, True, True, 1)
    ta, _, oa, ca = _tables(torch, ours, ua, p)
    tb, _, ob, cb = _tables(torch, ours, ub, p)
    mb, st = bounds(ours, ua + ub, ca + cb, p)
    for _ in range(3):
        _call(ta, p, mb, st, s1)
        _call(tb, p, mb, st, s2)
    _check_tables(ta, ua, ca, p, oa)
    _check_tables(tb, ub, cb, p, ob)


def test_integer_addresses(ours):
    torch = _torch()
    units = [_data(BS + 99 * k, k) for k in range(5)]
    p = lz.make_prefs(21, 1, True, True, 1)
    t, _, dst_off, caps = _tables(torch, ours, units, p)
    mb, st = bounds(ours, units, caps, p)
    ptr = {k: v.data_ptr() for k, v in t.items()}
    lz.compress_frames_async(ptr["src"], ptr["src_off"], ptr["size"], ptr["dst"], ptr["dst_off"], ptr["cap"], ptr["res"], p,
                             mb, st, 0, n_frames=len(units))
    _check_tables(t, units, caps, p, dst_off)


def test_capture_that_would_grow_is_refused(ours):
    """A capture whose call would have to grow the workspace returns LIZARDB200_ERR_ARGUMENT and enqueues nothing; the same
    call outside a capture then grows it and compresses."""
    torch = _torch()
    units = [_data(BS + 7 * k, k) for k in range(4)]
    p = lz.make_prefs(10, 1, True, False, 0)
    t, _, dst_off, caps = _tables(torch, ours, units, p)
    mb, st = bounds(ours, units, caps, p)
    _call(t, p, mb, st)
    torch.cuda.synchronize()
    big = 1 << 21                                                     # block tables for more blocks than any call before
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    before = ours.LizardB200_launchCount()
    with torch.cuda.graph(g, stream=s):
        with pytest.raises(lz.LizardB200Error, match="must grow"):
            _call(t, p, big, st)
    assert ours.LizardB200_launchCount() == before
    torch.cuda.synchronize()
    t["res"].zero_()
    _call(t, p, big, st)
    _check_tables(t, units, caps, p, dst_off)


def test_stage_bytes_without_bound(ours):
    units = [_data(2 * BS + 50 * k, k) for k in range(6)]
    p = lz.make_prefs(21, 1, True, True, 1)
    caps = [ours.LizardF_compressFrameBound(len(u), ctypes.byref(p)) for u in units]
    mb, _ = bounds(ours, units, caps, p)
    res = same_as_sync(ours, units, caps, p, max_blocks=mb, stage=SIZE_MAX)
    assert all(r < ERROR_LIMIT for r in res)


def test_null_table_is_an_argument_error(ours):
    L = lz.lib()
    r = L.LizardB200_compressFramesAsync(None, None, None, None, None, None, None, 3, None, 1, 1 << 20, None)
    assert r == -1003
    assert b"null" in L.LizardB200_lastError()


def test_one_gib_frame_round_trip(ours):
    torch = _torch()
    n = 1 << 30
    host = torch.empty(n, dtype=torch.uint8).pin_memory()
    lz.datagen_into(host.data_ptr(), n, 50, 0)
    p = lz.make_prefs(10, 1, True, False, 0)
    cap = ours.LizardF_compressFrameBound(n, ctypes.byref(p))
    d_src = host.to("cuda:0")
    d_frame = torch.empty(cap, dtype=torch.uint8, device="cuda:0")
    res = torch.zeros(1, dtype=torch.int64, device="cuda:0")
    nb = n // BS
    lz.compress_frames_async(d_src, _tab(torch, [0]), _tab(torch, [n]), d_frame, _tab(torch, [0]), _tab(torch, [cap]), res, p,
                             nb, n)
    d_back = torch.empty(n, dtype=torch.uint8, device="cuda:0")
    res2 = torch.zeros(1, dtype=torch.int64, device="cuda:0")
    lz.decompress_frames_async(d_frame, _tab(torch, [0]), res, d_back, _tab(torch, [0]), _tab(torch, [n]), res2, nb, nb * BS)
    torch.cuda.synchronize()
    assert 0 < int(res[0]) <= cap and int(res2[0]) == n
    expect(torch.equal(d_back, d_src), "1 GiB round trip")
