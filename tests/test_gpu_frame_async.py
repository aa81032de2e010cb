"""LizardB200_decompressFramesAsync on the GPU (DESIGN.md 3.4b): tables and results in device memory, enqueue-only.

- Every admitted frame gets LizardB200_decompressFrames's result and bytes, on the corpora of test_gpu_frame_device.py: reference
  frames at levels 10-49, short blocks, damage mixed with good frames, frames of many tiny blocks, 5000 frames, checksummed
  good and bad, truncated and trailing-byte frames; guard bytes around every range untouched.
- Admission: bounds of blocks or slot bytes that fit a prefix exactly, or miss it by one, admit exactly that prefix; the rest
  get ERROR_allocation_failed with their ranges untouched.
- The call returns while the stream is still busy; a captured graph decodes new contents of the same tables on replay; the
  launch count does not depend on the frames; two streams share the workspace; one 1 GiB frame."""
import ctypes

import numpy as np
import pytest

import lizard_b200 as lz
from tests.test_frame_device_cpu import MAX_BLOCK, _damaged, _data, _ref_frames, _stream, frame_of
from tests.test_gpu_frame_device import (ERROR_LIMIT, GUARD, Arena, check_guards, expect, first_diff, out_arena,
                                         ref, ours, run_decompress)   # noqa: F401 (fixtures)

pytestmark = pytest.mark.gpu
BS = lz.BLOCK_SIZE
ALLOC_FAILED = (1 << 64) - 9


def _torch():
    import torch
    return torch


def walk(f: bytes):
    """(complete blocks, slot bytes) the call plans for a frame with a valid header (0, 0 for a bad magic)."""
    if len(f) < 7 or int.from_bytes(f[:4], "little") != 0x184D2206:
        return 0, 0
    fh = 15 if (f[4] >> 3) & 1 else 7
    mb = MAX_BLOCK.get((f[5] >> 4) & 7, 0)
    if len(f) < fh or not mb:
        return 0, 0
    pos, nb, slots = fh, 0, 0
    while len(f) - pos >= 4:
        w = int.from_bytes(f[pos:pos + 4], "little")
        c = w & 0x7FFFFFFF
        pos += 4
        if c == 0 or c > mb or len(f) - pos < c:
            break
        nb += 1
        slots += 0 if w >> 31 else mb
        pos += c
    return nb, slots


def bounds(frames):
    nb = sum(walk(f)[0] for f in frames)
    return nb, sum(walk(f)[1] for f in frames)


def _tab(torch, v):
    return torch.tensor(v, dtype=torch.int64, device="cuda:0")


def run_async(frames, caps, max_blocks=None, stage=None, stream=None):
    """The frames laid out as run_decompress lays them out, through the async call; (results, output bytes, offsets)."""
    torch = _torch()
    mb, st = bounds(frames)
    max_blocks = mb if max_blocks is None else max_blocks
    stage = st if stage is None else stage
    src = Arena(9)
    for f in frames:
        src.put(f)
    d_src = src.device()
    dst = out_arena(caps, 3)
    d_dst = dst.device()
    res = torch.full((len(frames),), 0x7777, dtype=torch.int64, device="cuda:0")
    lz.decompress_frames_async(d_src, _tab(torch, src.off), _tab(torch, [len(f) for f in frames]), d_dst, _tab(torch, dst.off),
                               _tab(torch, caps), res, max_blocks, stage, stream)
    torch.cuda.synchronize()
    return [int(x) % (1 << 64) for x in res.cpu().tolist()], bytes(d_dst.cpu().numpy().tobytes()), dst.off


def same_as_sync(frames, caps, names, **kw):
    want, want_out, off = run_decompress(frames, caps)
    got, out, off2 = run_async(frames, caps, **kw)
    assert off == off2
    sizes = []
    for name, c, w, r, o in zip(names, caps, want, got, off):
        expect(r == w, name, c, r, w, lz.frame_error(r), lz.frame_error(w))
        if r < ERROR_LIMIT:
            expect(out[o:o + r] == want_out[o:o + r], name, first_diff(out[o:o + r], want_out[o:o + r]))
        sizes.append(r if r < ERROR_LIMIT else c)
    check_guards(out, off, caps, sizes)
    return got


# ---- same results and bytes as LizardB200_decompressFrames -------------------------------------------------------------------
def test_reference_frames_all_levels(ref, ours):
    frames, caps, names = [], [], []
    sk = (0x184D2A5F).to_bytes(4, "little") + (9).to_bytes(4, "little") + b"123456789"
    for level in range(10, 50):
        data = _data(3 * BS + 1000 + level, level)
        for checksum, csize in ((True, 1), (False, 0)):
            frames.append(frame_of(ref, data, lz.make_prefs(level, 1, True, checksum, csize)))
            caps.append(len(data)); names.append(f"L{level}c{int(checksum)}")
        frames.append(sk); caps.append(16); names.append("skippable")
    for name, f, n in _ref_frames(ref):
        frames += [f, f]; caps += [n, n + 4096]; names += [name, name + "+room"]
    res = same_as_sync(frames, caps, names)
    assert all(r < ERROR_LIMIT for r in res)


def test_short_blocks(ref, ours):
    data = _data(9 * BS + 4321, 21)
    frames, caps, names = [], [], []
    for af in (0, 1):
        for level in (10, 21, 41, 45):
            p = lz.make_prefs(level, 1, True, bool(af), len(data) if af else 0)
            p.autoFlush = af
            f = _stream(ref, data, p, [1, BS - 1, 3, 2 * BS + 7, 500, 3 * BS, len(data) - 5 * BS - 511], {0, 2, 4})
            for c in (len(data), len(data) + 1, len(data) - 1, len(data) + BS, 2 * BS):
                frames.append(f); caps.append(c); names.append(f"af{af}L{level}cap{c}")
    same_as_sync(frames, caps, names)


def test_damage_mixed_with_good_frames(ref, ours):
    """Every class of damage: truncated and trailing-byte frames, bad headers, bad checksums, bad payloads, small capacities."""
    good_data = _data(3 * BS + 17, 4)
    good = frame_of(ref, good_data, lz.make_prefs(41, 1, True, True, 1))
    frames, caps, names = [], [], []
    for name, f, c, _ in _damaged(ref):
        frames += [good, f]; caps += [len(good_data), c]; names += ["good", name]
    res = same_as_sync(frames, caps, names)
    assert all(r == len(good_data) for r in res[0::2])
    assert sum(r >= ERROR_LIMIT for r in res[1::2]) > 30


def test_frames_of_many_tiny_blocks(ref, ours):
    good_data = _data(3 * BS + 17, 4)
    good = frame_of(ref, good_data, lz.make_prefs(21, 1, True, True, 1))
    frames, caps, names = [], [], []
    for bsid, pieces, level in ((6, 40, 10), (4, 33, 41), (1, 3000, 10)):        # 5.4 GiB of slots in all
        data = lz.datagen(2000 * pieces, 90, bsid + pieces)
        p = lz.make_prefs(level, bsid, True, True, len(data))
        p.autoFlush = 1
        frames += [good, _stream(ref, data, p, [2000] * pieces)]
        caps += [len(good_data), len(data)]; names += ["good", f"tiny{bsid}x{pieces}"]
    bad, pos = bytearray(frames[1]), 15
    for _ in range(19):
        pos += 4 + (int.from_bytes(bad[pos:pos + 4], "little") & 0x7FFFFFFF)
    bad[pos + 4 + 40] ^= 0xFF
    frames += [bytes(bad), good]; caps += [caps[1], len(good_data)]; names += ["tiny_damaged", "good"]
    res = same_as_sync(frames, caps, names)
    assert res[1] == caps[1] and res[3] == caps[3] and res[5] == caps[5]


def _five_thousand(ours, checksum=True):
    rng = np.random.default_rng(5)
    sizes = [int(x) for x in rng.integers(0, 40000, 5000)]
    units = [lz.datagen(n, 50, i)[:n] for i, n in enumerate(sizes)]
    p = lz.make_prefs(10, 1, True, checksum, 1)
    caps = [ours.LizardF_compressFrameBound(n, ctypes.byref(p)) for n in sizes]
    src = Arena(7)
    for u in units:
        src.put(u)
    d_src = src.device()
    dst = out_arena(caps)
    d_dst, dst_off = dst.device(), dst.off
    res = lz.compress_frames(d_src.data_ptr(), src.off, sizes, d_dst.data_ptr(), dst_off, caps, p)
    out = bytes(d_dst.cpu().numpy().tobytes())
    return units, [out[o:o + r] for o, r in zip(dst_off, res)]


def test_five_thousand_frames_checksummed_good_and_bad(ours):
    units, frames = _five_thousand(ours)
    frames = list(frames)
    for k in range(3, 5000, 101):                                     # damaged content checksums
        if len(frames[k]) > 20:
            f = bytearray(frames[k]); f[-1] ^= 0x40; frames[k] = bytes(f)
    caps = [len(u) for u in units]
    res = same_as_sync(frames, caps, [str(k) for k in range(5000)])
    assert sum(lz.frame_error(r) == "ERROR_contentChecksum_invalid" for r in res) > 40


# ---- admission ----------------------------------------------------------------------------------------------------------------
def _admission_frames(ref):
    frames, caps = [], []
    sk = (0x184D2A50).to_bytes(4, "little") + (3).to_bytes(4, "little") + b"abc"
    for k in range(12):
        data = _data((k % 4 + 1) * BS + 100 * k, k)                    # 2-5 blocks, one of them raw from 4 blocks up
        frames.append(frame_of(ref, data, lz.make_prefs((10, 21, 41)[k % 3], 1, True, k % 2 == 0, k % 3 == 0)))
        caps.append(len(data))
        if k % 4 == 1:
            frames.append(sk); caps.append(8)                          # takes nothing
        if k % 5 == 2:
            bad = bytearray(frames[-1]); bad[0] ^= 1
            frames.append(bytes(bad)); caps.append(len(data))          # fails its header check: takes nothing
    return frames, caps


def check_admission(frames, caps, cuts, extra=()):
    """For each frame index k in `cuts`: bounds that end exactly at frame k's blocks or slot bytes, and one below.  Admitted
    frames get decompressFrames's result and bytes, the rest ERROR_allocation_failed with their ranges untouched."""
    want, want_out, off = run_decompress(frames, caps)
    per = [walk(f) for f in frames]
    cum_b, cum_s = np.cumsum([b for b, _ in per]), np.cumsum([s for _, s in per])
    assert any(s < b * (128 << 10) for b, s in per)                  # some raw blocks take no slot
    cases = list(extra)
    for k in cuts:
        cases += [(int(cum_b[k]), int(cum_s[-1])), (int(cum_b[k]) - 1, int(cum_s[-1])),
                  (int(cum_b[-1]), int(cum_s[k])), (int(cum_b[-1]), int(cum_s[k]) - 1)]
    for mb, st in cases:
        adm = [bool(b <= mb and s <= st) for b, s in zip(cum_b, cum_s)]
        assert adm == sorted(adm, reverse=True)
        got, out, off2 = run_async(frames, caps, mb, st)
        sizes = []
        for k, (a, w, r, o, c) in enumerate(zip(adm, want, got, off, caps)):
            if a:
                expect(r == w, mb, st, k, r, w)
                if r < ERROR_LIMIT:
                    expect(out[o:o + r] == want_out[o:o + r], mb, st, k)
                sizes.append(r if r < ERROR_LIMIT else c)
            else:
                expect(r == ALLOC_FAILED, mb, st, k, r, lz.frame_error(r))
                sizes.append(0)                                       # nothing written to its range
        check_guards(out, off, caps, sizes)


def test_admission_prefix(ref, ours):
    frames, caps = _admission_frames(ref)
    per = [walk(f) for f in frames]
    check_admission(frames, caps, (0, 3, 7, len(frames) - 2), [(0, sum(s for _, s in per)), (sum(b for b, _ in per), 0)])


def test_admission_cut_in_a_later_planning_tile(ref, ours):
    """3000 frames span three planning tiles of 1024: bounds that end inside the second and the third tile."""
    pool, pcaps = [], []
    rng = np.random.default_rng(21)
    for j in range(12):
        pieces = j % 4 + 1
        data = rng.integers(0, 256, 700 * pieces, dtype=np.uint8).tobytes() if j % 3 == 0 else lz.datagen(700 * pieces, 60, j)
        p = lz.make_prefs((10, 21, 41)[j % 3], 1, True, j % 2 == 0, 0)
        p.autoFlush = 1
        pool.append(_stream(ref, data, p, [700] * pieces)); pcaps.append(len(data))   # 1-4 blocks of 700 bytes
    sk = (0x184D2A50).to_bytes(4, "little") + (3).to_bytes(4, "little") + b"abc"
    bad = bytearray(pool[1]); bad[0] ^= 1
    pool += [sk, bytes(bad)]; pcaps += [8, pcaps[1]]
    pick = [int(x) for x in rng.integers(0, len(pool), 3000)]
    frames, caps = [pool[k] for k in pick], [pcaps[k] for k in pick]
    check_admission(frames, caps, (1100, 1500, 2047, 2048, 2600))


# ---- enqueue-only, graphs, launches, streams ----------------------------------------------------------------------------------
def _tables(torch, frames, caps, slot=None):
    """Device tables for frames at fixed source slots (slot[k] bytes each, default the frame's size)."""
    slot = slot or [len(f) for f in frames]
    src = Arena(11)
    for f, s in zip(frames, slot):
        src.put(f + bytes([GUARD]) * (s - len(f)))
    dst = out_arena(caps, 5)
    t = dict(src=src.device(), dst=dst.device(), src_off=_tab(torch, src.off), size=_tab(torch, [len(f) for f in frames]),
             dst_off=_tab(torch, dst.off), cap=_tab(torch, caps), res=torch.zeros(len(frames), dtype=torch.int64, device="cuda:0"))
    return t, src.off, dst.off


def _call(t, mb, st, stream=None):
    lz.decompress_frames_async(t["src"], t["src_off"], t["size"], t["dst"], t["dst_off"], t["cap"], t["res"], mb, st, stream)


def _check_tables(t, frames, datas, dst_off):
    torch = _torch()
    torch.cuda.synchronize()
    res = [int(x) for x in t["res"].cpu().tolist()]
    out = bytes(t["dst"].cpu().numpy().tobytes())
    for k, (d, r, o) in enumerate(zip(datas, res, dst_off)):
        expect(r == len(d) and out[o:o + r] == d, k, r, len(d))


def test_returns_before_the_work_is_done(ref, ours):
    torch = _torch()
    datas = [_data(2 * BS + 1000 * k, k) for k in range(16)]
    frames = [frame_of(ref, d, lz.make_prefs(10, 1, True, True, 1)) for d in datas]
    t, _, dst_off = _tables(torch, frames, [len(d) for d in datas])
    mb, st = bounds(frames)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        _call(t, mb, st)                                                # warm-up: grows the workspace
        s.synchronize()
        t["res"].zero_(); s.synchronize()
        torch.cuda._sleep(1 << 30)                                      # about a second of GPU time ahead of the call
        _call(t, mb, st)
        busy = not s.query()
    assert busy, "the call waited for the stream"
    _check_tables(t, frames, datas, dst_off)


def test_cuda_graph_replays_new_contents(ref, ours):
    torch = _torch()
    a = [_data(BS * (1 + k % 3) + 333 * k, k) for k in range(10)]
    b = [_data(BS * (1 + k % 3) + 333 * k, 50 + k) for k in range(10)]
    pa = [frame_of(ref, d, lz.make_prefs((10, 41, 21)[k % 3], 1, True, k % 2 == 0, 1)) for k, d in enumerate(a)]
    pb = [frame_of(ref, d, lz.make_prefs((21, 10, 41)[k % 3], 1, True, k % 2 == 1, 0)) for k, d in enumerate(b)]
    slot = [max(len(x), len(y)) for x, y in zip(pa, pb)]
    caps = [len(d) for d in a]
    t, src_off, dst_off = _tables(torch, pa, caps, slot)
    mb = max(bounds(pa)[0], bounds(pb)[0])
    st = max(bounds(pa)[1], bounds(pb)[1])
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        _call(t, mb, st)                                                # warm-up of the same shape
    s.synchronize()
    _check_tables(t, pa, a, dst_off)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        _call(t, mb, st)
    for frames, datas in ((pb, b), (pa, a), (pb, b)):
        host = bytearray(t["src"].cpu().numpy().tobytes())
        for f, o in zip(frames, src_off):
            host[o:o + len(f)] = f
        t["src"].copy_(torch.frombuffer(host, dtype=torch.uint8))
        t["size"].copy_(_tab(torch, [len(f) for f in frames]))
        t["res"].zero_()
        t["dst"].fill_(GUARD)
        torch.cuda.synchronize()
        g.replay()
        _check_tables(t, frames, datas, dst_off)


def test_launches_do_not_depend_on_the_frames(ours):
    units, frames = _five_thousand(ours, checksum=False)
    one = [frames[1]]
    mb, st = bounds(frames)
    counts = []
    for fr in (one, frames, one):
        before = ours.LizardB200_launchCount()
        res, _, _ = run_async(fr, [len(units[1])] if fr is one else [len(u) for u in units], mb, st)
        counts.append(ours.LizardB200_launchCount() - before)
        assert res[1 if fr is frames else 0] == len(units[1])
    assert counts[1] == counts[2], counts


def test_two_streams_share_the_workspace(ref, ours):
    torch = _torch()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    da = [_data(2 * BS + i * 1000, i) for i in range(20)]
    db = [lz.datagen(BS // 2 + i, 50, 100 + i) for i in range(30)]
    fa = [frame_of(ref, d, lz.make_prefs(41, 1, True, True, 0)) for d in da]
    fb = [frame_of(ref, d, lz.make_prefs(17, 1, True, False, 1)) for d in db]
    ta, _, oa = _tables(torch, fa, [len(d) for d in da])
    tb, _, ob = _tables(torch, fb, [len(d) for d in db])
    mb, st = bounds(fa + fb)
    for _ in range(3):
        _call(ta, mb, st, s1)
        _call(tb, mb, st, s2)
    _check_tables(ta, fa, da, oa)
    _check_tables(tb, fb, db, ob)


def test_integer_addresses(ref, ours):
    torch = _torch()
    datas = [_data(BS + 99 * k, k) for k in range(5)]
    frames = [frame_of(ref, d, lz.make_prefs(21, 1, True, True, 1)) for d in datas]
    t, _, dst_off = _tables(torch, frames, [len(d) for d in datas])
    mb, st = bounds(frames)
    ptr = {k: v.data_ptr() for k, v in t.items()}
    lz.decompress_frames_async(ptr["src"], ptr["src_off"], ptr["size"], ptr["dst"], ptr["dst_off"], ptr["cap"], ptr["res"],
                               mb, st, 0, n_frames=len(frames))
    _check_tables(t, frames, datas, dst_off)


def test_one_gib_frame_round_trip(ours):
    torch = _torch()
    n = 1 << 30
    host = torch.empty(n, dtype=torch.uint8).pin_memory()
    lz.datagen_into(host.data_ptr(), n, 50, 0)
    p = lz.make_prefs(10, 1, True, True, 0)
    cap = ours.LizardF_compressFrameBound(n, ctypes.byref(p))
    d_src = host.to("cuda:0")
    d_frame = torch.empty(cap, dtype=torch.uint8, device="cuda:0")
    r = lz.compress_frames(d_src.data_ptr(), [0], [n], d_frame.data_ptr(), [0], [cap], p)
    assert not ours.LizardF_isError(r[0])
    d_back = torch.empty(n, dtype=torch.uint8, device="cuda:0")
    res = torch.zeros(1, dtype=torch.int64, device="cuda:0")
    nb = n // BS
    lz.decompress_frames_async(d_frame, _tab(torch, [0]), _tab(torch, [r[0]]), d_back, _tab(torch, [0]), _tab(torch, [n]), res,
                               nb, nb * BS)
    torch.cuda.synchronize()
    assert int(res[0]) == n
    expect(torch.equal(d_back, d_src), "1 GiB round trip")


def test_stage_bytes_without_bound(ref, ours):
    """stageBytes = SIZE_MAX admits every frame that fits maxBlocks and decodes it (the arena is sized for maxBlocks slots of
    256 MiB at most); a maxBlocks whose tables and arena the device cannot hold gives LIZARDB200_ERR_MEMORY and no launch."""
    datas = [_data(2 * BS + 50 * k, k) for k in range(6)]
    frames = [frame_of(ref, d, lz.make_prefs(21, 1, True, True, 1)) for d in datas]
    mb, _ = bounds(frames)
    got, out, off = run_async(frames, [len(d) for d in datas], mb, (1 << 64) - 1)
    assert got == [len(d) for d in datas]
    assert all(out[o:o + len(d)] == d for o, d in zip(off, datas))
    torch = _torch()
    t, _, _ = _tables(torch, frames, [len(d) for d in datas])
    before = ours.LizardB200_launchCount()
    with pytest.raises(lz.LizardB200Error, match="status -1005"):
        _call(t, (1 << 32) - 1, (1 << 64) - 1)
    assert ours.LizardB200_launchCount() == before
    # the workspace is usable again after the failed growth
    got, out, off = run_async(frames, [len(d) for d in datas])
    assert got == [len(d) for d in datas]


def test_null_table_is_an_argument_error(ours):
    r = ours.LizardB200_decompressFramesAsync(None, None, None, None, None, None, None, 3, 1, 1 << 20, None)
    assert r == -1003
    assert b"null" in ours.LizardB200_lastError()


def test_capture_that_would_grow_is_refused(ref, ours):
    """A capture whose call would have to grow the decoder's pre-pass workspace -- more units than any call before, while the
    frame tables and the arena are already large enough -- returns LIZARDB200_ERR_ARGUMENT and enqueues nothing; the same call
    outside a capture then grows it and decodes."""
    torch = _torch()
    units = 1 << 19                                                   # pre-pass tables for more units than earlier calls
    n_big = 520000                                                    # frame tables at least as large as `units` blocks need
    empty = torch.zeros(n_big, dtype=torch.int64, device="cuda:0")    # frames of 0 bytes (frameSize_wrong), no blocks
    res = torch.zeros(n_big, dtype=torch.int64, device="cuda:0")
    d = torch.zeros(16, dtype=torch.uint8, device="cuda:0")
    lz.decompress_frames_async(d, empty, empty, d, empty, empty, res, 8, 8 * BS)
    torch.cuda.synchronize()
    assert lz.frame_error(int(res[0]) % (1 << 64)) == "ERROR_frameSize_wrong"
    datas = [_data(BS + 7 * k, k) for k in range(4)]
    frames = [frame_of(ref, d, lz.make_prefs(10, 1, True, False, 0)) for d in datas]
    t, _, dst_off = _tables(torch, frames, [len(d) for d in datas])
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    before = ours.LizardB200_launchCount()
    with torch.cuda.graph(g, stream=s):
        with pytest.raises(lz.LizardB200Error, match="must grow"):
            _call(t, units, 8 * BS)
    assert ours.LizardB200_launchCount() == before
    torch.cuda.synchronize()
    _call(t, units, 8 * BS)
    _check_tables(t, frames, datas, dst_off)
