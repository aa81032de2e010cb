"""Partial decoding on the H100: Lizard_decompress_safe_partial, LizardB200_decompress_partial_batch and
LizardB200_decompress_partial_device against the reference's Lizard_decompress_safe_partial (built with -DLIZARD_RESET_MEM).
Return codes always equal; bytes in front of the returned size equal where the reference's are defined (every offset >= 8);
nothing written outside a unit's [dst, dst + capacity).  A partial call is one launch of the partial kernel whatever the
decode variant, and a unit whose target is at or above its decoded size decodes exactly as LizardB200_decompress_batch."""
import ctypes
import random

import pytest

import lizard_b200 as lz
from tests import corpus, refs
from tests.test_gpu_corpus import _damage, _decode_case, _decode_variant, _families, _layout

pytestmark = pytest.mark.gpu
BS = lz.BLOCK_SIZE


@pytest.fixture(scope="module")
def ref():
    L = refs.ref_parity()
    if L is None:
        pytest.skip("oracle/_ref not built")
    L.Lizard_decompress_safe_partial.argtypes = [ctypes.c_char_p, ctypes.c_char_p, ctypes.c_int, ctypes.c_int, ctypes.c_int]
    return L


def _ref_partial(ref, comp, target, cap):
    dst = ctypes.create_string_buffer(2 * max(cap, 1) + 64)          # wild copies and raw blocks: see refs.ref_decompress
    r = ref.Lizard_decompress_safe_partial(comp, dst, len(comp), target, cap)
    return r, dst.raw[:max(r, 0)]


def _check(ref, units, targets, caps, results, outputs, what):
    """Return codes as the reference's, bytes where the reference's are defined.  The one documented exception (DESIGN.md
    3.5): behind a raw inner block the reference decodes past the capacity and reports more than `cap`; the device refuses."""
    bad, compared = [], 0
    for i, (u, t, cap, r, o) in enumerate(zip(units, targets, caps, results, outputs)):
        rr, ro = _ref_partial(ref, u, t, cap)
        if rr > cap:
            if r >= 0:
                bad.append((i, len(u), t, cap, r, rr, "accepted an overrun"))
        elif r != rr:
            bad.append((i, len(u), t, cap, r, rr))
        elif rr > 0 and refs.stream_obeys_min_offset(u, max(cap, rr)):
            compared += 1
            if o[:rr] != ro:
                bad.append((i, len(u), t, cap, "content"))
    assert not bad, (what, len(bad), bad[:10])
    return compared


def test_drop_in_symbol_matches_reference(ref):
    """Lizard_decompress_safe_partial on host buffers, one unit per call: targets below, inside and between the inner blocks
    of a three-block unit, and at or above its size."""
    L = lz.lib()
    assert L.Lizard_decompress_safe_partial(b"\x0a", None, 0, 5, 64) == 0        # compressedSize < 1: nothing is read
    for level in (10, 21, 41, 30, 45, 13, 26):
        data = lz.datagen(2 * BS + 5000, 50, level)
        comp = refs.ref_compress(ref, data, level)
        n = len(data)
        targets = [-1, 0, 1, 4096, BS - 1, BS + 1, 200000, n - 1, n, n + 1]
        out = [lz.decompress_partial(comp, t, n) for t in targets]
        _check(ref, [comp] * len(targets), targets, [n] * len(targets), [r for r, _ in out], [o for _, o in out], level)
        assert out[targets.index(200000)][0] == 2 * BS                  # the token loop's target is block relative


def _mixed_batch(ref, rnd, count):
    """`count` units of every level 10-49 and many sizes (a few of two and three inner blocks), a tenth of them damaged, with
    random targets; about a fifth have a target at or above the decoded size."""
    pool = lz.datagen(1 << 20, 50, 4) + b"".join(_families()["threshold"][:2]) + b"".join(_families()["periodic"])
    distinct = []
    for k in range(700):
        n = rnd.choice([0, 1, 5, 16, 100, 700, 2000, 4096, 9000, 30000, BS]) if k >= 12 else rnd.choice([2 * BS + 77, 3 * BS - 5])
        at = rnd.randrange(0, len(pool) - n)
        raw = pool[at:at + n]
        distinct.append((refs.ref_compress(ref, raw, rnd.randrange(10, 50)), n))
    units, targets, caps, full = [], [], [], []
    for _ in range(count):
        c, n = rnd.choice(distinct)
        if len(c) > 1 and rnd.random() < 0.1:
            c = _damage(rnd, c)
        pick = rnd.random()
        t = (rnd.choice([n, n + 1, 1 << 30]) if pick < 0.2 else rnd.choice([-1, 0, 1]) if pick < 0.3
             else rnd.randrange(0, max(n, 1)))
        units.append(c)
        targets.append(t)
        caps.append(n + rnd.choice([0, 0, 16, 100]))
        full.append(t >= n)
    return units, targets, caps, full


def test_thousands_of_units_of_every_level_with_random_targets(ref):
    """5000 units in one host batch under decode variants 3, 7 and 23: one launch each time, the same results each time, the
    reference's results, and the units whose target is at or above their size equal to LizardB200_decompress_batch."""
    L = lz.lib()
    units, targets, caps, full = _mixed_batch(ref, random.Random(11), 5000)
    seen = None
    for variant in (3, 7, 23):
        with _decode_variant(variant):
            before = L.LizardB200_launchCount()
            out = lz.decompress_partial_batch(units, targets, caps)
            assert L.LizardB200_launchCount() - before == 1, variant
        if seen is None:
            seen = out
        assert out == seen, variant
    assert _check(ref, units, targets, caps, [r for r, _ in seen], [o for _, o in seen], "batch") > 2000
    idx = [i for i, f in enumerate(full) if f]
    whole = lz.decompress_batch([units[i] for i in idx], [caps[i] for i in idx])
    assert [seen[i] for i in idx] == whole


def test_device_call_at_unaligned_offsets_writes_nothing_outside_a_unit(ref):
    """LizardB200_decompress_partial_device with the far-offset and codeword-threshold streams, intact and damaged, at every
    residue mod 16 of source and destination, random targets in device memory: the reference's results and bytes, and the
    guard bytes around every unit's [dst, dst + capacity) untouched."""
    import torch
    L = lz.lib()
    fams = _families()
    dev = torch.device("cuda", 0)
    for level in (20, 21, 22, 41, 10, 30, 45, 29):
        rnd = random.Random(level)
        _, comp = _decode_case(level)
        blocks = fams["far"] + fams["threshold"]
        streams = list(zip(comp[:len(blocks)], blocks))
        streams += [(_damage(rnd, c), b) for c, b in streams[:8]]
        units = [c for c, _ in streams]
        caps = [len(b) + rnd.choice([0, 0, 5]) for _, b in streams]
        targets = [rnd.choice([-1, 0, 1, len(b), rnd.randrange(0, len(b) + 1), rnd.randrange(0, min(len(b), BS) + 1)])
                   for _, b in streams]
        src_off, dst_off, n_src, n_dst = _layout(rnd, [len(c) for c in units], caps,
                                                 lambda i: (3 * i + level) % 16, lambda i: (7 * i + 1) % 16)
        h_src = bytearray(n_src)
        for o, c in zip(src_off, units):
            h_src[o:o + len(c)] = c
        d_src = torch.frombuffer(h_src, dtype=torch.uint8).to(dev)
        d_dst = torch.full((n_dst,), 0xEE, dtype=torch.uint8, device=dev)
        t = lambda v, dt: torch.tensor(v, dtype=dt, device=dev)
        t_so, t_sl = t(src_off, torch.int64), t([len(c) for c in units], torch.int32)
        t_do, t_dc, t_tg = t(dst_off, torch.int64), t(caps, torch.int32), t(targets, torch.int32)
        t_res = torch.zeros(len(units), dtype=torch.int32, device=dev)
        before = L.LizardB200_launchCount()
        st = L.LizardB200_decompress_partial_device(d_src.data_ptr(), t_so.data_ptr(), t_sl.data_ptr(), d_dst.data_ptr(),
                                                    t_do.data_ptr(), t_dc.data_ptr(), t_tg.data_ptr(), t_res.data_ptr(),
                                                    len(units), None)
        assert st == 0, L.LizardB200_lastError()
        torch.cuda.synchronize()
        assert L.LizardB200_launchCount() - before == 1
        out = bytes(d_dst.cpu().numpy())
        res = t_res.cpu().tolist()
        _check(ref, units, targets, caps, res, [out[o:o + c] for o, c in zip(dst_off, caps)], level)
        outside = bytearray(out)
        for o, c in zip(dst_off, caps):
            outside[o:o + c] = b"\xEE" * c
        assert outside == b"\xEE" * len(out), (level, "wrote outside a unit's destination")
