"""GPU parity of the optimal levels (19, 39) on the benchmark workload: 1 GiB `datagen -P50` in 8192 independent 128 KiB blocks
(capacity 128 KiB - 1), one launch over the whole grid, checked against the reference-generated facts of
tests/golden/optimal_1g.json (total compressed size and XXH64 of the concatenated blocks; tests/golden/make_opt_golden.py),
plus the round trip through the GPU decoder."""
import ctypes
import hashlib
import json
import os

import numpy as np
import pytest

import lizard_b200 as lz
from tests import refs

pytestmark = pytest.mark.gpu
BS = lz.BLOCK_SIZE
N = 1 << 30
with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "optimal_1g.json")) as _f:
    GOLDEN = json.load(_f)


@pytest.fixture(scope="module")
def ref():
    L = refs.ref_parity()
    if L is None:
        pytest.skip("oracle/_ref not built")
    L.Lizard_XXH64.restype = ctypes.c_ulonglong
    L.Lizard_XXH64.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_ulonglong]
    return L


@pytest.fixture(scope="module")
def data1g():
    a = np.empty(N, dtype=np.uint8)
    lz.datagen_into(a.ctypes.data, N, 50.0, 0)
    assert hashlib.md5(a).hexdigest() == GOLDEN["input"]["md5"]
    return a


@pytest.mark.parametrize("level", [19, 39])
def test_one_gib_matches_reference_facts(ref, data1g, level):
    L = lz.lib()
    L.LizardB200_compress_blocks.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t,
                                             ctypes.c_int, ctypes.c_void_p, ctypes.c_int]
    L.LizardB200_decompress_blocks.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t,
                                               ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]
    n = N // BS
    comp = np.empty(n * BS, dtype=np.uint8)
    sizes = np.zeros(n, dtype=np.int32)
    before = L.LizardB200_launchCount()
    st = L.LizardB200_compress_blocks(data1g.ctypes.data, N, BS, comp.ctypes.data, BS, BS - 1, sizes.ctypes.data, level)
    assert st == 0, L.LizardB200_lastError()
    assert L.LizardB200_launchCount() - before == 1
    assert int(sizes.min()) > 0
    fact = GOLDEN["facts"][str(level)]
    total = int(sizes.sum(dtype=np.int64))
    assert total == fact["total"]
    packed = np.concatenate([comp[i * BS:i * BS + int(sizes[i])] for i in range(n)])
    assert "%016x" % ref.Lizard_XXH64(packed.ctypes.data, total, 0) == fact["xxh64"]
    del packed
    back = np.zeros(N, dtype=np.uint8)
    res = np.zeros(n, dtype=np.int32)
    st = L.LizardB200_decompress_blocks(comp.ctypes.data, BS, sizes.ctypes.data, n, back.ctypes.data, BS, res.ctypes.data)
    assert st == 0, L.LizardB200_lastError()
    assert int(res.min()) == BS and int(res.max()) == BS
    assert np.array_equal(back, data1g)
