"""Generate tests/golden/optimal_1g.json from the UNMODIFIED reference compiled at oracle/_ref (-DLIZARD_RESET_MEM build):
for levels 19 and 39, the total compressed size and the XXH64 (seed 0, the reference's own lib/xxhash) of the 8192 blocks of
1 GiB `datagen -P50` compressed one 128 KiB block per `Lizard_compress` call with capacity 128 KiB - 1, concatenated.  These
are the facts tests/test_gpu_optimal_fullsize.py checks the GPU against, as tests/test_gpu_fullsize.py does for 10/21/41.
Run where oracle/_ref is built (blocks go to all host threads; on 8 threads of a build machine the reference took about
92 s at level 19 and 107 s at level 39):
    python tests/golden/make_opt_golden.py"""
import ctypes
import hashlib
import json
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import lizard_b200 as lz  # noqa: E402
from tests import refs  # noqa: E402

BS = 1 << 17
N = 1 << 30
MD5_1G = "b98d56d2653b6ab1b74ebe6c827ec231"       # `datagen -g1G -P50` of the reference (tests/test_gpu_fullsize.py)


def main():
    ref = refs.ref_parity()
    assert ref is not None, "build oracle/_ref first"
    ref.Lizard_compress.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int]
    ref.Lizard_XXH64.restype = ctypes.c_ulonglong
    ref.Lizard_XXH64.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_ulonglong]
    data = np.empty(N, dtype=np.uint8)
    lz.datagen_into(data.ctypes.data, N, 50.0, 0)
    assert hashlib.md5(data).hexdigest() == MD5_1G
    n = N // BS
    out = {"generator": "oracle/_ref/liblizard_ref_parity.so (gcc -O3 -DLIZARD_RESET_MEM), tests/golden/make_opt_golden.py",
           "input": {"kind": "datagen", "size": N, "pct": 50, "seed": 0, "md5": MD5_1G},
           "block": BS, "cap": BS - 1, "facts": {}}
    for level in (19, 39):
        t0 = time.time()
        comp = np.empty(n * BS, dtype=np.uint8)
        sizes = np.zeros(n, dtype=np.int64)

        def one(i):
            sizes[i] = ref.Lizard_compress(data.ctypes.data + i * BS, comp.ctypes.data + i * BS, BS, BS - 1, level)

        with ThreadPoolExecutor(os.cpu_count() or 1) as ex:
            list(ex.map(one, range(n)))
        assert int(sizes.min()) > 0
        packed = np.concatenate([comp[i * BS:i * BS + int(sizes[i])] for i in range(n)])
        out["facts"][str(level)] = {"total": int(sizes.sum()), "xxh64": "%016x" % ref.Lizard_XXH64(packed.ctypes.data, len(packed), 0)}
        print(level, out["facts"][str(level)], "%.0f s" % (time.time() - t0), flush=True)
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "optimal_1g.json"), "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
