"""Kernel time of the lowestPrice encoder on hostile input: `collide` units (tests/corpus.py) whose planted keys fill
consecutive hashLog-23 buckets, so that the per-warp map builds long linear-probe runs, against a datagen unit.

Each case is one launch of LizardB200_compress_device over `--units` copies of one 128 KiB unit (at most one per resident
warp, so the launch time is the time one warp takes for the unit), timed with CUDA events, mean of `--reps` launches after
one warm-up.  Prints one JSON line per case with the GPU's name and power limit."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--levels", default="24,25")
    ap.add_argument("--keys", default="512,2048,8192,16376")
    ap.add_argument("--units", type=int, default=1024)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    import torch
    import lizard_b200 as lz
    from tests import corpus
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE,
                         text=True).stdout.strip().splitlines()[0]
    dev = torch.device("cuda", 0)
    L = lz.lib()
    for level in (int(x) for x in a.levels.split(",")):
        mls = 4 if level in (25, 45) else 5
        cases = [("datagen", lz.datagen(corpus.BS, 50, 1))]
        cases += [("collide-%d" % k, corpus.collide_unit(7, mls, (1 << 23) - k, keys=k)) for k in map(int, a.keys.split(","))]
        for name, unit in cases:
            n, cap = len(unit), lz.compress_bound(len(unit))
            d_src = torch.frombuffer(bytearray(unit), dtype=torch.uint8).to(dev)
            d_dst = torch.empty(a.units * cap, dtype=torch.uint8, device=dev)
            so = torch.zeros(a.units, dtype=torch.int64, device=dev)
            sl = torch.full((a.units,), n, dtype=torch.int32, device=dev)
            do = torch.arange(a.units, dtype=torch.int64, device=dev) * cap
            dc = torch.full((a.units,), cap, dtype=torch.int32, device=dev)
            res = torch.zeros(a.units, dtype=torch.int32, device=dev)
            call = lambda: L.LizardB200_compress_device(d_src.data_ptr(), so.data_ptr(), sl.data_ptr(), d_dst.data_ptr(),
                                                        do.data_ptr(), dc.data_ptr(), res.data_ptr(), a.units, level, None)
            assert call() == 0
            torch.cuda.synchronize()
            ms = []
            for _ in range(a.reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                assert call() == 0
                e1.record()
                torch.cuda.synchronize()
                ms.append(e0.elapsed_time(e1))
            ok = bool((res > 0).all().item())
            print(json.dumps({"gpu": gpu, "level": level, "case": name, "units": a.units, "ms_per_launch": sum(ms) / len(ms),
                              "ms_min": min(ms), "ms_max": max(ms), "compressed": int(res[0].item()), "ok": ok}), flush=True)


if __name__ == "__main__":
    main()
