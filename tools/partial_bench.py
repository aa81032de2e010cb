#!/usr/bin/env python
"""partial_bench.py -- kernel time of the partial decode (LizardB200_decompress_partial_device) against the full decode
(LizardB200_decompress_device, default variant) on device-resident data: 1 GiB of datagen -P50 cut into 128 KiB units,
compressed on the GPU at each level, then decoded with every unit's target at 4 KiB, 16 KiB, 64 KiB and the full block.
A development tool; bench.py is the contract bench.

Times are CUDA events around each call, the mean of --steps calls after --warmup untimed ones.  "ms_per_GiB" is per GiB of
the units' decoded size (all of the input), whatever the target.  Prints one JSON line per case, then a table.

  python tools/partial_bench.py [--size-mib 1024] [--levels 10,21,41] [--targets 4096,16384,65536,full] [--steps 10]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
BS = 1 << 17


def gpu_info():
    """Card name and power limit, read in the same run as the numbers."""
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size-mib", type=int, default=1024)
    ap.add_argument("--levels", default="10,21,41")
    ap.add_argument("--targets", default="4096,16384,65536,full")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    import torch
    import lizard_b200 as lz
    if not torch.cuda.is_available():
        raise SystemExit("partial_bench.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    L = lz.lib()
    assert L.LizardB200_setDevice(0) == 0, L.LizardB200_lastError().decode()
    nbytes = args.size_mib << 20
    n = nbytes // BS
    h_src = torch.empty(nbytes, dtype=torch.uint8).pin_memory()
    lz.datagen_into(h_src.data_ptr(), nbytes, 50.0, 0)
    d_src = h_src.to(dev)
    stride = (L.Lizard_compressBound(BS) + 15) // 16 * 16
    d_comp = torch.empty(n * stride, dtype=torch.uint8, device=dev)
    d_back = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    idx = torch.arange(n, dtype=torch.int64, device=dev)
    d_src_off, d_comp_off = idx * BS, idx * stride
    d_src_len = torch.full((n,), BS, dtype=torch.int32, device=dev)
    d_cap = torch.full((n,), BS - 1, dtype=torch.int32, device=dev)
    d_back_cap = torch.full((n,), BS, dtype=torch.int32, device=dev)
    d_csize = torch.zeros(n, dtype=torch.int32, device=dev)
    d_dsize = torch.zeros(n, dtype=torch.int32, device=dev)
    stream = torch.cuda.current_stream()
    sp = ctypes.c_void_p(stream.cuda_stream)

    def timed(fn):
        for _ in range(args.warmup):
            fn()
        torch.cuda.synchronize()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(args.steps + 1)]
        ev[0].record(stream)
        for k in range(args.steps):
            fn()
            ev[k + 1].record(stream)
        torch.cuda.synchronize()
        ts = [ev[k].elapsed_time(ev[k + 1]) for k in range(args.steps)]
        return sum(ts) / len(ts), min(ts)

    gpu = gpu_info()
    rows = []
    for level in [int(x) for x in args.levels.split(",")]:
        s = L.LizardB200_compress_device(d_src.data_ptr(), d_src_off.data_ptr(), d_src_len.data_ptr(), d_comp.data_ptr(),
                                         d_comp_off.data_ptr(), d_cap.data_ptr(), d_csize.data_ptr(), n, level, sp)
        assert s == 0, L.LizardB200_lastError()
        torch.cuda.synchronize()
        assert int((d_csize <= 0).sum()) == 0, "a unit did not compress"

        def full():
            s = L.LizardB200_decompress_device(d_comp.data_ptr(), d_comp_off.data_ptr(), d_csize.data_ptr(), d_back.data_ptr(),
                                               d_src_off.data_ptr(), d_back_cap.data_ptr(), d_dsize.data_ptr(), n, sp)
            assert s == 0, L.LizardB200_lastError()

        for tname in args.targets.split(","):
            tgt = BS if tname == "full" else int(tname)
            d_tgt = torch.full((n,), tgt, dtype=torch.int32, device=dev)

            def partial():
                s = L.LizardB200_decompress_partial_device(d_comp.data_ptr(), d_comp_off.data_ptr(), d_csize.data_ptr(),
                                                           d_back.data_ptr(), d_src_off.data_ptr(), d_back_cap.data_ptr(),
                                                           d_tgt.data_ptr(), d_dsize.data_ptr(), n, sp)
                assert s == 0, L.LizardB200_lastError()

            d_back.zero_()
            avg, best = timed(partial)
            res = d_dsize
            head = min(tgt, BS)
            ok = bool(((res >= head) & (res <= BS)).all()) and bool(torch.equal(d_back.view(n, BS)[:, :head], d_src.view(n, BS)[:, :head]))
            rec = {"kernel": "decode_partial", "level": level, "target": tname, "ms_avg": round(avg, 3), "ms_best": round(best, 3),
                   "ms_per_GiB": round(avg * (1 << 30) / nbytes, 3), "mean_result": round(float(res.float().mean()), 1),
                   "prefix_ok": ok, "gpu": gpu}
            print(json.dumps(rec), flush=True)
            rows.append(rec)
        d_back.zero_()
        avg, best = timed(full)
        ok = bool(torch.equal(d_back, d_src)) and int((d_dsize != BS).sum()) == 0
        rec = {"kernel": "decode_full", "level": level, "target": "-", "ms_avg": round(avg, 3), "ms_best": round(best, 3),
               "ms_per_GiB": round(avg * (1 << 30) / nbytes, 3), "mean_result": BS, "prefix_ok": ok, "gpu": gpu}
        print(json.dumps(rec), flush=True)
        rows.append(rec)
    print(f"\n{gpu}; {args.size_mib} MiB datagen -P50 in 128 KiB units; mean of {args.steps} calls")
    print(f"{'level':>5} {'call':>14} {'target':>7} {'ms/GiB':>8} {'mean result':>12} {'ok':>4}")
    for r in rows:
        print(f"{r['level']:>5} {r['kernel']:>14} {r['target']:>7} {r['ms_per_GiB']:>8} {r['mean_result']:>12} {str(r['prefix_ok']):>4}")
    if not all(r["prefix_ok"] for r in rows):
        raise SystemExit("a decode returned wrong bytes")


if __name__ == "__main__":
    main()
