#!/usr/bin/env python
"""optimal_bench.py -- kernel time of the optimal encoder (levels 18, 19, 39) on device-resident data: 1 GiB of
datagen -P50 cut into 128 KiB units (LizardB200_compress_device, capacity 128 KiB - 1 as the frame layer asks), and the
unmodified reference on all host threads of the same box over a prefix of the same data, through the oracle's threaded
harness as bench.py --impl reference runs it.  A development tool; bench.py is the contract bench.

GPU times are CUDA events around each call, the mean of --steps calls after --warmup untimed ones.  The reference time is the
mean of --ref-iters passes.  Prints one JSON line per level, then a table.

  python tools/optimal_bench.py [--size-mib 1024] [--levels 18,19,39] [--steps 5] [--ref-mib 256]
"""
import argparse
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
BS = 1 << 17


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size-mib", type=int, default=1024)
    ap.add_argument("--levels", default="18,19,39")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--ref-mib", type=int, default=256, help="reference sample (0: skip the reference)")
    ap.add_argument("--ref-iters", type=int, default=1)
    args = ap.parse_args()
    import torch
    import lizard_b200 as lz
    import bench
    from partial_bench import gpu_info
    if not torch.cuda.is_available():
        raise SystemExit("optimal_bench.py needs a CUDA device")
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
    idx = torch.arange(n, dtype=torch.int64, device=dev)
    d_src_off, d_comp_off = idx * BS, idx * stride
    d_src_len = torch.full((n,), BS, dtype=torch.int32, device=dev)
    d_cap = torch.full((n,), BS - 1, dtype=torch.int32, device=dev)
    d_csize = torch.zeros(n, dtype=torch.int32, device=dev)
    stream = torch.cuda.current_stream()
    sp = ctypes.c_void_p(stream.cuda_stream)
    gpu = gpu_info()
    O = cfn = dfn = None
    threads = 0
    if args.ref_mib:
        O, cfn, dfn, kind = bench.load_checker_libs()
        threads, _ = bench.host_threads()
    ref_n = min(args.ref_mib << 20, nbytes)
    rows = []
    for level in [int(x) for x in args.levels.split(",")]:
        def call():
            s = L.LizardB200_compress_device(d_src.data_ptr(), d_src_off.data_ptr(), d_src_len.data_ptr(), d_comp.data_ptr(),
                                             d_comp_off.data_ptr(), d_cap.data_ptr(), d_csize.data_ptr(), n, level, sp)
            assert s == 0, L.LizardB200_lastError()
        for _ in range(args.warmup):
            call()
        torch.cuda.synchronize()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(args.steps + 1)]
        ev[0].record(stream)
        for k in range(args.steps):
            call()
            ev[k + 1].record(stream)
        torch.cuda.synchronize()
        ts = [ev[k].elapsed_time(ev[k + 1]) for k in range(args.steps)]
        avg = sum(ts) / len(ts)
        cs = d_csize.cpu()
        # the frame layer's record size: the compressed block, or the block itself when it did not shrink
        total = int(torch.where(cs > 0, cs, torch.full_like(cs, BS)).sum())
        rec = {"level": level, "gpu_ms": round(avg, 2), "gpu_ms_per_GiB": round(avg * (1 << 30) / nbytes, 2),
               "gpu_MBps": round(nbytes / 1e6 / (avg / 1e3), 1), "compressed_total": total,
               "ratio": round(nbytes / total, 4), "gpu": gpu, "size_mib": args.size_mib}
        if O is not None:
            t, ref_total, ok = bench.cpu_round_trip(O, cfn, dfn, h_src.data_ptr(), ref_n, level, threads, args.ref_iters)
            tc = t["mean"][0]
            ours_prefix = int(torch.where(cs[:ref_n // BS] > 0, cs[:ref_n // BS], torch.full_like(cs[:ref_n // BS], BS)).sum())
            rec.update({"ref_kind": kind, "ref_threads": threads, "ref_mib": ref_n >> 20, "ref_MBps": round(ref_n / 1e6 / tc, 1),
                        "ref_ms_per_GiB": round(tc * 1e3 * (1 << 30) / ref_n, 1), "ref_total_prefix": int(ref_total),
                        "ours_total_prefix": ours_prefix, "ref_round_trip_ok": ok})
        print(json.dumps(rec), flush=True)
        rows.append(rec)
    print(f"\n{gpu}; {args.size_mib} MiB datagen -P50 in 128 KiB units; GPU mean of {args.steps} calls; reference on "
          f"{threads} host threads over {ref_n >> 20} MiB")
    print(f"{'level':>5} {'GPU ms/GiB':>11} {'GPU MB/s':>9} {'ref MB/s':>9} {'ratio':>7}")
    for r in rows:
        print(f"{r['level']:>5} {r['gpu_ms_per_GiB']:>11} {r['gpu_MBps']:>9} {r.get('ref_MBps', '-'):>9} {r['ratio']:>7}")


if __name__ == "__main__":
    main()
