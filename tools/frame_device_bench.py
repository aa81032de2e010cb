#!/usr/bin/env python
"""frame_device_bench.py -- LizardF frames in device memory (LizardB200_compressFrames / LizardB200_decompressFrames) against
the same work through the host frame API (LizardF_compressFrame / LizardF_decompress on pinned host buffers).
A development tool; bench.py is the contract bench.

Workloads (datagen -P50): 8192 frames of 128 KiB, and one frame of 1 GiB; levels 10, 21 and 41; content checksum off and on.
For each: the device compress and decompress calls (CUDA events around each call; the calls synchronise), the time of the
frame index, frame assembly (scan + assemble) and XXH32 kernels on their own (torch.profiler, kernel durations summed over one
profiled calls), and the host path over the same frames.  Means of --steps calls after --warmup untimed ones; the host path
runs --host-steps times.  The card's name and power limit are read in the same run.  Prints one JSON line per case, then a
table.

  python tools/frame_device_bench.py [--levels 10,21,41] [--steps 5] [--warmup 1] [--host-steps 1] [--only small|big]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
BS = 1 << 17
KERNELS = {"index": ("lizard_frame_index_kernel",), "assembly": ("lizard_frame_scan_kernel", "lizard_frame_assemble_kernel"),
           "hash": ("lizard_frame_hash_kernel",)}


def gpu_info():
    """Card name and power limit, read in the same run as the numbers."""
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def timed(torch, fn, steps, warmup):
    for _ in range(warmup):
        fn()
    ms = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return sum(ms) / len(ms)


def kernel_ms(torch, fn, calls=2):
    """Kernel durations by name, per call, over `calls` profiled calls (torch.profiler, CUDA activity only)."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    out = {k: 0.0 for k in KERNELS}
    for e in prof.events():
        if getattr(e.device_type, "name", "") != "CUDA":
            continue
        for k, names in KERNELS.items():
            if any(n in e.name for n in names):
                out[k] += e.time_range.elapsed_us() / 1000.0 / calls
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--levels", default="10,21,41")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--host-steps", type=int, default=1)
    ap.add_argument("--only", choices=["small", "big"], default=None)
    args = ap.parse_args()
    import torch
    import lizard_b200 as lz
    if not torch.cuda.is_available():
        raise SystemExit("frame_device_bench.py needs a CUDA device")
    L = lz.bind_frame_api(lz.lib())
    assert L.LizardB200_setDevice(0) == 0, L.LizardB200_lastError().decode()
    card = gpu_info()
    dev = torch.device("cuda", 0)
    total = 1 << 30
    h_src = torch.empty(total, dtype=torch.uint8).pin_memory()
    lz.datagen_into(h_src.data_ptr(), total, 50.0, 0)
    d_src = h_src.to(dev)
    work = [("8192x128KiB", 8192, BS), ("1x1GiB", 1, total)]
    if args.only:
        work = work[:1] if args.only == "small" else work[1:]
    rows = []
    for name, n, size in work:
        src_off = [i * size for i in range(n)]
        for level in [int(x) for x in args.levels.split(",")]:
            for checksum in (0, 1):
                p = lz.make_prefs(level, 1, True, bool(checksum), 0)
                cap = L.LizardF_compressFrameBound(size, ctypes.byref(p))
                stride = (cap + 15) // 16 * 16
                d_frames = torch.empty(n * stride, dtype=torch.uint8, device=dev)
                d_back = torch.empty(total, dtype=torch.uint8, device=dev)
                dst_off = [i * stride for i in range(n)]
                res = []

                def comp():
                    res[:] = lz.compress_frames(d_src.data_ptr(), src_off, [size] * n, d_frames.data_ptr(), dst_off, [cap] * n, p)

                c_ms = timed(torch, comp, args.steps, args.warmup)
                assert not any(L.LizardF_isError(r) for r in res), lz.frame_error(res[0])
                fsize = list(res)
                back = []

                def dec():
                    back[:] = lz.decompress_frames(d_frames.data_ptr(), dst_off, fsize, d_back.data_ptr(), src_off, [size] * n)

                d_ms = timed(torch, dec, args.steps, args.warmup)
                assert back == [size] * n, lz.frame_error(back[0])
                assert torch.equal(d_back, d_src)
                kc, kd = kernel_ms(torch, comp), kernel_ms(torch, dec)
                # the host frame API over the same frames, on pinned host buffers
                h_frames = torch.empty(n * stride, dtype=torch.uint8).pin_memory()
                h_back = torch.empty(total, dtype=torch.uint8).pin_memory()
                hc, hd = [], []
                for _ in range(args.host_steps):
                    t0 = time.perf_counter()
                    for i in range(n):
                        r = L.LizardF_compressFrame(h_frames.data_ptr() + dst_off[i], cap, h_src.data_ptr() + src_off[i], size,
                                                    ctypes.byref(p))
                        assert r == fsize[i]
                    hc.append((time.perf_counter() - t0) * 1e3)
                    t0 = time.perf_counter()
                    for i in range(n):
                        ctx = ctypes.c_void_p()
                        L.LizardF_createDecompressionContext(ctypes.byref(ctx), 100)
                        si, so = ctypes.c_size_t(fsize[i]), ctypes.c_size_t(size)
                        r = L.LizardF_decompress(ctx, h_back.data_ptr() + src_off[i], ctypes.byref(so),
                                                 h_frames.data_ptr() + dst_off[i], ctypes.byref(si), None)
                        L.LizardF_freeDecompressionContext(ctx)
                        assert r == 0 and so.value == size
                    hd.append((time.perf_counter() - t0) * 1e3)
                gib = total / (1 << 30)
                row = {"card": card, "workload": name, "level": level, "checksum": checksum,
                       "compress_ms": round(c_ms, 3), "decompress_ms": round(d_ms, 3),
                       "compress_GBps": round(total / c_ms / 1e6, 2), "decompress_GBps": round(total / d_ms / 1e6, 2),
                       "index_ms": round(kd["index"], 3), "assembly_ms": round(kc["assembly"], 3),
                       "hash_compress_ms": round(kc["hash"], 3), "hash_decompress_ms": round(kd["hash"], 3),
                       "host_compress_ms": round(min(hc), 3), "host_decompress_ms": round(min(hd), 3),
                       "ratio": round(sum(fsize) / total, 4), "GiB": gib}
                print(json.dumps(row), flush=True)
                rows.append(row)
                del d_frames, d_back, h_frames, h_back
    print(f"\n{card}")
    print(f"{'workload':>12} {'lvl':>3} {'ck':>2} {'comp ms':>9} {'dec ms':>9} {'index':>7} {'asm':>7} {'hashC':>8} {'hashD':>8}"
          f" {'hostC ms':>9} {'hostD ms':>9}")
    for r in rows:
        print(f"{r['workload']:>12} {r['level']:>3} {r['checksum']:>2} {r['compress_ms']:>9.2f} {r['decompress_ms']:>9.2f}"
              f" {r['index_ms']:>7.3f} {r['assembly_ms']:>7.3f} {r['hash_compress_ms']:>8.2f} {r['hash_decompress_ms']:>8.2f}"
              f" {r['host_compress_ms']:>9.1f} {r['host_decompress_ms']:>9.1f}")


if __name__ == "__main__":
    main()
