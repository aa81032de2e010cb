#!/usr/bin/env python
"""frame_async_bench.py -- LizardB200_decompressFramesAsync against LizardB200_decompressFrames on the same frames.
A development tool; bench.py is the contract bench.

Workloads (datagen -P50): 8192 frames of 128 KiB with the content checksum, and one frame of 1 GiB without it (one warp hashes
a frame at about 1.2 GB/s, DESIGN.md 3.4a), levels 10, 21 and 41.  For each:
- sync_ms: LizardB200_decompressFrames per call, on the side stream: CUDA events recorded on that stream before and after
  the call.  The call synchronises the stream several times, so this is the call's whole cost to its caller: its kernels
  plus the host round trips between them, during which the GPU waits;
- async_ms: LizardB200_decompressFramesAsync per call on the same stream, events around the enqueue: the device time of the
  call's work (the host is free after enqueue_ms);
- enqueue_ms: host time for the async call to return (warm, no workspace growth), the median;
- graph_ms: one replay of a CUDA graph holding the async call (events around the replay);
- pad8x_ms: the async call with maxBlocks 8 times the blocks the frames have (what the padding units cost).
Each *_ms is the mean over --steps calls after --warmup untimed ones, with the fastest and slowest call beside it
(*_range).  The card's name and power limit are read in the same run.  One JSON line per case.

  python tools/frame_async_bench.py [--levels 10,21,41] [--steps 40] [--warmup 3] [--only small|big]
"""
import argparse
import ctypes
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from frame_device_bench import gpu_info  # noqa: E402

BS = 1 << 17


def timed(torch, fn, steps, warmup):
    """(mean, fastest, slowest) ms per call, CUDA events on the current stream around each call."""
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
    return sum(ms) / len(ms), min(ms), max(ms)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--levels", default="10,21,41")
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--only", choices=["small", "big"], default=None)
    args = ap.parse_args()
    import torch
    import lizard_b200 as lz
    if not torch.cuda.is_available():
        raise SystemExit("frame_async_bench.py needs a CUDA device")
    L = lz.bind_frame_api(lz.lib())
    card = gpu_info()
    dev = torch.device("cuda", 0)
    total = 1 << 30
    h_src = torch.empty(total, dtype=torch.uint8).pin_memory()
    lz.datagen_into(h_src.data_ptr(), total, 50.0, 0)
    d_src = h_src.to(dev)
    work = [("8192x128KiB", 8192, BS), ("1x1GiB", 1, total)]
    if args.only:
        work = work[:1] if args.only == "small" else work[1:]
    s = torch.cuda.Stream()
    for name, n, size in work:
        src_off = [i * size for i in range(n)]
        for level in [int(x) for x in args.levels.split(",")]:
            p = lz.make_prefs(level, 1, True, n > 1, 0)
            cap = L.LizardF_compressFrameBound(size, ctypes.byref(p))
            stride = (cap + 15) // 16 * 16
            d_frames = torch.empty(n * stride, dtype=torch.uint8, device=dev)
            d_back = torch.empty(total, dtype=torch.uint8, device=dev)
            dst_off = [i * stride for i in range(n)]
            fsize = lz.compress_frames(d_src.data_ptr(), src_off, [size] * n, d_frames.data_ptr(), dst_off, [cap] * n, p)
            assert not any(L.LizardF_isError(r) for r in fsize), lz.frame_error(fsize[0])
            nb = total // BS
            t = {k: torch.tensor(v, dtype=torch.int64, device=dev)
                 for k, v in (("off", dst_off), ("size", fsize), ("doff", src_off), ("dcap", [size] * n))}
            res = torch.zeros(n, dtype=torch.int64, device=dev)

            def sync_call():
                lz.decompress_frames(d_frames.data_ptr(), dst_off, fsize, d_back.data_ptr(), src_off, [size] * n, s.cuda_stream)

            def async_call(max_blocks=nb):
                lz.decompress_frames_async(d_frames, t["off"], t["size"], d_back, t["doff"], t["dcap"], res, max_blocks, nb * BS)

            with torch.cuda.stream(s):
                sync_ms = timed(torch, sync_call, args.steps, args.warmup)
                d_back.zero_()
                async_ms = timed(torch, async_call, args.steps, args.warmup)
                assert torch.equal(d_back, d_src) and all(int(r) == size for r in res.cpu().tolist())
                enq = []
                for _ in range(args.steps):
                    s.synchronize()
                    t0 = time.perf_counter()
                    async_call()
                    enq.append((time.perf_counter() - t0) * 1e3)
                s.synchronize()
                pad_ms = timed(torch, lambda: async_call(8 * nb), args.steps, args.warmup)
                async_call()                                           # the graph's pointers: the workspace of this shape
                s.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=s):
                async_call()
            d_back.zero_()
            res.zero_()
            graph_ms = timed(torch, g.replay, args.steps, args.warmup)
            assert torch.equal(d_back, d_src) and all(int(r) == size for r in res.cpu().tolist())
            row = {"card": card, "workload": name, "level": level, "checksum": int(n > 1), "steps": args.steps,
                   "enqueue_ms": round(sorted(enq)[len(enq) // 2], 3), "enqueue_range": [round(min(enq), 3), round(max(enq), 3)],
                   "async_GBps": round(total / async_ms[0] / 1e6, 2)}
            for k, v in (("sync", sync_ms), ("async", async_ms), ("graph", graph_ms), ("pad8x", pad_ms)):
                row[k + "_ms"] = round(v[0], 3)
                row[k + "_range"] = [round(v[1], 3), round(v[2], 3)]
            print(json.dumps(row), flush=True)
            del g, d_frames, d_back, t, res


if __name__ == "__main__":
    main()
