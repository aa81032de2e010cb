#!/usr/bin/env python
"""frame_compress_async_bench.py -- LizardB200_compressFramesAsync against LizardB200_compressFrames on the same inputs.
A development tool; bench.py is the contract bench.

Workloads (datagen -P50): 8192 inputs of 128 KiB compressed into frames with the content checksum, and one input of 1 GiB
without it (one warp hashes a frame at about 1.2 GB/s, DESIGN.md 3.4a), levels 10, 21 and 41.  For each:
- sync_ms: LizardB200_compressFrames per call, on the side stream: CUDA events recorded on that stream before and after the
  call.  The call builds its tables on the host, copies them up and reads the frame sizes back, so this is the call's whole
  cost to its caller;
- async_ms: LizardB200_compressFramesAsync per call on the same stream, events around the enqueue: the device time of the
  call's work (the host is free after enqueue_ms);
- enqueue_ms: host time for the async call to return (warm, no workspace growth), the median;
- graph_ms: one replay of a CUDA graph holding the async call (events around the replay);
- pad8x_ms: the async call with maxBlocks 8 times the blocks the inputs have (what the padding entries cost).
Each *_ms is the mean over --steps calls after --warmup untimed ones, with the fastest and slowest call beside it
(*_range).  The async frames are checked against the sync ones, byte for byte.  The card's name and power limit are read in
the same run.  One JSON line per case.

  python tools/frame_compress_async_bench.py [--levels 10,21,41] [--steps 40] [--warmup 3] [--only small|big]
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
from frame_async_bench import timed  # noqa: E402
from frame_device_bench import gpu_info  # noqa: E402

BS = 1 << 17


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
        raise SystemExit("frame_compress_async_bench.py needs a CUDA device")
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
            d_sync = torch.empty(n * stride, dtype=torch.uint8, device=dev)
            d_frames = torch.empty(n * stride, dtype=torch.uint8, device=dev)
            dst_off = [i * stride for i in range(n)]
            nb = total // BS
            t = {k: torch.tensor(v, dtype=torch.int64, device=dev)
                 for k, v in (("off", src_off), ("size", [size] * n), ("doff", dst_off), ("dcap", [cap] * n))}
            res = torch.zeros(n, dtype=torch.int64, device=dev)
            fsize = []

            def sync_call():
                fsize[:] = lz.compress_frames(d_src.data_ptr(), src_off, [size] * n, d_sync.data_ptr(), dst_off, [cap] * n, p,
                                              s.cuda_stream)

            def async_call(max_blocks=nb):
                lz.compress_frames_async(d_src, t["off"], t["size"], d_frames, t["doff"], t["dcap"], res, p, max_blocks, total)

            def same():
                got = [int(r) for r in res.cpu().tolist()]
                if got != fsize or any(L.LizardF_isError(r) for r in got):
                    return False
                a, b = d_frames.view(n, stride), d_sync.view(n, stride)
                return all(torch.equal(a[i, :fsize[i]], b[i, :fsize[i]]) for i in range(n))

            with torch.cuda.stream(s):
                sync_ms = timed(torch, sync_call, args.steps, args.warmup)
                async_ms = timed(torch, async_call, args.steps, args.warmup)
                s.synchronize()
                assert same(), "async frames differ from compressFrames"
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
            d_frames.zero_()
            res.zero_()
            graph_ms = timed(torch, g.replay, args.steps, args.warmup)
            torch.cuda.synchronize()
            assert same(), "graph replay frames differ from compressFrames"
            row = {"card": card, "workload": name, "level": level, "checksum": int(n > 1), "steps": args.steps,
                   "enqueue_ms": round(sorted(enq)[len(enq) // 2], 3), "enqueue_range": [round(min(enq), 3), round(max(enq), 3)],
                   "async_GBps": round(total / async_ms[0] / 1e6, 2)}
            for k, v in (("sync", sync_ms), ("async", async_ms), ("graph", graph_ms), ("pad8x", pad_ms)):
                row[k + "_ms"] = round(v[0], 3)
                row[k + "_range"] = [round(v[1], 3), round(v[2], 3)]
            print(json.dumps(row), flush=True)
            del g, d_sync, d_frames, t, res


if __name__ == "__main__":
    main()
