#!/usr/bin/env python
"""frame_compress_stream_bench.py -- LizardB200_compressStream* on 1 GiB fed in chunks.  A development tool; bench.py is the
contract bench.

Workloads: 1 GiB of datagen -P50 at levels 10, 21 and 41, into one frame of 128 KiB blocks or of 4 MiB blocks, with and without the
content checksum, fed in chunks of 4, 16, 64 and 256 MiB (--blocks, --levels, --chunks, --checksum choose a subset).  For each:
- stream_ms_per_gib: Begin, the Updates, End of one CompressionStream, enqueue-only with the results in device memory, CUDA
  events around all the calls;
- enqueue_ms: host time from the first call until the last call returns (timed runs only, not the warm-up that grows the
  buffers);
- async_ms_per_gib: one LizardB200_compressFramesAsync call over the whole input into one frame (events around the call);
- host_ms_per_gib: the host LizardF_compressBegin / Update / End from and to pinned host buffers, in the same chunks.
Each figure is the mean of --steps runs after --warmup untimed ones.  The card's name and power limit are read in the same run.
One JSON line per case.

  python tools/frame_compress_stream_bench.py [--levels 10,21,41] [--blocks 128,4096] [--chunks 4,16,64,256] [--checksum 0,1]
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

GIB = 1 << 30
BSID = {128: 1, 4096: 4}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--levels", default="10,21,41")
    ap.add_argument("--blocks", default="128,4096")
    ap.add_argument("--chunks", default="4,16,64,256")
    ap.add_argument("--checksum", default="0,1")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--size", type=int, default=GIB)
    args = ap.parse_args()
    import torch
    import lizard_b200 as lz
    if not torch.cuda.is_available():
        raise SystemExit("frame_compress_stream_bench.py needs a CUDA device")
    L = lz.bind_frame_api(lz.lib())
    card = gpu_info()
    n = args.size
    h_src = torch.empty(n, dtype=torch.uint8).pin_memory()
    lz.datagen_into(h_src.data_ptr(), n, 50.0, 0)
    d_src = h_src.cuda()
    s = torch.cuda.current_stream()

    def events(fn):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        return a.elapsed_time(b)

    def mean(fn):
        for _ in range(args.warmup):
            fn()
        return sum(fn() for _ in range(args.steps)) / args.steps

    for level in [int(x) for x in args.levels.split(",")]:
        for kib in [int(x) for x in args.blocks.split(",")]:
            for checksum in [x == "1" for x in args.checksum.split(",")]:
                p = lz.make_prefs(level, block_id=BSID[kib], checksum=checksum)
                frame_cap = L.LizardF_compressFrameBound(n, ctypes.byref(p))
                d_frame = torch.empty(frame_cap, dtype=torch.uint8, device="cuda")
                tab = torch.tensor([0, n, 0, frame_cap, 0], dtype=torch.int64, device="cuda")
                blocks = -(-n // (kib << 10))
                async_ms = mean(lambda: events(lambda: lz.compress_frames_async(
                    d_src, tab[0:1], tab[1:2], d_frame, tab[2:3], tab[3:4], tab[4:5], p, blocks, 1 << 62, stream=s.cuda_stream)))
                h_dst = torch.empty(frame_cap, dtype=torch.uint8).pin_memory()
                for chunk_mib in [int(x) for x in args.chunks.split(",")]:
                    chunk = chunk_mib << 20
                    k = -(-n // chunk)
                    cap = L.LizardF_compressBound(chunk, ctypes.byref(p))
                    d_out = torch.empty(64 + (k + 1) * cap, dtype=torch.uint8, device="cuda")
                    written = torch.zeros(k + 2, dtype=torch.int64, device="cuda")
                    host_t = []

                    with lz.CompressionStream() as cs:
                        def stream_run():
                            t = time.perf_counter()
                            base = d_out.data_ptr()
                            cs.begin(base, 15, p, written[0:1], s.cuda_stream)
                            for i in range(k):
                                m = min(chunk, n - i * chunk)
                                cs.update(d_src.data_ptr() + i * chunk, m, base + 64 + i * cap, cap, written[i + 1:i + 2], s.cuda_stream)
                            cs.end(base + 64 + k * cap, cap, written[k + 1:k + 2], s.cuda_stream)
                            host_t.append(time.perf_counter() - t)

                        for _ in range(args.warmup):                      # the first run grows the buffers, which synchronises
                            stream_run()
                        s.synchronize()
                        host_t.clear()
                        stream_ms = sum(events(stream_run) for _ in range(args.steps)) / args.steps
                    total = int(written.sum().item())
                    assert not any(L.LizardF_isError(int(w) & ((1 << 64) - 1)) for w in written.tolist())

                    def host_run():
                        t = time.perf_counter()
                        ctx = ctypes.c_void_p()
                        L.LizardF_createCompressionContext(ctypes.byref(ctx), 100)
                        o = L.LizardF_compressBegin(ctx, h_dst.data_ptr(), 15, ctypes.byref(p))
                        for i in range(k):
                            m = min(chunk, n - i * chunk)
                            r = L.LizardF_compressUpdate(ctx, h_dst.data_ptr() + o, frame_cap - o, h_src.data_ptr() + i * chunk, m, None)
                            assert not L.LizardF_isError(r)
                            o += r
                        r = L.LizardF_compressEnd(ctx, h_dst.data_ptr() + o, frame_cap - o, None)
                        assert not L.LizardF_isError(r)
                        L.LizardF_freeCompressionContext(ctx)
                        return (time.perf_counter() - t) * 1e3, o + r

                    host_ms = mean(lambda: host_run()[0])
                    assert host_run()[1] == total
                    print(json.dumps({
                        "card": card, "level": level, "block_kib": kib, "checksum": checksum, "chunk_mib": chunk_mib,
                        "frame_bytes": total, "stream_ms_per_gib": round(stream_ms * GIB / n, 2),
                        "enqueue_ms": round(1e3 * sum(host_t) / len(host_t), 3),
                        "async_ms_per_gib": round(async_ms * GIB / n, 2), "host_ms_per_gib": round(host_ms * GIB / n, 2)}),
                        flush=True)


if __name__ == "__main__":
    main()
