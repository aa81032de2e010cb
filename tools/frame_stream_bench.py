#!/usr/bin/env python
"""frame_stream_bench.py -- LizardB200_decompressStream on 1 GiB frames fed in chunks.  A development tool; bench.py is the
contract bench.

Workloads: 1 GiB of datagen -P50 at levels 10, 21 and 41, as one frame of 128 KiB blocks and as one frame of 4 MiB blocks (the
CLI's default), with and without the content checksum, fed in chunks of 4, 16, 64 and 256 MiB into a 1 GiB output.  For each:
- stream_ms_per_gib: the whole frame through one DecompressionStream, CUDA events around the calls (the calls synchronise
  their stream, so this is the device time plus the host's share between the calls);
- call_ms: host time per call, the mean;
- frames_ms: the same frame through LizardB200_decompressFrames as one whole frame (events around the call);
- host_ms: the same frame through the host LizardF_decompress, from and to pinned host buffers, in the same chunks.
Each figure is the mean of --steps runs after --warmup untimed ones.  The card's name and power limit are read in the same
run.  One JSON line per case.

  python tools/frame_stream_bench.py [--levels 10,21,41] [--chunks 4,16,64,256] [--steps 3] [--warmup 1]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--levels", default="10,21,41")
    ap.add_argument("--chunks", default="4,16,64,256")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--size", type=int, default=GIB)
    args = ap.parse_args()
    import torch
    import lizard_b200 as lz
    if not torch.cuda.is_available():
        raise SystemExit("frame_stream_bench.py needs a CUDA device")
    L = lz.bind_frame_api(lz.lib())
    card = gpu_info()
    n = args.size
    data = torch.empty(n, dtype=torch.uint8).pin_memory()
    lz.datagen_into(data.data_ptr(), n, 50.0, 0)
    d_out = torch.empty(n, dtype=torch.uint8, device="cuda")
    h_out = torch.empty(n, dtype=torch.uint8).pin_memory()
    src_bytes = bytes(data.numpy())

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
        for bsid in (1, 4):
            for checksum in (False, True):
                frame = lz.frame_compress(L, src_bytes, lz.make_prefs(level, block_id=bsid, checksum=checksum))
                h_src = torch.frombuffer(bytearray(frame), dtype=torch.uint8).pin_memory()
                d_src = h_src.cuda()
                frames_ms = mean(lambda: events(lambda: lz.decompress_frames(d_src.data_ptr(), [0], [len(frame)], d_out.data_ptr(), [0], [n],
                                                                             stream=torch.cuda.current_stream().cuda_stream)))
                for chunk_mib in [int(x) for x in args.chunks.split(",")]:
                    chunk = chunk_mib << 20
                    calls = []

                    def stream_run():
                        pos = made = 0
                        with lz.DecompressionStream() as s:
                            while pos < len(frame):
                                t = time.perf_counter()
                                r, u, m = s.decompress(d_src.data_ptr() + pos, min(chunk, len(frame) - pos), d_out.data_ptr() + made,
                                                       n - made, stream=torch.cuda.current_stream().cuda_stream)
                                calls.append(time.perf_counter() - t)
                                assert not L.LizardF_isError(r), lz.frame_error(r)
                                pos += u
                                made += m
                        assert made == n

                    stream_ms = mean(lambda: events(stream_run))
                    assert torch.equal(d_out[:4096].cpu(), data[:4096]) and torch.equal(d_out[-4096:].cpu(), data[-4096:])

                    def host_run():
                        t = time.perf_counter()
                        ctx = ctypes.c_void_p()
                        L.LizardF_createDecompressionContext(ctypes.byref(ctx), 100)
                        pos = made = 0
                        while pos < len(frame):
                            si, so = ctypes.c_size_t(min(chunk, len(frame) - pos)), ctypes.c_size_t(n - made)
                            r = L.LizardF_decompress(ctx, h_out.data_ptr() + made, ctypes.byref(so), h_src.data_ptr() + pos,
                                                     ctypes.byref(si), None)
                            assert not L.LizardF_isError(r)
                            pos += si.value
                            made += so.value
                        L.LizardF_freeDecompressionContext(ctx)
                        return (time.perf_counter() - t) * 1e3

                    host_ms = mean(host_run)
                    print(json.dumps({
                        "card": card, "level": level, "block_kib": (128 if bsid == 1 else 4096), "checksum": checksum,
                        "chunk_mib": chunk_mib, "frame_bytes": len(frame),
                        "stream_ms_per_gib": round(stream_ms * GIB / n, 2), "call_ms": round(1e3 * sum(calls) / len(calls), 3),
                        "calls": len(calls) // (args.steps + args.warmup),
                        "frames_ms_per_gib": round(frames_ms * GIB / n, 2), "host_ms_per_gib": round(host_ms * GIB / n, 2)}),
                        flush=True)


if __name__ == "__main__":
    main()
