#!/usr/bin/env python
"""dict_bench.py -- small records against a shared dictionary: what a dictionary buys in size, and what decoding against one
costs on the GPU.  A development tool; bench.py is the contract bench.

Workload: --records seeded JSON-like records of 1-8 KiB drawn from a fixed vocabulary, and a 64 KiB dictionary built from
sample records of another seed.  The compiled reference (oracle/_ref/liblizard_ref_parity.so) compresses every record twice:
with the dictionary (Lizard_loadDict + Lizard_compress_continue, the record in its own buffer: an external dictionary) and
without (Lizard_compress).  Reported per level: both compressed totals, and the kernel ms per call of
LizardB200_decompress_dict_device (every record against the one dictionary in device memory) and of LizardB200_decompress_device
(the records compressed without it), CUDA events around each call, the mean of --steps calls after --warmup untimed ones.
Both decodes are checked against the records.  At the levels that compress with a dictionary on the GPU (13-17, 21, 22, 34-38,
41, 42) it also times the encode side the same way: LizardB200_compress_dict_device (every record against the dictionary in
device memory) against LizardB200_compress_device (no dictionary), both checked byte for byte against the reference's streams;
a dictionary call of the first record alone (what loading the dictionary's table costs, plus one record); and
the reference's own Lizard_loadDict + Lizard_compress_continue over all records on --threads host threads (wall clock, the
best of three).  Prints one JSON line per level with the card's name and power limit, then a table.

  python tools/dict_bench.py [--records 4000] [--levels 10,17,21,36,41] [--steps 20] [--threads 8]
"""
import argparse
import ctypes
import json
import os
import random
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
STRIDE = 8192

KEYS = ["id", "name", "email", "status", "created_at", "updated_at", "tags", "score", "country", "device", "session", "plan"]
WORDS = ["alpha", "bravo", "charlie", "delta", "echo", "foxtrot", "golf", "hotel", "india", "juliet", "kilo", "lima",
         "active", "pending", "closed", "suspended", "mobile", "desktop", "tablet", "DE", "FR", "US", "JP", "BR", "premium",
         "basic", "trial", "enterprise"]


def record(rnd, size):
    out = bytearray()
    while len(out) < size:
        parts = []
        for k in rnd.sample(KEYS, rnd.randint(5, len(KEYS))):
            v = rnd.choice([str(rnd.randrange(10 ** rnd.randint(1, 9))), '"%s"' % rnd.choice(WORDS),
                            '["%s","%s","%s"]' % (rnd.choice(WORDS), rnd.choice(WORDS), rnd.choice(WORDS)),
                            '"%s@%s.example"' % (rnd.choice(WORDS), rnd.choice(WORDS))])
            parts.append('"%s":%s' % (k, v))
        out += ("{" + ",".join(parts) + "}\n").encode()
    return bytes(out[:size])


def gpu_info():
    """Card name and power limit, read in the same run as the numbers."""
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def reference():
    p = os.path.join(ROOT, "oracle", "_ref", "liblizard_ref_parity.so")
    if not os.path.exists(p):
        raise SystemExit("dict_bench.py needs oracle/_ref (built by __graft_entry__.build())")
    L = ctypes.CDLL(p)
    vp, ci = ctypes.c_void_p, ctypes.c_int
    L.Lizard_createStream.restype = vp
    L.Lizard_createStream.argtypes = [ci]
    L.Lizard_freeStream.argtypes = [vp]
    L.Lizard_loadDict.argtypes = [vp, vp, ci]
    L.Lizard_compress_continue.argtypes = [vp, vp, vp, ci, ci]
    L.Lizard_compress.argtypes = [vp, vp, ci, ci, ci]
    return L


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=int, default=4000)
    ap.add_argument("--levels", default="10,17,21,36,41")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--threads", type=int, default=8)
    args = ap.parse_args()
    import torch
    import lizard_b200 as lz
    if not torch.cuda.is_available():
        raise SystemExit("dict_bench.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    L = lz.lib()
    assert L.LizardB200_setDevice(0) == 0, L.LizardB200_lastError().decode()
    R = reference()

    rnd = random.Random(1)
    recs = [record(rnd, rnd.randint(1024, STRIDE)) for _ in range(args.records)]
    drnd = random.Random(2)
    dictionary = b"".join(record(drnd, 2048) for _ in range(32))[: 64 << 10]
    n, total = len(recs), sum(len(r) for r in recs)
    dbuf = ctypes.create_string_buffer(dictionary, len(dictionary))
    cap = STRIDE + STRIDE // 8 + 64
    out = ctypes.create_string_buffer(cap)

    # 16 bytes of slack: no record can start right behind the dictionary (that would be the prefix layout)
    d_dict = torch.frombuffer(bytearray(dictionary + bytes(16)), dtype=torch.uint8).to(dev)
    d_back = torch.empty(n * STRIDE, dtype=torch.uint8, device=dev)
    idx = torch.arange(n, dtype=torch.int64, device=dev)
    d_back_off = idx * STRIDE
    d_back_cap = torch.tensor([len(r) for r in recs], dtype=torch.int32, device=dev)
    d_dict_off = torch.zeros(n, dtype=torch.int64, device=dev)
    d_dict_len = torch.full((n,), len(dictionary), dtype=torch.int32, device=dev)
    d_res = torch.zeros(n, dtype=torch.int32, device=dev)
    want = torch.zeros(n * STRIDE, dtype=torch.uint8)
    for i, r in enumerate(recs):
        want[i * STRIDE:i * STRIDE + len(r)] = torch.frombuffer(bytearray(r), dtype=torch.uint8)
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
        return sum(ts) / len(ts)

    def upload(units):
        offs, at = [], 0
        for u in units:
            offs.append(at)
            at += len(u)
        return (torch.frombuffer(bytearray(b"".join(units)), dtype=torch.uint8).to(dev),
                torch.tensor(offs, dtype=torch.int64, device=dev), torch.tensor([len(u) for u in units], dtype=torch.int32, device=dev))

    def decoded_ok():                                          # d_back was zeroed before the calls
        return bool((d_res == d_back_cap).all()) and torch.equal(d_back.cpu(), want)

    rs, rs_off, rs_len = upload(recs)
    d_cout = torch.empty(n * cap, dtype=torch.uint8, device=dev)
    d_cout_off = idx * cap
    d_cout_cap = torch.full((n,), cap, dtype=torch.int32, device=dev)

    def encode_side(level, with_dict, plain):
        """kernel ms of the dictionary and plain encode device calls, the reference on host threads, and the byte check"""
        def dict_call():
            s = L.LizardB200_compress_dict_device(rs.data_ptr(), rs_off.data_ptr(), rs_len.data_ptr(), d_cout.data_ptr(),
                                                  d_cout_off.data_ptr(), d_cout_cap.data_ptr(), d_dict.data_ptr(),
                                                  d_dict_off.data_ptr(), d_dict_len.data_ptr(), d_res.data_ptr(), n, level, sp)
            assert s == 0, L.LizardB200_lastError()

        def plain_call():
            s = L.LizardB200_compress_device(rs.data_ptr(), rs_off.data_ptr(), rs_len.data_ptr(), d_cout.data_ptr(),
                                             d_cout_off.data_ptr(), d_cout_cap.data_ptr(), d_res.data_ptr(), n, level, sp)
            assert s == 0, L.LizardB200_lastError()

        def same(streams):
            res, o = d_res.cpu().tolist(), d_cout.cpu().numpy().tobytes()
            return all(res[i] == len(c) and o[i * cap:i * cap + res[i]] == c for i, c in enumerate(streams))

        def one_call():
            s = L.LizardB200_compress_dict_device(rs.data_ptr(), rs_off.data_ptr(), rs_len.data_ptr(), d_cout.data_ptr(),
                                                  d_cout_off.data_ptr(), d_cout_cap.data_ptr(), d_dict.data_ptr(),
                                                  d_dict_off.data_ptr(), d_dict_len.data_ptr(), d_res.data_ptr(), 1, level, sp)
            assert s == 0, L.LizardB200_lastError()

        ms_enc_one = timed(one_call)
        ms_enc_dict = timed(dict_call)
        ok = same(with_dict)
        ms_enc = timed(plain_call)
        ok = ok and same(plain)

        def ref_one(r):
            o = ctypes.create_string_buffer(cap)
            src = ctypes.create_string_buffer(r, len(r))
            st = R.Lizard_createStream(level)
            R.Lizard_loadDict(st, dbuf, len(dictionary))
            k = R.Lizard_compress_continue(st, src, o, len(r), cap)
            R.Lizard_freeStream(st)
            return k
        best = None
        with ThreadPoolExecutor(args.threads) as pool:
            for _ in range(3):
                t0 = time.perf_counter()
                list(pool.map(ref_one, recs))
                t = (time.perf_counter() - t0) * 1e3
                best = t if best is None else min(best, t)
        return {"ms_enc_dict_device": round(ms_enc_dict, 4), "ms_enc_device": round(ms_enc, 4), "ms_enc_dict_one_record": round(ms_enc_one, 4),
                "ms_enc_dict_ref_threads": round(best, 1), "threads": args.threads, "enc_ok": ok}

    gpu = gpu_info()
    rows = []
    for level in [int(x) for x in args.levels.split(",")]:
        with_dict, plain = [], []
        for r in recs:
            st = R.Lizard_createStream(level)
            R.Lizard_loadDict(st, dbuf, len(dictionary))
            src = ctypes.create_string_buffer(r, len(r))
            k = R.Lizard_compress_continue(st, src, out, len(r), cap)
            R.Lizard_freeStream(st)
            assert k > 0
            with_dict.append(out.raw[:k])
            k = R.Lizard_compress(r, out, len(r), cap, level)
            assert k > 0
            plain.append(out.raw[:k])
        ds, ds_off, ds_len = upload(with_dict)
        ps, ps_off, ps_len = upload(plain)

        def dict_call():
            s = L.LizardB200_decompress_dict_device(ds.data_ptr(), ds_off.data_ptr(), ds_len.data_ptr(), d_back.data_ptr(),
                                                    d_back_off.data_ptr(), d_back_cap.data_ptr(), d_dict.data_ptr(),
                                                    d_dict_off.data_ptr(), d_dict_len.data_ptr(), d_res.data_ptr(), n, sp)
            assert s == 0, L.LizardB200_lastError()

        def plain_call():
            s = L.LizardB200_decompress_device(ps.data_ptr(), ps_off.data_ptr(), ps_len.data_ptr(), d_back.data_ptr(),
                                               d_back_off.data_ptr(), d_back_cap.data_ptr(), d_res.data_ptr(), n, sp)
            assert s == 0, L.LizardB200_lastError()

        d_back.zero_()
        ms_dict = timed(dict_call)
        ok_dict = decoded_ok()
        d_back.zero_()
        ms_plain = timed(plain_call)
        ok_plain = decoded_ok()
        rec = {"level": level, "records": n, "bytes": total, "dict_bytes": len(dictionary),
               "compressed_with_dict": sum(map(len, with_dict)), "compressed_without": sum(map(len, plain)),
               "ms_dict_device": round(ms_dict, 4), "ms_device": round(ms_plain, 4), "ok": ok_dict and ok_plain, "gpu": gpu}
        if 13 <= level <= 17 or 34 <= level <= 38 or level in (21, 22, 41, 42):
            rec.update(encode_side(level, with_dict, plain))
            rec["ok"] = rec["ok"] and rec.pop("enc_ok")
        print(json.dumps(rec), flush=True)
        rows.append(rec)
    print(f"\n{gpu}; {n} records, {total} bytes, 64 KiB dictionary; mean of {args.steps} calls")
    print(f"{'level':>5} {'with dict':>10} {'without':>10} {'ms dict':>8} {'ms plain':>9} {'ok':>4}")
    for r in rows:
        print(f"{r['level']:>5} {r['compressed_with_dict']:>10} {r['compressed_without']:>10} {r['ms_dict_device']:>8} "
              f"{r['ms_device']:>9} {str(r['ok']):>4}")
    enc = [r for r in rows if "ms_enc_dict_device" in r]
    if enc:
        print(f"\nencode: kernel ms per call on the GPU, wall ms of the reference on {args.threads} host threads")
        print(f"{'level':>5} {'ms dict':>8} {'ms plain':>9} {'ms 1 record':>12} {'ms ref dict':>12}")
        for r in enc:
            print(f"{r['level']:>5} {r['ms_enc_dict_device']:>8} {r['ms_enc_device']:>9} {r['ms_enc_dict_one_record']:>12} "
                  f"{r['ms_enc_dict_ref_threads']:>12}")
    if not all(r["ok"] for r in rows):
        raise SystemExit("a decode returned wrong bytes")


if __name__ == "__main__":
    main()
