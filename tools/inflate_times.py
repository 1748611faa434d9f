#!/usr/bin/env python
"""Device-resident inflate rates (output GB/s) on bench.py's text, with the zstd and S2 decode of the same content and a
CPU zlib line.  --gib of helpers.synth_text_torch text is cut into 64 KiB pieces (and 4 MiB pieces) and compressed on the
host with Python's zlib on a thread pool: gzip members at levels 1, 6, 9 and 0 (stored), raw DEFLATE at level 6, and 4 MiB
gzip members at level 6.  Each batch is decoded whole, timed with CUDA events (3 warm-ups, 10 steps); the walk / exec /
checksum kernels are timed with torch.profiler in a run of their own.  The 4 MiB row runs one lane per 4 MiB stream for
seconds per call: one warm-up and one timed step, no profiler run.  zlib.decompress on every host core over the same
streams is the CPU line.  Prints one JSON line (and writes it to --out).
--shapes picks rows (the GPU calls of a shared machine are time-limited, so the rows can be split across runs) and
--other adds the zstd / S2 rows.
usage: inflate_times.py [--gib G] [--shapes K1,K2,...] [--other] [--out FILE]"""
import argparse
import json
import os
import sys
import time
import zlib
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import bench
import helpers as H
from compress_b200 import flate, s2, zstd

WARMUP, STEPS = 3, 10
KERNELS = ["b2c_inflate_walk_kernel", "b2c_inflate_exec_kernel", "b2c_inflate_check_kernel"]


def timed(fn, warmup=WARMUP, steps=STEPS):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def kernel_ms(fn, names):
    from torch.profiler import profile, ProfilerActivity
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
    tot = {k: 0.0 for k in names}
    for ev in prof.events():
        if ev.name in tot:
            tot[ev.name] += ev.device_time / 1000.0
    return {k: round(v / 3, 4) for k, v in tot.items()}


def packed(blobs, dev):
    stride = (max(len(b) for b in blobs) + 15) // 16 * 16
    src = np.zeros(len(blobs) * stride, dtype=np.uint8)
    for i, b in enumerate(blobs):
        src[i * stride:i * stride + len(b)] = np.frombuffer(b, dtype=np.uint8)
    return torch.from_numpy(src).to(dev), torch.tensor([len(b) for b in blobs], dtype=torch.int32, device=dev), stride


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=1.0)
    ap.add_argument("--shapes", default="")
    ap.add_argument("--other", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    nbytes = int(a.gib * (1 << 30))
    content = H.synth_text_torch(nbytes, dev).cpu().numpy().tobytes()
    ncpu = os.cpu_count() or 1
    res = {"metric": "inflate", "content_bytes": nbytes, "gpu": bench.gpu_identity(0), "warmup": WARMUP, "steps": STEPS,
           "host_cores": ncpu}
    dec = flate.Decoder()
    shapes = [("gzip_L1_64k", 1 << 16, 1, 31), ("gzip_L6_64k", 1 << 16, 6, 31), ("gzip_L9_64k", 1 << 16, 9, 31),
              ("gzip_L0_64k", 1 << 16, 0, 31), ("raw_L6_64k", 1 << 16, 6, -15), ("gzip_L6_4m", 4 << 20, 6, 31)]
    if a.shapes:
        shapes = [x for x in shapes if x[0] in a.shapes.split(",")]
    for key, block, level, wbits in shapes:
        n = nbytes // block
        pieces = [content[i * block:(i + 1) * block] for i in range(n)]

        def comp(p):
            c = zlib.compressobj(level, zlib.DEFLATED, wbits)
            return c.compress(p) + c.flush()
        with ThreadPoolExecutor(ncpu) as ex:
            blobs = list(ex.map(comp, pieces))
        d_src, sizes, stride = packed(blobs, dev)
        dst = torch.empty((n, block), dtype=torch.uint8, device=dev)
        outs = torch.empty(n, dtype=torch.int64, device=dev)
        fmt = flate.GZIP if wbits > 15 else flate.RAW
        fn = lambda: dec.decode_device(d_src, sizes, stride, dst=dst, dst_cap=block, out_sizes=outs, format=fmt)
        long_lane = block > (1 << 16)            # one lane per 4 MiB stream: seconds per call, so one warm-up and one step
        ms = timed(fn, 1, 1) if long_lane else timed(fn)
        assert (outs.cpu().numpy() == block).all(), "inflate failed"
        assert dst[0].cpu().numpy().tobytes() == pieces[0] and dst[n - 1].cpu().numpy().tobytes() == pieces[n - 1]
        comp_bytes = sum(len(b) for b in blobs)
        r = {"n": n, "ms": round(ms, 3), "GBps": round(n * block / ms / 1e6, 2), "in_bytes": comp_bytes}
        if not long_lane:
            r.update(kernel_ms(fn, KERNELS))
        # CPU line: zlib.decompress of the same streams on every host core
        t0 = time.perf_counter()
        with ThreadPoolExecutor(ncpu) as ex:
            list(ex.map(lambda b: zlib.decompress(b, wbits), blobs))
        r["cpu_zlib_GBps"] = round(n * block / (time.perf_counter() - t0) / 1e9, 2)
        res[key] = r
        print(key, r, flush=True)
        del d_src, dst
        torch.cuda.empty_cache()
    dec.close()
    # zstd (level 1, 64 KiB frames) and S2 (64 KiB blocks) decode of the same content, device-resident
    if a.other:
        try:
            other_decoders(res, content, nbytes, dev)
        except Exception as e:                 # the inflate rows above stand on their own
            res["other_decoders_error"] = repr(e)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


def other_decoders(res, content, nbytes, dev):
    B = 1 << 16
    n = nbytes // B
    src = torch.frombuffer(bytearray(content[:n * B]), dtype=torch.uint8).to(dev)
    enc = zstd.Encoder(level=1, max_chunks=64)
    zd, zs = enc.encode_device(src)
    torch.cuda.synchronize()
    zdec = zstd.Decoder()
    zdst = torch.empty(n * B, dtype=torch.uint8, device=dev)
    zres = torch.empty(n, dtype=torch.int64, device=dev)
    zsz = zs.to(torch.int32)
    fn = lambda: zdec.decode_device(zd, zsz, src_stride=zd.shape[1], dst=zdst, dst_cap=B, out_sizes=zres)
    ms = timed(fn)
    assert (zres.cpu().numpy() == B).all()
    res["zstd_L1_decode_64k"] = {"ms": round(ms, 3), "GBps": round(n * B / ms / 1e6, 2)}
    codec = s2.Codec()
    sd, ss = codec.encode_device(src)
    torch.cuda.synchronize()
    sdst = torch.empty((n, B), dtype=torch.uint8, device=dev)
    sres = torch.empty(n, dtype=torch.int64, device=dev)
    ssz = ss.to(torch.int32)
    fn = lambda: codec.decode_device(sd, ssz, sd.shape[1], dst=sdst, dst_cap=B, out_sizes=sres)
    ms = timed(fn)
    assert (sres.cpu().numpy() == B).all()
    res["s2_decode_64k"] = {"ms": round(ms, 3), "GBps": round(n * B / ms / 1e6, 2)}

if __name__ == "__main__":
    main()
