#!/usr/bin/env python
"""Wall time of each pointer-table call through the C ABI, from pageable host buffers to pageable host buffers: zstd
decode, S2 block encode and decode, LZ4 -> S2 conversion, inflate (gzip members of stored blocks, so that the copies and
not the serial walk dominate), stateless deflate, huff0 compress and decompress.  256 MiB of synthetic text in 4 096 x 64 KiB
pieces and in 64 x 4 MiB pieces (S2 encode and huff0 take 64 KiB pieces only).  Each call runs --warmup times, then --reps
times (3 times for a call that takes over a second); the median and the spread (min, max) are reported in ms.  Loads the
library named by B2C_LIB (default: the package's build), so that two builds can be timed alternately in one session.
Prints one JSON line (and writes it to --out).
usage: host_batch_times.py [--reps R] [--warmup W] [--out FILE]"""
import argparse
import ctypes
import json
import os
import sys
import time
import zlib
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import bench
import helpers as H
import lz4_util
from compress_b200._lib import lib, check, Context, PointerTable, LIB_PATH

TOTAL = 256 << 20


def _gzip_stored(data):
    c = zlib.compressobj(0, zlib.DEFLATED, 31)
    return c.compress(data) + c.flush()


def timed(fn, warmup, reps):
    for _ in range(warmup):
        t0 = time.perf_counter()
        fn()
    if time.perf_counter() - t0 > 1.0:  # the seconds-long calls (4 MiB stateless deflate, one lane per input): 3 runs
        reps = 3
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()                        # every pointer-table call synchronises before it returns
        ts.append((time.perf_counter() - t0) * 1e3)
    ts.sort()
    return {"ms": round(ts[len(ts) // 2], 3), "min": round(ts[0], 3), "max": round(ts[-1], 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    ctx = Context(0, 4096)
    c = ctx._ctx
    text = H.synth_text(TOTAL, 21)
    res = {"metric": "host_batch_times", "lib": LIB_PATH, "gpu": bench.gpu_identity(0), "warmup": a.warmup, "reps": a.reps}

    def call(fn, pre, blobs, caps, post=()):
        """One timed call: -> (timing, outputs) with the outputs of the last run."""
        t = PointerTable(blobs, caps)
        extra = [(ctypes.c_int64 * t.n)()] if post == "lz4" else []
        if fn is lib.b2c_flate_stateless_chunks:
            args = (c, 0, 0, t.srcs, t.ssz, None, None, None, None, 0, t.dsts, t.dcap, t.res, None, None, t.n)
        else:
            args = (c, *pre, t.srcs, t.ssz, t.dsts, t.dcap, t.res, *extra, t.n)
        r = timed(lambda: check(fn(*args), c), a.warmup, a.reps)
        outs, codes = t.results()
        assert all(x >= 0 for x in codes), fn.__name__
        return r, outs

    for piece in (64 << 10, 4 << 20):
        n = TOTAL // piece
        data = [text[i * piece:(i + 1) * piece] for i in range(n)]
        shape = "%dx%dk" % (n, piece >> 10)
        r = {}
        if piece == 64 << 10:
            t = PointerTable(data, [lib.b2c_zstd_bound(piece, 1) + 16] * n)
            check(lib.b2c_zstd_encode_chunks(c, 1, 3, t.srcs, t.ssz, t.dsts, t.dcap, t.res, t.n), c)
        else:
            t = PointerTable(data, [lib.b2c_zstd_frame_bound(piece, 1) + 16] * n)
            check(lib.b2c_zstd_encode_frames(c, 1, 1, t.srcs, t.ssz, t.dsts, t.dcap, t.res, t.n), c)
        frames = t.results()[0]
        r["zstd_decode"], _ = call(lib.b2c_zstd_decode_chunks, (), frames, [piece] * n)
        if piece == 64 << 10:
            r["s2_encode"], s2b = call(lib.b2c_s2_encode_chunks, (1, 0), data, [lib.b2c_s2_bound(piece) + 16] * n)
            r["s2_decode"], _ = call(lib.b2c_s2_decode_chunks, (), s2b, [piece] * n)
            r["huf_compress"], hc = call(lib.b2c_huf_compress_chunks, (1,), data, [piece + 16] * n)
            r["huf_decompress"], _ = call(lib.b2c_huf_decompress_chunks, (1,), hc, [piece] * n)
        with ThreadPoolExecutor(8) as ex:
            lz4 = list(ex.map(lz4_util.compress, data))
            gz = list(ex.map(_gzip_stored, data))
        r["lz4_convert"], _ = call(lib.b2c_s2_convert_lz4_chunks, (0, 0), lz4, [piece + piece // 4 + 64] * n, post="lz4")
        r["inflate_stored"], _ = call(lib.b2c_flate_decode_chunks, (2, 0), gz, [piece] * n)
        r["stateless_deflate"], _ = call(lib.b2c_flate_stateless_chunks, (), data, [piece + piece // 8 + 4096] * n)
        for k, v in r.items():
            v["GBps"] = round(TOTAL / v["ms"] / 1e6, 2)
        res[shape] = r
        print(shape, r, flush=True)
    ctx.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
