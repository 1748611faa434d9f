#!/usr/bin/env python
"""Device-resident StatelessDeflate, BestSpeed, HuffmanOnly and NoCompression rates (input GB/s) and ratios on helpers.synth_text_torch text, raw and as
gzip members (BestSpeed also as zlib streams), in two shapes: --gib of text as 64 KiB inputs and as 64 MiB inputs.  Each batch is encoded whole and timed with CUDA events
(--warmup warm-ups, --steps steps, --big-steps for the 64 MiB shape; --shapes / --formats pick rows, so that the rows
can be split across runs); the
parse / encode / crc (BestSpeed: l1 / l1_check; HuffmanOnly / NoCompression: analyse / plan / emit / finish) kernels are timed with torch.profiler in a run of their own.  The device inflate of the raw output
is timed in the same session, and zlib.compress at level 1 on every host core over the same inputs is a CPU line for
context (it is zlib's level 1, not the reference's StatelessDeflate, which is Go and does not run here).  Records the card's
name and power limit.  Prints one JSON line (and writes it to --out).
usage: deflate_times.py [--gib G] [--warmup W] [--steps K] [--big-steps K] [--big-mib M] [--shapes small,big]
       [--formats raw,zlib,gzip] [--levels stateless,best_speed,huffman_only,no_compression] [--no-inflate] [--out FILE]
HuffmanOnly / NoCompression rows run with --big-mib 1024 as one 1 GiB input: those levels write every window of a member
in parallel.  (One 1 GiB member at the other two levels is one lane's work, a minute or more per call.)"""
import argparse
import json
import os
import subprocess
import sys
import time
import zlib
from concurrent.futures import ThreadPoolExecutor

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import helpers as H
from compress_b200 import flate

KERNELS = ["b2c_deflate_parse_kernel", "b2c_deflate_encode_kernel", "b2c_deflate_crc_kernel"]
KERNELS_L1 = ["b2c_deflate_l1_kernel", "b2c_deflate_l1_check_kernel"]
KERNELS_NOLZ = ["b2c_deflate_nolz_analyse_kernel", "b2c_deflate_nolz_plan_kernel", "b2c_deflate_nolz_emit_kernel",
                "b2c_deflate_nolz_finish_kernel"]
NOLZ_LEVELS = (("huffman_only", flate.HuffmanOnly), ("no_compression", flate.NoCompression))
HDR = b"\x1f\x8b\x08\x00\x00\x00\x00\x00\x00\xff"
HDR_L1 = b"\x1f\x8b\x08\x00\x00\x09\x6e\x88\x04\xff"    # XFL 4, as gzip.NewWriterLevel(w, BestSpeed) writes it


def timed(fn, warmup, steps):
    """Mean ms per call over `steps` calls, each between its own pair of events (a 64 MiB-input call runs for seconds, so
    each step reports its progress on stderr)."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    total = 0.0
    for k in range(steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        total += e0.elapsed_time(e1)
        print("step %d/%d %.1f ms" % (k + 1, steps, e0.elapsed_time(e1)), file=sys.stderr, flush=True)
    return total / steps


def kernel_ms(fn, kernels=KERNELS):
    from torch.profiler import profile, ProfilerActivity
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {k: 0.0 for k in kernels}
    for e in prof.key_averages():
        if e.key in out:
            out[e.key] = round(e.device_time_total / 1000.0, 3)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=1.0)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--big-steps", type=int, default=20)
    ap.add_argument("--big-mib", type=int, default=64)
    ap.add_argument("--shapes", default="small,big", help="small: 64 KiB inputs, big: --big-mib inputs")
    ap.add_argument("--formats", default="raw,zlib,gzip", help="zlib: not for stateless rows")
    ap.add_argument("--levels", default="stateless,best_speed")
    ap.add_argument("--no-inflate", action="store_true", help="skip the device inflate of the raw output")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dev = "cuda"
    total = int(a.gib * (1 << 30))
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    res = {"gpu": q.stdout.strip(), "gib": a.gib, "rows": []}
    src = H.synth_text_torch(total, dev)
    enc, dec = flate.Encoder(), flate.Decoder()
    shapes = [(64 << 10, a.steps, a.warmup)] if "small" in a.shapes else []
    shapes += [(a.big_mib << 20, a.big_steps, a.warmup)] if "big" in a.shapes else []
    for piece, steps, warm in shapes:
        n = total // piece
        sizes = torch.full((n,), piece, dtype=torch.int32, device=dev)
        cap = flate.StatelessBound(piece) + len(HDR) + 10
        dst = torch.empty((n, cap), dtype=torch.uint8, device=dev)
        out = torch.empty((n,), dtype=torch.int64, device=dev)
        for fmt, name, hdr in ((flate.RAW, "raw", b""), (flate.GZIP, "gzip", HDR)):
            if name not in a.formats or "stateless" not in a.levels:
                continue
            call = lambda: enc.encode_device(src, sizes, piece, dst=dst, dst_cap=cap, out_sizes=out, format=fmt, header=hdr)  # noqa: E731
            ms = timed(call, warm, steps)
            o = out.cpu()
            assert int(o.min()) > 0
            row = {"shape": "%d x %d KiB" % (n, piece >> 10), "format": name, "ms": round(ms, 3),
                   "input_GBps": round(total / ms / 1e6, 2), "ratio": round(total / int(o.sum()), 4), "steps": steps}
            if piece == 64 << 10:
                row["kernel_ms"] = kernel_ms(call)
            if fmt == flate.RAW and not a.no_inflate:
                call()
                torch.cuda.synchronize()
                comp = dst.clone()
                csz = out.to(torch.int32)
                dsz = torch.empty((n,), dtype=torch.int64, device=dev)
                back = torch.empty((n, piece), dtype=torch.uint8, device=dev)
                dcall = lambda: dec.decode_device(comp.reshape(-1), csz, cap, dst=back, dst_cap=piece, out_sizes=dsz, format=flate.RAW)  # noqa: E731
                dms = timed(dcall, 1, max(1, steps // 4))
                assert bool((dsz == piece).all()) and bool((back.reshape(-1) == src[:n * piece]).all())
                row["inflate_ms"] = round(dms, 3)
                row["inflate_output_GBps"] = round(total / dms / 1e6, 2)
            res["rows"].append(row)
            print(json.dumps(row), flush=True)
        del dst
        for lname, level in NOLZ_LEVELS:
            if lname not in a.levels:
                continue
            cap = flate.NoLZBound(level, piece) + len(HDR) + 8
            dst = torch.empty((n, cap), dtype=torch.uint8, device=dev)
            for fmt, name, hdr in ((flate.RAW, "raw", b""), (flate.ZLIB, "zlib", b""), (flate.GZIP, "gzip", HDR)):
                if name not in a.formats:
                    continue
                call = lambda: enc.nolz_device(level, src, sizes, piece, dst=dst, dst_cap=cap, out_sizes=out, format=fmt, header=hdr)  # noqa: E731
                ms = timed(call, warm, steps)
                o = out.cpu()
                assert int(o.min()) > 0
                row = {"shape": "%d x %d KiB" % (n, piece >> 10), "level": lname, "format": name, "ms": round(ms, 3),
                       "input_GBps": round(total / ms / 1e6, 2), "ratio": round(total / int(o.sum()), 4), "steps": steps,
                       "kernel_ms": kernel_ms(call, KERNELS_NOLZ)}
                res["rows"].append(row)
                print(json.dumps(row), flush=True)
            del dst
        if "best_speed" not in a.levels:
            continue
        cap = flate.BestSpeedBound(piece) + len(HDR_L1) + 8
        dst = torch.empty((n, cap), dtype=torch.uint8, device=dev)
        for fmt, name, hdr in ((flate.RAW, "raw", b""), (flate.ZLIB, "zlib", b""), (flate.GZIP, "gzip", HDR_L1)):
            if name not in a.formats:
                continue
            call = lambda: enc.best_speed_device(src, sizes, piece, dst=dst, dst_cap=cap, out_sizes=out, format=fmt, header=hdr)  # noqa: E731
            ms = timed(call, warm, steps)
            o = out.cpu()
            assert int(o.min()) > 0
            row = {"shape": "%d x %d KiB" % (n, piece >> 10), "level": "best_speed", "format": name, "ms": round(ms, 3),
                   "input_GBps": round(total / ms / 1e6, 2), "ratio": round(total / int(o.sum()), 4), "steps": steps,
                   "kernel_ms": kernel_ms(call, KERNELS_L1)}
            res["rows"].append(row)
            print(json.dumps(row), flush=True)
        del dst
    host = src[:min(total, 256 << 20)].cpu().numpy().tobytes()
    pieces = [host[i:i + (64 << 10)] for i in range(0, len(host), 64 << 10)]
    t0 = time.perf_counter()
    with ThreadPoolExecutor(os.cpu_count()) as ex:
        csum = sum(ex.map(lambda p: len(zlib.compress(p, 1)), pieces))
    dt = time.perf_counter() - t0
    res["cpu_zlib_level1"] = {"what": "Python zlib.compress level 1, 64 KiB pieces, %d host threads (not StatelessDeflate)"
                              % os.cpu_count(), "input_GBps": round(len(host) / dt / 1e9, 3),
                              "ratio": round(len(host) / csum, 4)}
    enc.close(); dec.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        open(a.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()
