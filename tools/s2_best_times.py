#!/usr/bin/env python
"""Device-resident S2 / Snappy block encode rates of the three levels (fast / better / best) on bench.py's text, in one
session on one card: 1 GiB (--gib) of bench.make_data in 64 KiB blocks, the whole batch timed with CUDA events (3 warm-ups,
20 steps), output bytes and ratio per level, and the parse kernel's time from torch.profiler in a run of its own (so
`kernel_ms` and `ms` come from different runs, and the first can come out slightly larger than the second).  The card's
name and power limit are recorded with the numbers.  Prints one JSON line (and writes it to --out).
usage: s2_best_times.py [--gib G] [--out FILE]"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import bench
from compress_b200 import s2

WARMUP, STEPS = 3, 20
KERNELS = {("fast", False): "b2c_lz_s2_fast_kernel", ("fast", True): "b2c_lz_snappy_fast_kernel",
           ("better", False): "b2c_lz_s2_better_kernel", ("better", True): "b2c_lz_snappy_better_kernel",
           ("best", False): "b2c_lz_s2_best_kernel", ("best", True): "b2c_lz_snappy_best_kernel"}


def timed(fn):
    for _ in range(WARMUP):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(STEPS):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / STEPS


def kernel_ms(fn, name):
    from torch.profiler import profile, ProfilerActivity
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
    return round(sum(ev.device_time for ev in prof.events() if ev.name == name) / 3000.0, 3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=1.0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    nbytes = int(a.gib * (1 << 30)) // 65536 * 65536
    src = bench.make_data(nbytes, dev, 0)
    codec = s2.Codec()
    n = nbytes // 65536
    dst = torch.empty((n, s2.SLOT), dtype=torch.uint8, device=dev)
    outs = torch.empty(n, dtype=torch.int64, device=dev)
    res = {"metric": "s2_encode_levels", "content_bytes": nbytes, "block": 65536, "gpu": bench.gpu_identity(0),
           "warmup": WARMUP, "steps": STEPS}
    for level in ("fast", "better", "best"):
        for snappy in (False, True):
            fn = lambda: codec.encode_device(src, snappy=snappy, dst=dst, out_sizes=outs, better=level == "better",
                                             best=level == "best")
            ms = timed(fn)
            o = outs.cpu()
            assert bool((o > 0).all()), "encode failed"
            key = "%s_%s" % ("snappy" if snappy else "s2", level)
            r = {"ms": round(ms, 3), "GBps": round(nbytes / ms / 1e6, 2), "out_bytes": int(o.sum()),
                 "ratio": round(float(o.sum()) / nbytes, 4), "kernel_ms": kernel_ms(fn, KERNELS[(level, snappy)])}
            res[key] = r
            print(key, r, flush=True)
    codec.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
