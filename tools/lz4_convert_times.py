#!/usr/bin/env python
"""Device-resident LZ4 / LZ4s -> S2 / Snappy block conversion rates on bench.py's text, with the S2 block decode of the same
content as the yardstick.  1 GiB (--gib) of bench.make_data is cut into 64 KiB and 4 MiB blocks and compressed on the host by
the oracle's lz4ref restatement; the conversion of the whole batch is timed with CUDA events (3 warm-ups, 20 steps) and the
walk / emit kernels with torch.profiler in a run of their own.  Prints one JSON line (and writes it to --out).
usage: lz4_convert_times.py [--gib G] [--out FILE]"""
import argparse
import json
import os
import sys
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import bench
import lz4_util as U
from compress_b200 import s2

WARMUP, STEPS = 3, 20


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


def kernel_ms(fn, names):
    from torch.profiler import profile, ProfilerActivity
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            fn()
        torch.cuda.synchronize()
    tot = {k: 0.0 for k in names}
    for ev in prof.events():
        for k in names:
            if ev.name == k:
                tot[k] += ev.device_time / 1000.0
    return {k: round(v / 5, 4) for k, v in tot.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=1.0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    nbytes = int(a.gib * (1 << 30))
    content = bench.make_data(nbytes, dev, 0).cpu().numpy().tobytes()
    codec = s2.Codec()
    res = {"metric": "lz4_convert", "content_bytes": nbytes, "gpu": bench.gpu_identity(0), "warmup": WARMUP, "steps": STEPS}
    # s2.Encode of the content (64 KiB blocks, the device encoder's block size) for the size comparison
    B64 = 1 << 16
    n64 = nbytes // B64
    _, enc_sizes = codec.encode_device(torch.frombuffer(bytearray(content[:n64 * B64]), dtype=torch.uint8).to(dev))
    torch.cuda.synchronize()
    s2_encode_bytes = int(enc_sizes.sum())
    res["s2_encode_bytes_64k"] = s2_encode_bytes
    for block in (B64, 4 << 20):
        n = nbytes // block
        pieces = [content[i * block:(i + 1) * block] for i in range(n)]
        for lz4s in (False, True):
            with ThreadPoolExecutor(8) as ex:
                blocks = list(ex.map(lambda p: U.compress(p, lz4s), pieces))
            stride = (max(len(b) for b in blocks) + 15) // 16 * 16
            src = np.zeros(n * stride, dtype=np.uint8)
            for i, b in enumerate(blocks):
                src[i * stride:i * stride + len(b)] = np.frombuffer(b, dtype=np.uint8)
            d_src = torch.from_numpy(src).to(dev)
            sizes = torch.tensor([len(b) for b in blocks], dtype=torch.int32, device=dev)
            cap = block + block // 4 + 64
            dst = torch.empty((n, cap), dtype=torch.uint8, device=dev)
            outs = torch.empty(n, dtype=torch.int64, device=dev)
            dec = torch.empty(n, dtype=torch.int64, device=dev)
            lz4_bytes = sum(len(b) for b in blocks)
            for snappy in (False, True):
                fn = lambda: codec.convert_lz4_device(d_src, sizes, stride, lz4s=lz4s, snappy=snappy, dst=dst, dst_cap=cap,
                                                      out_sizes=outs, decoded=dec)
                ms = timed(fn)
                o, nd = outs.cpu().numpy(), dec.cpu().numpy()
                assert (o > 0).all() and (nd == block).all(), "conversion failed"
                key = "%s_%s_%dk" % ("lz4s" if lz4s else "lz4", "snappy" if snappy else "s2", block >> 10)
                r = {"ms": round(ms, 3), "GBps": round(nbytes / ms / 1e6, 2), "out_bytes": int(o.sum()), "lz4_bytes": lz4_bytes,
                     "vs_lz4": round(float(o.sum()) / lz4_bytes, 4), "vs_s2_encode": round(float(o.sum()) / s2_encode_bytes, 4)}
                r.update(kernel_ms(fn, ["b2c_lz4_cvt_walk_kernel", "b2c_lz4_cvt_emit_kernel"]))
                # yardstick: S2 block decode of the same content (the converted blocks), staged kernels where they apply
                if not snappy and not lz4s:
                    dd = torch.empty((n, block), dtype=torch.uint8, device=dev)
                    dres = torch.empty(n, dtype=torch.int64, device=dev)
                    ssz = outs.to(torch.int32)
                    dfn = lambda: codec.decode_device(dst, ssz, cap, dst=dd, dst_cap=block, out_sizes=dres)
                    dms = timed(dfn)
                    assert (dres.cpu().numpy() == block).all()
                    assert dd[0].cpu().numpy().tobytes() == pieces[0] and dd[n - 1].cpu().numpy().tobytes() == pieces[n - 1]
                    res["s2_decode_%dk" % (block >> 10)] = {"ms": round(dms, 3), "GBps": round(nbytes / dms / 1e6, 2)}
                    del dd
                res[key] = r
                print(key, r, flush=True)
            del d_src, dst
            torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
