#!/usr/bin/env python3
"""Per-phase cycle breakdown of the histogram kernel (b2c_zstd_hist_kernel) on the bench text at level 1: lane 0 of every
warp stamps clock64 right after the kernel's barriers (B2C_HIST_PHASE; warp w in row 12 + w, columns 8..15 of the rows
b2c_zstd_encode_device_timed fills).  Prints, for the chunks that reached every stamp (compressed candidates), the mean
cycles per chunk between consecutive stamps: between the slowest warps (barrier release to release) and per warp.
B2C_LIB selects another build of the library.

usage: hist_phase_times.py [NCHUNKS]"""
import os, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np, torch
import helpers as H
from compress_b200 import zstd
from compress_b200._lib import lib, check

# stamp id -> the point it marks
NAMES = {0: "start", 1: "counters zeroed", 2: "literals and codes counted", 3: "copies reduced, histograms written"}


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        return torch.cuda.get_device_name(0)


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 16384
    enc = zstd.Encoder()
    src = H.synth_text_torch(n * 65536, "cuda", seed=42)
    dst = torch.empty((n, zstd.SLOT), dtype=torch.uint8, device="cuda")
    outs = torch.empty(n, dtype=torch.int64, device="cuda")
    cyc = torch.zeros((n, 16, 32), dtype=torch.int64, device="cuda")
    for _ in range(2):
        cyc.zero_()
        rc = lib.b2c_zstd_encode_device_timed(enc._ctx, 3, src.data_ptr(), 65536, 65536, dst.data_ptr(), zstd.SLOT,
                                              outs.data_ptr(), n, cyc.data_ptr(), None)
        check(rc, enc._ctx)
        torch.cuda.synchronize()
    c = cyc.cpu().numpy().astype(np.int64)[:, 12:16, 8:16].transpose(0, 2, 1)   # [n, stamp, warp] (0: not stamped)
    stamped = [k for k in range(8) if (c[:, k, 0] != 0).any()]
    full = np.all(c[:, stamped, :] != 0, axis=(1, 2))
    c = c[full]
    tot = c[:, stamped[-1], :].max(axis=1) - c[:, stamped[0], :].min(axis=1)
    print("%s, %s, %d chunks of the bench text, level 1" % (card(), os.path.basename(os.environ.get("B2C_LIB", "libb200comp.so")), n))
    print("hist kernel: %d of %d chunks counted, mean cycles/chunk %.0f (min %d, max %d)" % (len(c), n, tot.mean(), tot.min(), tot.max()))
    for a, b in zip(stamped[:-1], stamped[1:]):
        d = (c[:, b, :] - c[:, a, :]).astype(np.float64)          # per-warp time between the two stamps
        rel = c[:, b, :].max(axis=1) - c[:, a, :].max(axis=1)     # between the slowest warps
        nm = "%s -> %s" % (NAMES.get(a, a), NAMES.get(b, b))
        print("%-56s slowest-warp %8.0f (%4.1f%%)   mean-warp %8.0f" % (nm, rel.mean(), 100 * rel.mean() / tot.mean(), d.mean()))


if __name__ == "__main__":
    main()
