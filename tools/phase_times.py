#!/usr/bin/env python3
"""Per-phase cycle breakdown of the level-1 parse kernel (b2c_lz_parse1_kernel):
lane 0 of every warp stamps clock64 at the phase boundaries (B2C_PHASE), dumped through b2c_zstd_encode_device_timed."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np, torch
import helpers as H
from compress_b200 import zstd
from compress_b200._lib import lib, check

# stamp order inside lz_parse_chunk and what lies between two consecutive stamps
ORDER = [0, 1, 2, 6, 3, 8, 9, 10, 11, 4, 5]
NAMES = ["dense pass (tiles: probe | store | fix | probe)", "stage chunk into shared memory (TMA)", "walk (per-thread greedy scan)",
         "long matches (warp 0) + barriers", "prefix-max of match ends", "trim loop", "two block scans",
         "emit loop (sequences, codes, literal mask)", "RLE test + literal scan", "literal compaction + header"]


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 132 * 8
    enc = zstd.Encoder()
    src = H.synth_text_torch(n * 65536, "cuda", seed=42)
    dst = torch.empty((n, zstd.SLOT), dtype=torch.uint8, device="cuda")
    outs = torch.empty(n, dtype=torch.int64, device="cuda")
    cyc = torch.zeros((n, 16, 32), dtype=torch.int64, device="cuda")
    for _ in range(2):
        rc = lib.b2c_zstd_encode_device_timed(enc._ctx, 3, src.data_ptr(), 65536, 65536, dst.data_ptr(), zstd.SLOT,
                                              outs.data_ptr(), n, cyc.data_ptr(), None)
        check(rc, enc._ctx)
        torch.cuda.synchronize()
    c = cyc.cpu().numpy().astype(np.int64)[:, :, :16]   # [n, 16, 16]: arrival of warp w at stamp k (0 where the warp does not exist); columns 16.. are the pack kernel's
    nw = int((c[0, 0] != 0).sum())
    c = c[:, :, :nw]
    order, names = ORDER, NAMES
    tot = c[:, order[-1], :].max(axis=1) - c[:, order[0], :].min(axis=1)
    print("parse kernel: chunks %d, warps/CTA %d, mean cycles/chunk %.0f (min %d, max %d)" % (n, nw, tot.mean(), tot.min(), tot.max()))
    for a, b, nm in zip(order[:-1], order[1:], names):
        d = (c[:, b, :] - c[:, a, :]).astype(np.float64)          # per-warp time between the two stamps
        rel = c[:, b, :].max(axis=1) - c[:, a, :].max(axis=1)     # between the slowest warps (~ barrier release to release)
        print("%-52s slowest-warp %8.0f (%4.1f%%)   mean-warp %8.0f" % (nm, rel.mean(), 100 * rel.mean() / tot.mean(), d.mean()))


if __name__ == "__main__":
    main()
