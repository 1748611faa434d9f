#!/usr/bin/env python3
"""Per-phase cycle breakdown of the level-1 pack kernel (b2c_zstd_pack_kernel): lane 0 of every warp stamps clock64 at
the phase boundaries (B2C_PACK_PHASE, columns 16..31 of the rows b2c_zstd_encode_device_timed fills), for the chunks that
end as compressed blocks.  Stamps are ordered by their mean time, so kernels that place them differently print their own
phase order.  B2C_LIB selects another build of the library.

usage: pack_phase_times.py [NCHUNKS]"""
import os, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np, torch
import helpers as H
from compress_b200 import zstd
from compress_b200._lib import lib, check

# stamp id -> the point it marks
NAMES = {0: "start", 1: "literals in shared memory", 2: "Huffman sizes + scan", 3: "literal mode decided",
         4: "sequence sizes + scan", 5: "stage zeroed", 6: "Huffman streams packed", 7: "sequence bitstream packed",
         8: "headers written", 9: "written back"}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        return q
    except Exception:
        return torch.cuda.get_device_name(0)


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 132 * 16
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
    c = cyc.cpu().numpy().astype(np.int64)[:, :, 16:]   # [n, 16, 16]: arrival of pack warp w at stamp k (0: not stamped)
    nw = int((c[:, 0] != 0).sum(axis=1).max())
    c = c[:, :, :nw]
    stamped = [k for k in range(16) if (c[:, k, 0] != 0).any()]
    full = np.all(c[:, stamped, 0] != 0, axis=1)          # chunks that went through every stamp (compressed blocks)
    c = c[full]
    t0 = c[:, 0, :].min(axis=1)[:, None]
    order = sorted(stamped, key=lambda k: (c[:, k, :] - t0).mean())
    tot = c[:, order[-1], :].max(axis=1) - c[:, order[0], :].min(axis=1)
    print("%s, %s" % (card(), os.environ.get("B2C_LIB", "libb200comp.so")))
    print("pack kernel: %d of %d chunks compressed, warps/CTA %d, mean cycles/chunk %.0f (min %d, max %d)"
          % (len(c), n, nw, tot.mean(), tot.min(), tot.max()))
    for a, b in zip(order[:-1], order[1:]):
        d = (c[:, b, :] - c[:, a, :]).astype(np.float64)          # per-warp time between the two stamps
        rel = c[:, b, :].max(axis=1) - c[:, a, :].max(axis=1)     # between the slowest warps
        nm = "%s -> %s" % (NAMES.get(a, a), NAMES.get(b, b))
        print("%-62s slowest-warp %8.0f (%4.1f%%)   mean-warp %8.0f" % (nm, rel.mean(), 100 * rel.mean() / tot.mean(), d.mean()))


if __name__ == "__main__":
    main()
