#!/usr/bin/env python3
"""Per-phase cycle breakdown of the tables kernel (b2c_zstd_tables_kernel, K2) on the bench text at level 1: lane 0 of
the warp that builds a table stamps clock64 at the phase boundaries (stamp_clock; rows 12..15 of the rows
b2c_zstd_encode_device_timed fills: the Huffman build in row 12, the LL / OF / ML builds in rows 13..15).  Prints the
mean cycles per chunk of every phase, over the chunks that reached both of its stamps.  B2C_LIB selects another build
of the library.

usage: tables_phase_times.py [NCHUNKS]"""
import os, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np, torch
import helpers as H
from compress_b200 import zstd
from compress_b200._lib import lib, check

HUF = ["start", "stats + sort", "tree merge", "depths", "setMaxHeight + valPerRank", "bits + vals",
       "weights + table description", "written back"]
FSE = ["start", "normalize", "state fill", "size estimates", "NCount", "written back", "chunk barrier released"]


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        return torch.cuda.get_device_name(0)


def report(rows, names, label):
    """rows: [n, 32] stamps of one table's build (0: not stamped)."""
    print("%s" % label)
    for a in range(len(names) - 1):
        for b in range(a + 1, len(names)):       # next stamp this build reached (the early outs skip some)
            ok = (rows[:, a] != 0) & (rows[:, b] != 0)
            if ok.any():
                break
        else:
            continue
        d = (rows[ok, b] - rows[ok, a]).astype(np.float64)
        print("  %-34s -> %-30s %8.0f cycles/chunk  (%d chunks)" % (names[a], names[b], d.mean(), int(ok.sum())))
    first = rows[:, 0] != 0
    last = np.max(rows, axis=1)
    if first.any():
        print("  %-67s %8.0f cycles/chunk" % ("first -> last stamp", (last[first] - rows[first, 0]).astype(np.float64).mean()))


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
    c = cyc.cpu().numpy().astype(np.int64)
    print("%s, %s, %d chunks of the bench text, level 1" % (card(), os.path.basename(os.environ.get("B2C_LIB", "libb200comp.so")), n))
    report(c[:, 12, :8], HUF, "Huffman table (row 12)")
    for t, nm in enumerate(("LL", "OF", "ML")):
        report(c[:, 13 + t, :len(FSE)], FSE, "%s table (row %d)" % (nm, 13 + t))


if __name__ == "__main__":
    main()
