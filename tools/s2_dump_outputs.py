#!/usr/bin/env python
"""S2 / Snappy block-encode outputs of the benchmark's level-1 input, for comparing two builds output for output.

usage: s2_dump_outputs.py DIR [--nchunks N]

Encodes bench.py's level-1 batch (16384 x 64 KiB of synthetic text, the same seed) with the four device block
encoders (S2 / Snappy, fast / better) and writes, per encoder, `<name>_sizes.npy` (every block's size) and
`<name>_sample.npy` (the slots of a fixed, seeded sample of blocks, bytes past the block's end zeroed).  Run it once
per build (B2C_LIB selects the library) and compare the two directories with tools/compare_dumps.py."""
import argparse
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.dont_write_bytecode = True
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import helpers as H
from compress_b200 import s2

CHUNK = 65536
DATA_SEED = 1000       # bench.py's rank-0 seed
SAMPLE_SEED = 7
SAMPLE_BLOCKS = 256


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("dir")
    ap.add_argument("--nchunks", type=int, default=16384)
    a = ap.parse_args()
    os.makedirs(a.dir, exist_ok=True)
    dev = torch.device("cuda", 0)
    n = a.nchunks
    src = H.synth_text_torch(n * CHUNK, dev, seed=DATA_SEED)
    codec = s2.Codec()
    dst = torch.empty((n, s2.SLOT), dtype=torch.uint8, device=dev)
    sz = torch.empty((n,), dtype=torch.int64, device=dev)
    pick = np.sort(np.random.default_rng(SAMPLE_SEED).choice(n, size=min(n, SAMPLE_BLOCKS), replace=False))
    for name, snappy, better in (("s2", False, False), ("snappy", True, False), ("s2_better", False, True),
                                 ("snappy_better", True, True)):
        codec.encode_device(src, snappy=snappy, better=better, dst=dst, out_sizes=sz)
        torch.cuda.synchronize()
        sizes = sz.cpu().numpy()
        assert (sizes > 0).all(), name
        rows = dst[torch.from_numpy(pick).to(dev)].cpu().numpy()
        rows[np.arange(rows.shape[1])[None, :] >= sizes[pick][:, None]] = 0
        np.save(os.path.join(a.dir, name + "_sizes.npy"), sizes)
        np.save(os.path.join(a.dir, name + "_sample.npy"), rows)
        print("%s: %d blocks, %d bytes" % (name, n, int(sizes.sum())))
    codec.close()


if __name__ == "__main__":
    main()
