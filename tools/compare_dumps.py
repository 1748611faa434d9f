#!/usr/bin/env python
"""Compare two output dumps file by file (bench.py --dump-outputs, tools/s2_dump_outputs.py): every .npy file of DIR_A
must exist in DIR_B with identical contents.  Exit code 1 on any difference.

usage: compare_dumps.py DIR_A DIR_B"""
import os
import sys

import numpy as np


def main():
    a, b = sys.argv[1], sys.argv[2]
    names = sorted(f for f in os.listdir(a) if f.endswith(".npy"))
    bad = 0
    for f in names:
        pb = os.path.join(b, f)
        if not os.path.exists(pb):
            print("%s: missing in %s" % (f, b))
            bad += 1
            continue
        x, y = np.load(os.path.join(a, f)), np.load(pb)
        same = x.shape == y.shape and x.dtype == y.dtype and np.array_equal(x, y)
        print("%s: %s %s" % (f, "identical" if same else "DIFFERENT", x.shape))
        bad += not same
    print("%d of %d files identical" % (len(names) - bad, len(names)))
    sys.exit(1 if bad or not names else 0)


if __name__ == "__main__":
    main()
