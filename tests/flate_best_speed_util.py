"""BestSpeed test helpers: the oracle (oracle/liboracle_flate_best_speed.so, built on demand: the level-1 compressor over
orc_deflate.c's bit writer), its decision counters, and a seeded input pool around every window edge.  The content
generators and corpora are deflate_util's."""
import ctypes
import os
import random
import subprocess

import helpers as H
from deflate_util import (PATHS as WRITER_PATHS, fuzz_inputs, huff_runs, skewed, sparse, testdata,  # noqa: F401
                          testdata_names, text)

ORACLE_SO = os.path.join(H.ORACLE_DIR, "liboracle_flate_best_speed.so")
WINDOW = 65535                      # BestSpeed's window: maxStoreBlockSize
RAW, ZLIB, GZIP = 0, 1, 2
GZIP_HDR_BEST_SPEED = b"\x1f\x8b\x08\x00\x00\x09\x6e\x88\x04\xff"   # gzip.NewWriterLevel(w, BestSpeed): XFL 4
# storeFast's branches and fastEncL1's history (orc_best_speed_paths, L1P_* order)
L1_PATHS = ["sf_stored", "sf_huff", "sf_dyn", "sf_final_stored", "sf_final_huff", "l1_prev_window", "l1_hist_move",
            "l1_back_stop", "l1_back_stop_moved"]
_L = None


def oracle():
    global _L
    if _L is None:
        if not os.path.exists(ORACLE_SO):
            subprocess.run(["make", "-s", "-C", H.ORACLE_DIR, "-f", "flate_best_speed.mk"], check=True)
        L = ctypes.CDLL(ORACLE_SO)
        c = ctypes
        L.orc_flate_best_speed.restype = c.c_int64
        L.orc_flate_best_speed.argtypes = [c.c_int, c.c_char_p, c.c_size_t, c.c_char_p, c.c_void_p, c.c_size_t, c.c_char_p,
                                           c.c_size_t, c.c_void_p]
        L.orc_deflate_paths.argtypes = [c.c_void_p]
        L.orc_best_speed_paths.argtypes = [c.c_void_p]
        _L = L
    return _L


def bound(n):
    """b2c_flate_best_speed_bound: at most 176 bytes over each 65 535-byte window, and 4 for Close."""
    return n + 176 * (n // WINDOW + 1) + 4


def best_speed(data, fmt=RAW, header=GZIP_HDR_BEST_SPEED, writes=None, cap=None, check=False):
    """The reference's writer at BestSpeed by the oracle: flate.NewWriter(w, 1) (RAW), zlib.NewWriterLevel(w, 1) (ZLIB)
    or gzip.NewWriterLevel(w, 1) with this member header (GZIP), for Write(p) of each piece of `writes` (default: one
    Write of all of data) and Close.  Returns the bytes or a negative code (and the CRC-32 / Adler-32 with check)."""
    data = bytes(data)
    if writes is None:
        writes = [len(data)]
    assert sum(writes) == len(data)
    hdr = header if fmt == GZIP else b""
    if cap is None:
        cap = bound(len(data)) + len(hdr) + 8
    out = ctypes.create_string_buffer(max(cap, 1))
    ws = (ctypes.c_size_t * max(len(writes), 1))(*writes)
    ck = ctypes.c_uint32()
    r = oracle().orc_flate_best_speed(fmt, hdr, len(hdr), data, ws, len(writes), out, cap, ctypes.byref(ck))
    res = out.raw[:r] if r >= 0 else r
    return (res, ck.value) if check else res


def paths_reset():
    oracle().orc_deflate_paths_reset()
    oracle().orc_best_speed_paths_reset()


def paths():
    """The bit writer's counters (deflate_util.PATHS names) and the BestSpeed ones (L1_PATHS) of this oracle library."""
    a = (ctypes.c_int64 * len(WRITER_PATHS))()
    b = (ctypes.c_int64 * len(L1_PATHS))()
    oracle().orc_deflate_paths(a)
    oracle().orc_best_speed_paths(b)
    return {**dict(zip(WRITER_PATHS, list(a))), **dict(zip(L1_PATHS, list(b)))}


def sizes():
    """Sizes around the storeFast thresholds and every window edge, across the history move before the sixth window."""
    s = [0, 1, 12, 13, 32, 33, 127, 128, WINDOW - 1, WINDOW, WINDOW + 1]
    for k in range(2, 13):
        s += [k * WINDOW - 1, k * WINDOW + 1]
    return s


def pool(seed=11):
    """(label, data): the sizes of sizes() as text, random, zeros and periodic content, and mixed content."""
    rng = random.Random(seed)
    out = []
    for n in sizes():
        out.append(("text", text(rng, n)))
        out.append(("random", rng.randbytes(n)))
        out.append(("zeros", bytes(n)))
        per = rng.randbytes(rng.randint(1, 300))
        out.append(("periodic", (per * (n // max(len(per), 1) + 1))[:n]))
    mix = b""
    while len(mix) < 7 * WINDOW:
        k = rng.randrange(7)
        m = rng.randint(200, 40000)
        mix += [text(rng, m), rng.randbytes(m), bytes(m), b"ab" * (m // 2), bytes(rng.choice(b"acgt") for _ in range(m)),
                sparse(rng, m), skewed(rng, m)][k]
    out.append(("mixed", mix))
    for n in (3000, WINDOW, 3 * WINDOW + 7):
        out.append(("sparse", sparse(rng, n)))
        out.append(("skewed", skewed(rng, n)))
    return out
