"""HuffmanOnly / NoCompression test helpers: the oracle (oracle/liboracle_flate_nolz.so, built on demand: the two levels'
compressor over orc_deflate.c's bit writer), its decision counters, and a seeded input pool around every window edge.
The content generators and corpora are deflate_util's."""
import ctypes
import os
import random
import subprocess

import helpers as H
from deflate_util import (PATHS as WRITER_PATHS, fuzz_inputs, huff_runs, skewed, sparse, testdata,  # noqa: F401
                          testdata_names, text)

ORACLE_SO = os.path.join(H.ORACLE_DIR, "liboracle_flate_nolz.so")
HUFFMAN_ONLY, NO_COMPRESSION = -2, 0
LEVELS = (HUFFMAN_ONLY, NO_COMPRESSION)
WINDOW = {HUFFMAN_ONLY: 32768, NO_COMPRESSION: 65535}
RAW, ZLIB, GZIP = 0, 1, 2
FORMATS = (RAW, ZLIB, GZIP)
GZIP_HDR = b"\x1f\x8b\x08\x00\x00\x09\x6e\x88\x00\xff"   # gzip.NewWriterLevel(w, -2 | 0): XFL 0
# writeBlockHuff outcomes this level adds to the writer's counters (orc_nolz_paths, NP_* order)
NOLZ_PATHS = ["est_stored_small", "est_stored_large", "new_owes_eob", "final_full", "final_tiny", "empty"]
_L = None


def oracle():
    global _L
    if _L is None:
        if not os.path.exists(ORACLE_SO):
            subprocess.run(["make", "-s", "-C", H.ORACLE_DIR, "-f", "flate_nolz.mk"], check=True)
        L = ctypes.CDLL(ORACLE_SO)
        c = ctypes
        L.orc_flate_nolz.restype = c.c_int64
        L.orc_flate_nolz.argtypes = [c.c_int, c.c_int, c.c_char_p, c.c_size_t, c.c_char_p, c.c_void_p, c.c_size_t,
                                     c.c_char_p, c.c_size_t, c.c_void_p]
        L.orc_deflate_paths.argtypes = [c.c_void_p]
        L.orc_nolz_paths.argtypes = [c.c_void_p]
        _L = L
    return _L


def bound(level, n):
    """b2c_flate_nolz_bound: level 0 stores len + 5 bytes per 65 535-byte window; level -2 writes at most len + 242 per
    32 768-byte window; Close adds 2."""
    if level == NO_COMPRESSION:
        return n + 5 * (n // 65535 + 1) + 2
    return n + 242 * (n // 32768 + 1) + 2


def container(fmt, header=GZIP_HDR):
    return 6 if fmt == ZLIB else (len(header) + 8 if fmt == GZIP else 0)


def nolz(data, level, fmt=RAW, header=GZIP_HDR, writes=None, cap=None, check=False):
    """The reference's writer at `level` by the oracle: flate.NewWriter(w, level) (RAW), zlib.NewWriterLevel (ZLIB) or
    gzip.NewWriterLevel with this member header (GZIP), for Write(p) of each piece of `writes` (default: one Write of all
    of data) and Close.  Returns the bytes or a negative code (and the CRC-32 / Adler-32 with check)."""
    data = bytes(data)
    if writes is None:
        writes = [len(data)]
    assert sum(writes) == len(data)
    hdr = header if fmt == GZIP else b""
    if cap is None:
        cap = bound(level, len(data)) + container(fmt, hdr)
    out = ctypes.create_string_buffer(max(cap, 1))
    ws = (ctypes.c_size_t * max(len(writes), 1))(*writes)
    ck = ctypes.c_uint32()
    r = oracle().orc_flate_nolz(level, fmt, hdr, len(hdr), data, ws, len(writes), out, cap, ctypes.byref(ck))
    res = out.raw[:r] if r >= 0 else r
    return (res, ck.value) if check else res


def paths_reset():
    oracle().orc_deflate_paths_reset()
    oracle().orc_nolz_paths_reset()


def paths():
    """The bit writer's counters (deflate_util.PATHS names) and this level's (NOLZ_PATHS) of this oracle library."""
    a = (ctypes.c_int64 * len(WRITER_PATHS))()
    b = (ctypes.c_int64 * len(NOLZ_PATHS))()
    oracle().orc_deflate_paths(a)
    oracle().orc_nolz_paths(b)
    return {**dict(zip(WRITER_PATHS, list(a))), **dict(zip(NOLZ_PATHS, list(b)))}


def sizes(scale=4):
    """0-200, and k windows +- 1 of either level for k up to `scale`."""
    s = list(range(0, 201, 7)) + [1, 2, 3, 200, 1023, 1024, 1025]
    for w in (32768, 65535):
        for k in range(1, scale + 1):
            s += [k * w - 1, k * w, k * w + 1]
    return sorted(set(s))


def equal256(n):
    """Every byte value equally often: the float64 test's zero-variance case."""
    return (bytes(range(256)) * (n // 256 + 1))[:n]


def pool(seed=17, scale=4):
    """(label, data): the sizes of sizes() as text, random, zeros, one repeated byte, all-256-equal, skewed and mixed
    content."""
    rng = random.Random(seed)
    out = []
    for n in sizes(scale):
        out.append(("text", text(rng, n)))
        out.append(("random", rng.randbytes(n)))
        out.append(("zeros", bytes(n)))
        out.append(("byte", bytes([rng.randrange(256)]) * n))
        out.append(("equal256", equal256(n)))
        out.append(("skewed", skewed(rng, n)))
    mix = b""
    while len(mix) < 5 * 32768 + 77:
        m = rng.randint(100, 40000)
        mix += [text(rng, m), rng.randbytes(m), bytes(m), b"ab" * (m // 2), bytes(rng.choice(b"acgt") for _ in range(m)),
                sparse(rng, m), skewed(rng, m), equal256(m)][rng.randrange(8)]
    out.append(("mixed", mix))
    return out
