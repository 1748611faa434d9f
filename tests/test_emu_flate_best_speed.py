"""The BestSpeed kernels (b2c_deflate.cuh: l1, l1_check) under the CPU SIMT emulator, in both lane orders: bytes and
checksums equal the oracle's (oracle/orc_deflate.c) on the seeded pool and the reference's encoder fuzz corpus, raw, zlib
and gzip, with passes small enough that a batch spans several of them."""
import ctypes
import os
import subprocess
import zlib

import numpy as np
import pytest

import flate_best_speed_util as D
import helpers as H

EMU_SO = os.path.join(H.EMU_DIR, "libb2c_emu_flate_best_speed.so")
_E = None


def _emu():
    global _E
    if _E is None:
        subprocess.run(["make", "-s", "-C", H.EMU_DIR, "-f", "flate_best_speed.mk"], check=True)
        _E = ctypes.CDLL(EMU_SO)
        c = ctypes
        _E.emu_flate_best_speed.restype = c.c_int
        _E.emu_flate_best_speed.argtypes = [c.c_int] + [c.c_void_p] * 3 + [c.c_char_p, c.c_uint32, c.c_uint32] + [
            c.c_void_p] * 5 + [c.c_uint32]
        _E.emu_best_speed_set_lane_order.argtypes = [c.c_int]
    return _E


def emu_best_speed(inputs, fmt=D.RAW, lanes=4096, desc=0):
    """The kernels over a packed batch with odd input offsets and guarded destinations; returns (outputs, checks)."""
    E = _emu()
    E.emu_best_speed_set_lane_order(desc)
    n = len(inputs)
    soff = np.zeros(n, dtype=np.uint64)
    pos = 1
    for i, b in enumerate(inputs):
        soff[i] = pos
        pos += len(b) + 3
    src = np.zeros(pos + 16, dtype=np.uint8)
    for o, b in zip(soff, inputs):
        src[int(o):int(o) + len(b)] = np.frombuffer(b, dtype=np.uint8)
    sizes = np.array([len(b) for b in inputs], dtype=np.uint32)
    hdr = D.GZIP_HDR_BEST_SPEED if fmt == D.GZIP else b""
    caps = np.array([D.bound(len(b)) + len(hdr) + 8 for b in inputs], dtype=np.uint32)
    dst_off = np.zeros(n, dtype=np.uint64)
    pos = 3
    for i in range(n):
        dst_off[i] = pos
        pos += int(caps[i]) + 5
    dst = np.full(pos + 16, 0xA5, dtype=np.uint8)
    res = np.zeros(n, dtype=np.int64)
    chk = np.zeros(n, dtype=np.uint32)
    p = lambda a: a.ctypes.data  # noqa: E731
    E.emu_flate_best_speed(fmt, p(src), p(soff), p(sizes), hdr, len(hdr), n, p(dst), p(dst_off), p(caps), p(res), p(chk),
                           lanes)
    for o, c in zip(dst_off, caps):                  # nothing outside the destinations was written
        assert (dst[int(o) + int(c):int(o) + int(c) + 5] == 0xA5).all()
    outs = [dst[int(o):int(o) + int(r)].tobytes() if r >= 0 else None for o, r in zip(dst_off, res)]
    return outs, chk.tolist()


@pytest.mark.parametrize("desc", [0, 1])
def test_pool(desc):
    pool = [d for _, d in D.pool()]
    for fmt in (D.RAW, D.ZLIB, D.GZIP):
        outs, chk = emu_best_speed(pool, fmt, lanes=7, desc=desc)
        assert outs == [D.best_speed(d, fmt) for d in pool], fmt
        want = [zlib.adler32(d) for d in pool] if fmt == D.ZLIB else [zlib.crc32(d) for d in pool]
        assert chk == want


@pytest.mark.parametrize("desc", [0, 1])
def test_fuzz_corpus(desc):
    items = D.fuzz_inputs()
    outs, _ = emu_best_speed(items, D.RAW, lanes=500, desc=desc)
    assert outs == [D.best_speed(d) for d in items]
