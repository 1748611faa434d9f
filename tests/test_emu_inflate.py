"""The inflate kernels (b2c_inflate.cuh: walk, exec, checksum) under the CPU SIMT emulator, in both lane orders: bytes and
outcome classes equal the oracle's (oracle/orc_flate.c) on the seeded pool, the reference's fixtures, hand-written and
stale-table streams, and mutated streams."""
import ctypes
import os
import random
import subprocess

import numpy as np
import pytest

import flate_util as F
import helpers as H

EMU_SO = os.path.join(H.EMU_DIR, "libb2c_emu_inflate.so")
_E = None


def _emu():
    global _E
    if _E is None:
        subprocess.run(["make", "-s", "-C", H.EMU_DIR, "-f", "inflate.mk"], check=True)
        _E = ctypes.CDLL(EMU_SO)
        c = ctypes
        _E.emu_inflate.restype = c.c_int
        _E.emu_inflate.argtypes = [c.c_int, c.c_int, c.c_void_p, c.c_void_p, c.c_void_p, c.c_uint32, c.c_void_p, c.c_void_p,
                                   c.c_void_p, c.c_void_p]
        _E.emu_inflate_set_lane_order.argtypes = [c.c_int]
    return _E


def emu_decode(fmt, streams, cap, multistream=True):
    E = _emu()
    n = len(streams)
    src_off = np.zeros(n, dtype=np.uint64)
    pos = 1                                          # odd source and destination positions
    for i, b in enumerate(streams):
        src_off[i] = pos
        pos += len(b) + 3
    src = np.zeros(pos + 16, dtype=np.uint8)
    for o, b in zip(src_off, streams):
        src[int(o):int(o) + len(b)] = np.frombuffer(b, dtype=np.uint8)
    dst_off = np.array([3 + i * (cap + 5) for i in range(n)], dtype=np.uint64)
    dst = np.full(3 + n * (cap + 5) + 16, 0xA5, dtype=np.uint8)
    sizes = np.array([len(b) for b in streams], dtype=np.uint32)
    caps = np.full(n, cap, dtype=np.uint32)
    res = np.zeros(n, dtype=np.int64)
    E.emu_inflate(fmt, int(multistream), src.ctypes.data, src_off.ctypes.data, sizes.ctypes.data, n, dst.ctypes.data,
                  dst_off.ctypes.data, caps.ctypes.data, res.ctypes.data)
    for o in dst_off:                                # nothing outside the destinations was written
        assert (dst[int(o) + cap:int(o) + cap + 5] == 0xA5).all()
    return [dst[int(o):int(o) + int(r)].tobytes() if r >= 0 else None for o, r in zip(dst_off, res)], res.tolist()


def _check(fmt, streams, cap, multistream=True):
    outs, codes = emu_decode(fmt, streams, cap, multistream)
    for i, s in enumerate(streams):
        r, want = F.orc_decode(fmt, s, cap, multistream)
        assert codes[i] == r, (i, fmt, codes[i], r)
        if r >= 0:
            assert outs[i] == want, i


@pytest.fixture(params=[0, 1], ids=["asc", "desc"])
def lane_order(request):
    _emu().emu_inflate_set_lane_order(request.param)
    yield request.param
    _emu().emu_inflate_set_lane_order(0)


def test_pool(lane_order):
    pool = F.pool(n=60)
    for fmt in (F.RAW, F.ZLIB, F.GZIP):
        for multi in (True, False):
            items = [s for f, s, d, m in pool if f == fmt and m == multi]
            if items:
                _check(fmt, items, 110000, multi)


def test_fixtures_and_invalid(lane_order):
    for fmt in (F.RAW, F.ZLIB, F.GZIP):
        streams = [s for _, f, s, _ in F.fixture_streams() if f == fmt]
        streams += [c[1] for c in F.invalid_streams() if c[0] == fmt and (len(c) < 4 or c[3])]
        streams += [s for f, s, _ in F.stale_streams() if f == fmt]
        _check(fmt, streams, 1 << 17)


def test_mutations(lane_order):
    rng = random.Random(31 + lane_order)
    for fmt in (F.RAW, F.ZLIB, F.GZIP):
        base = [F.deflate(F.text(rng, n), fmt, lv) for n, lv in ((1500, 1), (3000, 6), (400, 9), (900, 0))]
        base += [s for f, s, _ in F.stale_streams() if f == fmt]
        _check(fmt, [F.mutate(rng, rng.choice(base)) for _ in range(150)], 6000)
