"""The inflate kernels (b2c_inflate.cuh) under the CPU SIMT emulator, in both lane orders, on the hand-built streams of
inflate_streams.py -- code shapes, exec layouts, checksum sizes, record-bound streams and header edges -- and on every
truncation of a few streams: bytes and outcome classes equal the oracle's (oracle/orc_flate.c).  Also the self-checks of
inflate_streams.py: every `valid` stream decodes with Python's zlib to the oracle's bytes, every checksum trailer is
zlib's, the record-bound streams reach the terms they target, and no family is empty."""
import ctypes
import os
import subprocess
import zlib

import numpy as np
import pytest

import flate_util as F
import helpers as H
import inflate_streams as S

EMU_SO = os.path.join(H.EMU_DIR, "libb2c_emu_inflate.so")
_E = None
BIG_CAP = 1 << 21


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


@pytest.fixture(params=[0, 1], ids=["asc", "desc"])
def lane_order(request):
    _emu().emu_inflate_set_lane_order(request.param)
    yield request.param
    _emu().emu_inflate_set_lane_order(0)


def emu_decode(fmt, streams, caps, multistream=True):
    """The emulated kernels with per-input caps, at odd source and destination offsets; a guard after each row."""
    n = len(streams)
    src_off = np.zeros(n, dtype=np.uint64)
    pos = 1
    for i, b in enumerate(streams):
        src_off[i] = pos
        pos += len(b) + 3
    src = np.zeros(pos + 16, dtype=np.uint8)
    for o, b in zip(src_off, streams):
        src[int(o):int(o) + len(b)] = np.frombuffer(b, dtype=np.uint8)
    dst_off = np.zeros(n, dtype=np.uint64)
    pos = 3
    for i, c in enumerate(caps):
        dst_off[i] = pos
        pos += c + 5
    dst = np.full(pos + 16, 0xA5, dtype=np.uint8)
    sizes = np.array([len(b) for b in streams], dtype=np.uint32)
    caps_a = np.array(caps, dtype=np.uint32)
    res = np.zeros(n, dtype=np.int64)
    _emu().emu_inflate(fmt, int(multistream), src.ctypes.data, src_off.ctypes.data, sizes.ctypes.data, n, dst.ctypes.data,
                       dst_off.ctypes.data, caps_a.ctypes.data, res.ctypes.data)
    for o, c in zip(dst_off, caps):
        assert (dst[int(o) + c:int(o) + c + 5] == 0xA5).all()
    return [dst[int(o):int(o) + int(r)].tobytes() if r >= 0 else None for o, r in zip(dst_off, res)], res.tolist()


def caps_of(streams):
    """Each stream's cap: its own, else the oracle's content length (into BIG_CAP) + 64."""
    return [s.cap if s.cap is not None else max(F.orc_decode(s.fmt, s.data, BIG_CAP)[0], 0) + 64 for s in streams]


def check(streams):
    for fmt in (S.RAW, S.ZLIB, S.GZIP):
        part = [s for s in streams if s.fmt == fmt]
        if not part:
            continue
        caps = caps_of(part)
        outs, codes = emu_decode(fmt, [s.data for s in part], caps)
        for s, c, out, code in zip(part, caps, outs, codes):
            r, want = F.orc_decode(fmt, s.data, c)
            assert code == r, (s.name, code, r)
            if r >= 0:
                assert out == want, s.name


FAMILIES = {"code_shapes": S.code_shapes, "exec_layouts": S.exec_layouts,
            "checksum_sizes": lambda: S.checksum_sizes(big=False), "record_bound": lambda: S.record_bound(big=False),
            "header_edges": S.header_edges}


@pytest.mark.parametrize("family", sorted(FAMILIES))
def test_family_valid_streams_equal_zlib(family):
    streams = FAMILIES[family]()
    assert streams
    assert any(s.valid for s in streams)
    for s in streams:
        if not s.valid:
            continue
        want = S.zlib_decode(s.fmt, s.data)
        assert want is not None, s.name
        r, out = F.orc_decode(s.fmt, s.data, s.cap if s.cap is not None else BIG_CAP)
        assert r == len(want) and out == want, (s.name, r, len(want))


def test_checksum_trailers_are_zlibs():
    for s in S.checksum_sizes(big=False):
        if s.fmt == S.ZLIB:
            content = zlib.decompress(s.data) if s.valid else None
            if content is not None:
                assert s.data[-4:] == zlib.adler32(content).to_bytes(4, "big"), s.name
        elif s.valid and s.name.startswith("gzip "):              # (one member: its CRC-32 is the content's)
            content = S.zlib_decode(S.GZIP, s.data)
            assert s.data[-8:-4] == zlib.crc32(content).to_bytes(4, "little"), s.name
    # a bad trailer differs from the right one in one bit
    streams = S.checksum_sizes(big=False)
    pairs = [(a, b) for a, b in zip(streams, streams[1:]) if a.valid and not b.valid and b.name == a.name + ", bad checksum"]
    assert len(pairs) > 600
    for a, b in pairs:
        x = int.from_bytes(a.data, "little") ^ int.from_bytes(b.data, "little")
        assert len(a.data) == len(b.data) and bin(x).count("1") == 1, a.name


def rec_cap(slen, cap):
    """inf_rec_cap (b2c_inflate.cuh)."""
    return min(cap // 3, 4 * slen) + slen // 5 + slen // 18 + 2


def test_record_bound_streams_reach_their_terms():
    streams = S.record_bound(big=True)
    assert len(streams) == 4
    for s in streams:
        records, want = S.record_term(s)
        assert want <= records <= rec_cap(len(s.data), s.cap), (s.name, records, want)
        assert F.orc_decode(s.fmt, s.data, s.cap)[0] >= 0, s.name
    m258, m3 = streams[0], streams[1]
    assert 4 * len(m258.data) < m258.cap // 3                      # the 4 * slen term binds
    assert m3.cap // 3 < 4 * len(m3.data)                          # the cap / 3 term binds ...
    assert F.orc_decode(m3.fmt, m3.data, m3.cap)[0] == m3.cap      # ... with the content filling the cap exactly


@pytest.mark.parametrize("family", sorted(FAMILIES))
def test_family(lane_order, family):
    check(FAMILIES[family]())


def test_truncations(lane_order):
    for fmt, s in S.truncation_set():
        cuts = [S.Stream(fmt, s[:i], False, "cut %d" % i, 8192) for i in range(len(s) + 1)]
        check(cuts)
