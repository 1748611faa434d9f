"""The stateless deflate kernels (b2c_deflate.cuh: parse, encode, crc) under the CPU SIMT emulator, in both lane orders:
bytes equal the oracle's (oracle/orc_deflate.c) on the seeded pool, the reference's encoder fuzz corpus, the dict cases and
the Huffman-only reuse runs, raw and gzip, with passes small enough that inputs span them."""
import ctypes
import os
import subprocess
import zlib

import numpy as np
import pytest

import deflate_util as D
import helpers as H

EMU_SO = os.path.join(H.EMU_DIR, "libb2c_emu_deflate.so")
HDR = b"\x1f\x8b\x08\x00\x00\x00\x00\x00\x00\xff"
_E = None


def _emu():
    global _E
    if _E is None:
        subprocess.run(["make", "-s", "-C", H.EMU_DIR, "-f", "deflate.mk"], check=True)
        _E = ctypes.CDLL(EMU_SO)
        c = ctypes
        _E.emu_deflate.restype = c.c_int
        _E.emu_deflate.argtypes = [c.c_int] + [c.c_void_p] * 7 + [c.c_char_p, c.c_uint32, c.c_uint32] + [c.c_void_p] * 5 + [
            c.c_uint32]
        _E.emu_deflate_set_lane_order.argtypes = [c.c_int]
    return _E


def _pack(bufs, first=1):
    off = np.zeros(len(bufs), dtype=np.uint64)
    pos = first                                      # odd positions
    for i, b in enumerate(bufs):
        off[i] = pos
        pos += len(b) + 3
    a = np.zeros(pos + 16, dtype=np.uint8)
    for o, b in zip(off, bufs):
        a[int(o):int(o) + len(b)] = np.frombuffer(b, dtype=np.uint8)
    return a, off


def emu_encode(inputs, fmt=0, eofs=None, dicts=None, pass_slots=8192, desc=0):
    E = _emu()
    E.emu_deflate_set_lane_order(desc)
    n = len(inputs)
    src, soff = _pack(inputs)
    sizes = np.array([len(b) for b in inputs], dtype=np.uint32)
    eof = None if eofs is None else np.array([1 if e else 0 for e in eofs], dtype=np.uint8)
    dsrc = doff = dsz = None
    if dicts is not None:
        dl = [d or b"" for d in dicts]
        dsrc, doff = _pack(dl)
        dsz = np.array([len(d) for d in dl], dtype=np.uint32)
    caps = np.array([D.bound(len(b)) + len(HDR) + 16 for b in inputs], dtype=np.uint32)
    dst_off = np.zeros(n, dtype=np.uint64)
    pos = 3
    for i in range(n):
        dst_off[i] = pos
        pos += int(caps[i]) + 5
    dst = np.full(pos + 16, 0xA5, dtype=np.uint8)
    res = np.zeros(n, dtype=np.int64)
    crc = np.zeros(n, dtype=np.uint32)
    p = lambda a: None if a is None else a.ctypes.data  # noqa: E731
    hdr = HDR if fmt == 2 else b""
    E.emu_deflate(fmt, p(src), p(soff), p(sizes), p(eof), p(dsrc), p(doff), p(dsz), hdr, len(hdr), n, p(dst), p(dst_off),
                  p(caps), p(res), p(crc), pass_slots)
    for o, c in zip(dst_off, caps):                  # nothing outside the destinations was written
        assert (dst[int(o) + int(c):int(o) + int(c) + 5] == 0xA5).all()
    assert crc.tolist() == [zlib.crc32(b) for b in inputs]
    return [dst[int(o):int(o) + int(r)].tobytes() if r >= 0 else None for o, r in zip(dst_off, res)]


@pytest.mark.parametrize("desc", [0, 1])
def test_pool(desc):
    pool = [d for _, d in D.pool()]
    assert emu_encode(pool, desc=desc, pass_slots=7) == [D.stateless(d) for d in pool]
    assert emu_encode(pool, fmt=2, desc=desc) == [D.gzip_member(d, HDR) for d in pool]


@pytest.mark.parametrize("desc", [0, 1])
def test_fuzz_corpus(desc):
    items = [p for data in D.fuzz_inputs() for p in D.fuzz_split(data)]
    got = emu_encode([p[0] for p in items], eofs=[p[1] for p in items], dicts=[p[2] for p in items], desc=desc)
    assert got == [D.stateless(*p) for p in items]


@pytest.mark.parametrize("desc", [0, 1])
def test_dicts_and_huffman_runs(desc):
    cases = D.dict_cases()
    ins, dicts = [c[0] for c in cases], [c[1] for c in cases]
    eofs = [i % 2 == 0 for i in range(len(ins))]
    assert emu_encode(ins, eofs=eofs, dicts=dicts, desc=desc, pass_slots=5) == [
        D.stateless(d, e, dc) for d, e, dc in zip(ins, eofs, dicts)]
    runs = [D.huff_runs(n) for n in (3 * D.STEP + 7, 4 * D.STEP)]
    for eof in (False, True):
        assert emu_encode(runs, eofs=[eof] * 2, desc=desc, pass_slots=3) == [D.stateless(r, eof) for r in runs]
