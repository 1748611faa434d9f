"""The HuffmanOnly / NoCompression kernels (b2c_deflate.cuh: nolz analyse, plan, emit, finish) under the CPU SIMT
emulator, in both lane orders: bytes and checksums equal the oracle's (oracle/orc_flate_nolz.c) on the seeded pool and
the reference's encoder fuzz corpus, for both levels and raw, zlib and gzip, with passes small enough that a batch spans
several of them; nothing outside a destination is written, and a destination one byte short is left untouched."""
import ctypes
import os
import subprocess
import zlib

import numpy as np
import pytest

import flate_nolz_util as D
import helpers as H

EMU_SO = os.path.join(H.EMU_DIR, "libb2c_emu_flate_nolz.so")
_E = None


def _emu():
    global _E
    if _E is None:
        subprocess.run(["make", "-s", "-C", H.EMU_DIR, "-f", "flate_nolz.mk"], check=True)
        _E = ctypes.CDLL(EMU_SO)
        c = ctypes
        _E.emu_flate_nolz.restype = c.c_int
        _E.emu_flate_nolz.argtypes = [c.c_int, c.c_int] + [c.c_void_p] * 3 + [c.c_char_p, c.c_uint32, c.c_uint32] + [
            c.c_void_p] * 5 + [c.c_uint32]
        _E.emu_nolz_set_lane_order.argtypes = [c.c_int]
    return _E


def emu_nolz(inputs, level, fmt=D.RAW, inputs_per_pass=4096, desc=0, caps=None):
    """The kernels over a packed batch with odd input offsets and guarded destinations; returns (outputs, codes, checks)."""
    E = _emu()
    E.emu_nolz_set_lane_order(desc)
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
    hdr = D.GZIP_HDR if fmt == D.GZIP else b""
    if caps is None:
        caps = [D.bound(level, len(b)) + D.container(fmt) for b in inputs]
    caps = np.array(caps, dtype=np.uint32)
    dst_off = np.zeros(n, dtype=np.uint64)
    pos = 3
    for i in range(n):
        dst_off[i] = pos
        pos += int(caps[i]) + 5
    dst = np.full(pos + 16, 0xA5, dtype=np.uint8)
    res = np.zeros(n, dtype=np.int64)
    chk = np.zeros(n, dtype=np.uint32)
    p = lambda a: a.ctypes.data  # noqa: E731
    E.emu_flate_nolz(level, fmt, p(src), p(soff), p(sizes), hdr, len(hdr), n, p(dst), p(dst_off), p(caps), p(res), p(chk),
                     inputs_per_pass)
    for o, c, r in zip(dst_off, caps, res):          # nothing outside the destinations, nor in a refused one, was written
        assert (dst[int(o) + int(c):int(o) + int(c) + 5] == 0xA5).all()
        if r < 0:
            assert (dst[int(o):int(o) + int(c)] == 0xA5).all()
    outs = [dst[int(o):int(o) + int(r)].tobytes() if r >= 0 else None for o, r in zip(dst_off, res)]
    return outs, res.tolist(), chk.tolist()


@pytest.mark.parametrize("desc", [0, 1])
@pytest.mark.parametrize("level", D.LEVELS)
def test_pool(level, desc):
    pool = [d for _, d in D.pool(scale=3)]
    for fmt in D.FORMATS:
        outs, _, chk = emu_nolz(pool, level, fmt, inputs_per_pass=13, desc=desc)
        assert outs == [D.nolz(d, level, fmt) for d in pool], fmt
        want = [zlib.adler32(d) for d in pool] if fmt == D.ZLIB else [zlib.crc32(d) for d in pool]
        assert chk == want


@pytest.mark.parametrize("desc", [0, 1])
@pytest.mark.parametrize("level", D.LEVELS)
def test_fuzz_corpus(level, desc):
    items = D.fuzz_inputs()
    for fmt in D.FORMATS:                            # a third of the corpus in each format
        part = items[fmt::3]
        outs, _, _ = emu_nolz(part, level, fmt, inputs_per_pass=230, desc=desc)
        assert outs == [D.nolz(d, level, fmt) for d in part], fmt


@pytest.mark.parametrize("level", D.LEVELS)
def test_dst_one_byte_short(level):
    import random
    rng = random.Random(9)
    items = [D.text(rng, 70000), rng.randbytes(40000), b"", D.skewed(rng, 33000)]
    for fmt in D.FORMATS:
        want = [D.nolz(d, level, fmt) for d in items]
        caps = [len(w) - 1 if k % 2 == 0 else len(w) for k, w in enumerate(want)]
        outs, codes, _ = emu_nolz(items, level, fmt, caps=caps)
        for k, w in enumerate(want):
            if k % 2 == 0:
                assert codes[k] == -4 and outs[k] is None
            else:
                assert outs[k] == w
