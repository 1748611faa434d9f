"""The LZ4 / LZ4s -> S2 / Snappy conversion kernels (b2c_lz4_cvt.cuh: walk + emit) under the CPU SIMT emulator, in both
lane orders: bytes, decoded sizes and error codes equal the oracle's (oracle/orc_lz4.c) over the seeded pool, both formats
and both outputs, at each sampled block's smallest accepted slot and one byte below."""
import numpy as np
import pytest

import lz4_util as U

MODES = [(False, False), (False, True), (True, False), (True, True)]   # (lz4s, snappy)


def emu_convert(blocks, caps, lz4s, snappy, lib=None):
    E = lib or _emu()
    n = len(blocks)
    src_off = np.zeros(n, dtype=np.uint64)
    pos = 1                                          # odd source and slot positions
    for i, b in enumerate(blocks):
        src_off[i] = pos
        pos += len(b) + 3
    src = np.zeros(pos + 16, dtype=np.uint8)
    for o, b in zip(src_off, blocks):
        src[int(o):int(o) + len(b)] = np.frombuffer(b, dtype=np.uint8)
    dst_off = np.zeros(n, dtype=np.uint64)
    pos = 3
    for i, cp in enumerate(caps):
        dst_off[i] = pos
        pos += cp + 5
    dst = np.full(pos + 16, 0xA5, dtype=np.uint8)
    sizes = np.array([len(b) for b in blocks], dtype=np.uint32)
    dcaps = np.array(caps, dtype=np.uint32)
    res = np.zeros(n, dtype=np.int64)
    dec = np.zeros(n, dtype=np.int64)
    E.emu_lz4_convert(src.ctypes.data, src_off.ctypes.data, sizes.ctypes.data, n, dst.ctypes.data, dst_off.ctypes.data,
                      dcaps.ctypes.data, res.ctypes.data, dec.ctypes.data, int(lz4s), int(snappy))
    for o, cp in zip(dst_off, caps):                 # nothing outside the slots was written
        assert (dst[int(o) + cp:int(o) + cp + 5] == 0xA5).all()
    outs = [dst[int(o):int(o) + int(r)].tobytes() if r >= 0 else None for o, r in zip(dst_off, res)]
    return outs, res.tolist(), dec.tolist()


def check(blocks, caps, lz4s, snappy, lib=None):
    outs, codes, ns = emu_convert(blocks, caps, lz4s, snappy, lib)
    for i, (b, cp) in enumerate(zip(blocks, caps)):
        want = U.slot_result(b, cp, lz4s, snappy)
        got = (codes[i], outs[i], ns[i] if codes[i] >= 0 or codes[i] == U.TOO_BIG else 0)
        assert got == want, (i, len(b), cp, lz4s, snappy, got[0], want[0])
    return codes


_E = None


def _emu():
    global _E
    if _E is None:
        _E = U.emu()
    return _E


@pytest.fixture(scope="module")
def pools():
    return {lz4s: U.pool(seed=7, lz4s=lz4s) for lz4s in (False, True)}


@pytest.mark.parametrize("desc", [0, 1])
@pytest.mark.parametrize("lz4s,snappy", MODES)
def test_emulated_kernels_equal_oracle(pools, lz4s, snappy, desc):
    _emu().emu_lz4_set_lane_order(desc)
    try:
        blocks = pools[lz4s]
        check(blocks, [2 * len(b) + 64 for b in blocks], lz4s, snappy)
        rng = np.random.default_rng(desc * 4 + lz4s * 2 + snappy)
        sample, caps = [], []
        for i in rng.choice(len(blocks), size=30, replace=False):
            m = U.min_cap(blocks[i], lz4s, snappy)
            if m is not None:
                sample += [blocks[i], blocks[i]]
                caps += [m, m - 1]
        codes = check(sample, caps, lz4s, snappy)
        assert all(codes[k] >= 0 and codes[k + 1] < 0 for k in range(0, len(sample), 2))
    finally:
        _emu().emu_lz4_set_lane_order(0)


def test_emulated_hand_built_edges():
    lits = (bytes(range(256)) * 12)[:3000]
    blocks = [U.block([(lits, 3000, 70000)], b"x"),                        # the inlined-emitter room case
              U.block([(b"abcd", 4, 4), (b"", 4, 4 + 65536 + (1 << 24))], b"x"),   # split repeat
              U.block([], b"\x99" * 70000),                                 # 4-byte literal header
              U.block([(b"abcd", 4, 65), (b"", 4, 67)], b"xy")]             # Snappy pieces with a remainder below 4
    for lz4s, snappy in MODES:
        if lz4s:
            continue
        for cp in (3027, 3026, 1 << 17):
            check(blocks, [cp] * len(blocks), lz4s, snappy)
