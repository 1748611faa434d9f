"""The S2 best kernels (b2c_lz_s2_best_kernel / b2c_lz_snappy_best_kernel, b2c_lz.cuh) under the CPU SIMT emulator, in
both lane orders: round trips through the oracle decoder (and pyarrow's Snappy), MaxEncodedLen, lane-order independence,
the stored-or-tags decision and the ratio against the emulated better class and the serial oracle.  CPU only."""
import pytest

import s2best_util as U
from emu_util import emu_s2_encode
from test_s2_best_oracle import _blocks


@pytest.fixture(scope="module")
def E():
    return U.emu()


@pytest.mark.parametrize("snappy", [False, True])
def test_emu_best_roundtrip_both_orders(E, snappy):
    L = U.oracle()
    blocks = _blocks() + U.fuzz_seeds()
    blocks = [b for b in blocks if len(b) <= 65536]
    a, outs = U.emu_encode(E, blocks, snappy=snappy, desc=0)
    b, _ = U.emu_encode(E, blocks, snappy=snappy, desc=1)
    assert a == b
    for i, (blk, c, r) in enumerate(zip(blocks, a, outs)):
        assert r == len(c) > 0 and r <= L.orc_s2_max_encoded_len(len(blk)), (i, r)
        n, got = U.decode(c, len(blk))
        assert n == len(blk) and got == blk, (snappy, i)
    if snappy:
        pa = pytest.importorskip("pyarrow")
        codec = pa.Codec("snappy")
        for blk, c in zip(blocks, a):
            if blk:
                assert codec.decompress(c, decompressed_size=len(blk)).to_pybytes() == blk


@pytest.mark.parametrize("snappy", [False, True])
def test_emu_best_stored_or_tags(E, snappy):
    """Short blocks and incompressible ones are one literal; the random block with one repeated 1 KiB run is tags, as the
    oracle decides (EncodeBetter stores it)."""
    rnd = _blocks()[16]
    rr = U.random_with_repeat()
    out, _ = U.emu_encode(E, [b"abc" * 5, bytes(31), rnd, rr], snappy=snappy)
    assert out[0] == bytes([15, 14 << 2]) + b"abc" * 5
    assert out[1] == bytes([31, 30 << 2]) + bytes(31)
    assert len(out[2]) == 3 + 3 + 65536
    ref = U.encode(rr, U.SNAPPY_BEST if snappy else U.BEST)
    assert len(ref) < 65536 and len(out[3]) < 65536 - 900
    assert U.decode(out[3], len(rr))[1] == rr


@pytest.mark.parametrize("snappy", [False, True])
def test_emu_best_ratio(E, emu_lib, snappy):
    """Per corpus the best class is within +5 % of the serial EncodeBest / EncodeSnappyBest (the contract of every GPU
    class) and strictly smaller than the emulated better class of the same format."""
    for name, chunks in U.corpora().items():
        ours = sum(len(x) for x in U.emu_encode(E, chunks, snappy=snappy)[0])
        better = sum(len(x) for x in emu_s2_encode(emu_lib, chunks, snappy=snappy, better=True)[0])
        ref = sum(len(U.encode(c, U.SNAPPY_BEST if snappy else U.BEST)) for c in chunks)
        assert ours <= 1.05 * ref, (name, ours, ref)
        assert ours < better, (name, ours, better)
