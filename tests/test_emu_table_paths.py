"""The table builders of K2 and standalone huff0 (warp-parallel depths, setMaxHeight, weight normalisation, table
description, sequence-table normalisation and mode choice) on inputs aimed at their rarer paths, under the emulator:
huff0 blocks must equal the oracle's bytes, zstd blocks the oracle's blockEnc.encode for the same parse."""
import numpy as np

from check_util import check_frames
from emu_util import emu_encode, emu_huf_compress
from test_emu_huf0 import orc_compress


def _block(counts, seed):
    """Bytes with exactly counts[s] copies of symbol s, in a seeded random order."""
    a = np.repeat(np.arange(len(counts), dtype=np.uint8), counts)
    np.random.Generator(np.random.PCG64(seed)).shuffle(a)
    return a.tobytes()


def _fib(n):
    f = [1, 1]
    while len(f) < n:
        f.append(f[-1] + f[-2])
    return f


def _inputs():
    geo = [max(1, int(4000 * 0.97 ** s)) for s in range(256)]
    return {
        # Fibonacci counts: an unlimited Huffman tree 21 levels deep, so setMaxHeight repairs it down to 11 bits
        "fib22": _block(_fib(22), 1),
        "fib18+flat": _block(_fib(18) + [40] * 60, 2),
        # two and three symbols: the table description takes the 4-bit form
        "two": _block([9000, 3000], 3),
        "three": _block([5000, 3000, 2000], 4),
        # every byte value, geometric counts: 255 weights through FSE
        "all256": _block(geo, 5),
        "all256-flat": _block([200] * 255 + [20000], 6),
    }


def test_huff0_table_paths_match_oracle(emu_lib, oracle_lib):
    inputs = _inputs()
    names = list(inputs)
    for four in (False, True):
        got = emu_huf_compress(emu_lib, [inputs[n] for n in names], four)
        for n, (out, code) in zip(names, got):
            assert (out, code) == orc_compress(inputs[n], four), (n, four)
            assert code > 0, (n, four)
            if n in ("two", "three"):
                assert out[0] >= 128, (n, four)   # 4-bit weights


def test_zstd_table_paths_match_oracle(emu_lib, oracle_lib):
    rng = np.random.Generator(np.random.PCG64(9))
    chunks = [c[:65536] for c in _inputs().values()]
    chunks += [
        b"abcd" * 5000,                                  # one sequence code per table: RLE modes
        b"0123456789abcdef" * 8 + bytes(rng.integers(0, 256, 200, dtype=np.uint8)) + b"0123456789abcdef" * 4,   # few sequences: predefined
        bytes(rng.integers(0, 2, 40000, dtype=np.uint8)),   # long runs of short matches
        bytes(rng.integers(0, 3, 40000, dtype=np.uint8)),
    ]
    frames, outs, hdr, seqs, lits = emu_encode(emu_lib, chunks)
    assert (outs > 0).all()
    check_frames(chunks, frames, hdr, seqs, lits, label="emu-table-paths")
