"""The S2 best oracle (oracle/orc_s2best.c): its size helpers against the emitters the KATs pin, round trips of
EncodeBest / EncodeSnappyBest through the oracle decoder and pyarrow's Snappy, and hand-built inputs that pin the choices
EncodeBetter does not make.  CPU only."""
import ctypes

import numpy as np
import pytest

import helpers as H
import s2best_util as U


def _blocks():
    rng = np.random.default_rng(11)
    tw = H.golden("twain.txt")
    return [b"", b"a", b"abc" * 5, bytes(31), bytes(32), bytes(33), bytes(100), tw[:33], tw[:1000], tw[:65536],
            H.golden("html.txt")[:65536], H.golden("e.txt")[:65536], H.synth_text(65536), bytes(65536), b"ab" * 32768,
            bytes(rng.integers(0, 256, 5000, dtype=np.uint8)), bytes(rng.integers(0, 256, 65536, dtype=np.uint8)),
            bytes(rng.integers(0, 3, 65536, dtype=np.uint8)), tw[:3000] + bytes(rng.integers(0, 256, 60000, dtype=np.uint8)),
            (tw[:700] + bytes(rng.integers(0, 256, 300, dtype=np.uint8))) * 60, U.random_with_repeat()]


OFFSETS = [1, 2047, 2048, 65535, 65536, (1 << 21) - 1, 1 << 21]


@pytest.mark.parametrize("offset", OFFSETS)
def test_size_helpers_equal_emitters(offset):
    """emitCopySize / emitRepeatSize give the length emitCopy / emitRepeat write, for every length of their domain,
    4 .. 2^24 (s2/encode_best.go:723-726)."""
    L = U.oracle()
    top = 1 << 24
    assert L.orc_s2_size_helper_mismatch(0, offset, 4, top) == -1
    assert L.orc_s2_size_helper_mismatch(1, offset, 4, top) == -1


@pytest.mark.parametrize("offset", OFFSETS)
def test_norepeat_size_estimate(offset):
    """emitCopyNoRepeatSize is exact below 64 bytes and, as in the reference, an estimate from there on: never below what
    emitCopyNoRepeat writes, by at most one piece header (5 bytes with a 4-byte offset, 3 otherwise)."""
    L = U.oracle()
    assert L.orc_s2_size_helper_mismatch(2, offset, 4, 63) == -1
    buf = ctypes.create_string_buffer(1 << 20)
    for ln in list(range(64, 5000)) + list(range(5000, 1 << 20, 9973)) + [(1 << 20) - 1]:
        est, got = L.orc_s2_emit_copy_norepeat_size(offset, ln), L.orc_s2_emit_copy_norepeat(buf, offset, ln)
        assert got <= est <= got + (5 if offset >= 65536 else 3), (offset, ln, est, got)


def _check_roundtrip(inputs, modes=(U.BEST, U.SNAPPY_BEST)):
    L = U.oracle()
    for i, s in enumerate(inputs):
        for mode in modes:
            comp = U.encode(s, mode)
            assert len(comp) <= L.orc_s2_max_encoded_len(len(s)), (i, mode)
            r, got = U.decode(comp, len(s))
            assert r == len(s) and got == s, (i, mode)


def test_roundtrip_blocks_and_golden():
    tw = H.golden("twain.txt")
    _check_roundtrip(_blocks() + [tw, H.golden("html.txt"), H.golden("e.txt"), tw[:200000] * 2])


def test_roundtrip_fuzz_seeds():
    _check_roundtrip(U.fuzz_seeds())


def test_snappy_best_is_snappy():
    pa = pytest.importorskip("pyarrow")
    codec = pa.Codec("snappy")
    for i, s in enumerate(_blocks() + U.fuzz_seeds()):
        if len(s):
            comp = U.encode(s, U.SNAPPY_BEST)
            assert codec.decompress(comp, decompressed_size=len(s)).to_pybytes() == s, i


def test_modes_0_to_2_unchanged():
    """The new library compiles the S2 oracle in: modes 0-2 give exactly the bytes of oracle/liboracle.so."""
    from test_oracle_s2 import s2_encode
    for s in _blocks():
        for mode in (0, 1, 2):
            assert U.encode(s, mode) == s2_encode(s, mode)


def _tags(comp):
    """(kind, offset, length) of every element of an S2 block: 'lit', 'copy' or 'rep'."""
    r = []
    i = 0
    while comp[i] & 0x80:
        i += 1
    i += 1
    while i < len(comp):
        t = comp[i]
        if t & 3 == 0:
            x = t >> 2
            if x < 60:
                ln, i = x + 1, i + 1
            else:
                k = x - 59
                ln, i = int.from_bytes(comp[i + 1:i + 1 + k], "little") + 1, i + 1 + k
            r.append(("lit", 0, ln))
            i += ln
        elif t & 3 == 1:
            off, code = ((t & 0xe0) << 3) | comp[i + 1], (t >> 2) & 7
            if off:
                r.append(("copy", off, code + 4))
                i += 2
            else:                                   # (a repeat's length beyond its 3-bit code is not decoded here)
                r.append(("rep", 0, code + 4))
                i += 2 + {5: 1, 6: 2, 7: 3}.get(code, 0)
        elif t & 3 == 2:
            r.append(("copy", int.from_bytes(comp[i + 1:i + 3], "little"), (t >> 2) + 1))
            i += 3
        else:
            r.append(("copy", int.from_bytes(comp[i + 1:i + 5], "little"), (t >> 2) + 1))
            i += 5
    return r


def test_best_tags_where_better_stores():
    """Random bytes with one repeated 1 KiB run: the saving is below EncodeBetter's n/32 limit, above EncodeBest's 5 bytes."""
    b = U.random_with_repeat()
    better, best = U.encode(b, U.BETTER), U.encode(b, U.BEST)
    assert len(better) == 3 + 3 + len(b)                      # stored: uvarint + 3-byte literal header + n
    assert len(best) < len(b) - 900 and any(k == "copy" for k, _, _ in _tags(best))
    assert U.decode(best, len(b))[1] == b


def _rand(n, seed):
    return np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8).tobytes()


def test_match_only_at_s_plus_2():
    """At s = 100 only a 4-byte match exists (offset 80); two bytes later a 40-byte one (offset 42) starts, which no
    probe reaches before the 4-byte match would be emitted.  The search at s+2 takes the longer match."""
    d = _rand(42, 3)                         # the data at 100: two bytes, then the 40 bytes of the source at 60
    src = bytearray(_rand(300, 2))
    src[20:24] = d[:4]                       # 4-byte source of the match at s
    src[60:100] = d[2:]                      # 40-byte source of the match at s+2
    src[100:142] = d
    src = bytes(src)
    assert src[24] != src[104]
    comp = U.encode(src, U.BEST)
    assert U.decode(comp, len(src))[1] == src
    copies = [(o, ln) for k, o, ln in _tags(comp) if k == "copy"]
    assert (42, 40) in copies and (80, 4) not in copies, copies


def test_repeat_at_s_plus_1():
    """After a copy at offset d, data that matches at offset d again one byte later is emitted as a repeat tag."""
    blk = _rand(64, 4)
    src = blk + _rand(3, 5) + blk[:40] + b"Z" + blk[41:64] + _rand(200, 6)
    comp = U.encode(src, U.BEST)
    assert U.decode(comp, len(src))[1] == src
    kinds = [k for k, _, _ in _tags(comp)]
    assert "rep" in kinds and kinds.index("rep") > kinds.index("copy"), kinds


def test_match_end_probe_finds_longer():
    """A 64-byte run x at 100, then two copies of its first 10 bytes at 300 and 350, then x again at 400.  At 400 the
    table candidates (both slots of both tables) are the two 10-byte heads; the match-end probe at 409 finds the run
    at 100 through the long table and replaces the 10-byte match by the 64-byte one at offset 300."""
    x = _rand(64, 7)
    src = bytearray(_rand(600, 8))
    src[100:164] = x
    src[300:310] = x[:10]
    src[350:360] = x[:10]
    src[400:464] = x
    src = bytes(src)
    comp = U.encode(src, U.BEST)
    assert U.decode(comp, len(src))[1] == src
    copies = [(o, ln) for k, o, ln in _tags(comp) if k == "copy"]
    assert (300, 64) in copies, copies
