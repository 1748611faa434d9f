"""The LZ4 / LZ4s -> S2 / Snappy converter oracle (oracle/orc_lz4.c) and its lz4ref restatement, pinned by vectors written
from the block formats by hand, the reference fuzz test's invariants over its seeds (s2/lz4convert_test.go:354-448) and
round trips.  CPU only."""
import pytest

import lz4_util as U
from test_oracle_s2 import s2_decode

BIG = 1 << 26
ABCD = b"abcd"


def body(src, lz4s=False, snappy=False):
    r, b, n = U.convert(src, BIG, lz4s, snappy)
    assert r >= 0, r
    return b, n


def h(s):
    return bytes.fromhex(s.replace(" ", ""))


def test_empty_source_appends_nothing():
    r, b, n = U.convert(b"", 0, prefix=b"xyz")
    assert (r, b, n) == (3, b"", 0)


@pytest.mark.parametrize("ll,hdr", [(1, "00"), (60, "ec"), (61, "f03c"), (256, "f0ff"), (257, "f40001"), (65536, "f4ffff"),
                                    (65537, "f8000001"), (1 << 24, "f8ffffff"), ((1 << 24) + 1, "fc00000001")])
def test_literal_headers(ll, hdr):
    lits = b"\x99" * ll
    for snappy in (False, True):
        assert body(U.block([], lits), snappy=snappy) == (h(hdr) + lits, ll)


@pytest.mark.parametrize("ml,tag", [(4, "0104"), (11, "1d04"), (12, "2e0400"), (64, "fe0400"),
                                    (65, "1104 150031"),             # > 64, offset < 2048: copy1 of 8, then a 3-byte repeat
                                    (70, "1104 150036")])
def test_copies_offset_below_2048(ml, tag):
    b, n = body(U.block([(ABCD, 4, ml)], b"x"))
    assert b == h("0c61626364") + h(tag) + h("0078") and n == 4 + ml + 1


def test_copies_offset_2048_and_above():
    lits = bytes(range(256)) * 12
    lits = lits[:3000]
    hdr = h("f4b70b")                                                 # 3000 literals: 3-byte header, n - 1 = 2999
    assert body(U.block([(lits, 3000, 4)], b"x"))[0] == hdr + lits + h("0eb80b") + h("0078")
    assert body(U.block([(lits, 3000, 64)], b"x"))[0] == hdr + lits + h("feb80b") + h("0078")
    # > 64: copy2 of 60, the rest (5) as a repeat
    assert body(U.block([(lits, 3000, 65)], b"x"))[0] == hdr + lits + h("eeb80b 0500") + h("0078")
    # a repeat of 4 .. 8 bytes at an offset >= 2048 keeps the zero-offset form; 9 .. 11 takes the 3-byte form
    assert body(U.block([(lits, 3000, 4), (b"", 3000, 9)], b"x"))[0] == hdr + lits + h("0eb80b 150001") + h("0078")


@pytest.mark.parametrize("ml,tag", [
    (4, "0100"), (8, "1100"),
    (9, "1504"),                                  # length - 4 < 8 at an offset < 2048: a copy1 that states the offset
    (12, "150004"), (263, "1500ff"),              # 3-byte repeat
    (264, "19000400"), (65795, "1900ffff"),       # 4-byte repeat
    (65796, "1d00000100"),                        # 5-byte repeat
    (4 + 65536 + (1 << 24), "1d00fbffff 0500"),   # above 2^24 - 1 + 2^16: split into a 5-byte repeat and the rest
])
def test_repeats(ml, tag):
    b, n = body(U.block([(ABCD, 4, 4), (b"", 4, ml)], b"x"))
    assert b == h("0c61626364 0104") + h(tag) + h("0078") and n == 4 + 4 + ml + 1


@pytest.mark.parametrize("ml,tag", [(4, "0104"), (12, "2e0400"), (64, "fe0400"), (65, "fe0400 020400"), (67, "fe0400 0a0400"),
                                    (128, "fe0400 fe0400"), (140, "fe0400 fe0400 2e0400")])
def test_snappy_pieces(ml, tag):
    b, n = body(U.block([(ABCD, 4, ml)], b"x"), snappy=True)
    assert b == h("0c61626364") + h(tag) + h("0078") and n == 4 + ml + 1


def test_snappy_has_no_repeats():
    assert body(U.block([(ABCD, 4, 4), (b"", 4, 4)], b"x"), snappy=True)[0] == h("0c61626364 0104 0104 0078")


def test_lz4s_tokens_without_match():
    # 0x30 "abc": match length 3 = no match; 0x00 in the middle emits nothing; 0x11 "d" + offset 4, length 4; final 0x00
    src = h("30616263 00 1164 0400 00")
    for snappy in (False, True):
        assert body(src, lz4s=True, snappy=snappy) == (h("08616263 0064 0104"), 8)
    assert U.block([(b"abc", None, None), (b"", None, None), (b"d", 4, 4)], lz4s=True) == src
    # LZ4 reads the same bytes as a match of 4 after "abc": offset 0x0100 > 3 bytes produced
    assert U.convert(src, BIG)[0] == U.CORRUPT
    # an LZ4s match length of 18 needs the extension byte
    b, n = body(U.block([(ABCD, 4, 18), (b"", 4, 40)], lz4s=True), lz4s=True)
    assert b == h("0c61626364 460400 150020") and n == 4 + 18 + 40


def test_final_token_rule():
    assert body(h("30616263")) == (h("08616263"), 3)
    assert body(h("40 61626364 0400 00")) == (h("0c61626364 0104"), 8)
    assert U.convert(h("31616263"), BIG)[0] == U.CORRUPT            # a match code on the last token needs an offset
    assert U.convert(h("40 61626364 0400"), BIG)[0] == U.CORRUPT     # a match must not end the block


@pytest.mark.parametrize("src", [
    "f0", "f0ff",                                # literal length extension runs off the end
    "3061 62",                                   # literals run off the end (s + ll >= len(src))
    "41 61626364 04", "41 61626364 0400",        # fewer than 3 bytes after the literals
    "41 61626364 0000 00",                       # offset 0
    "41 61626364 0500 00",                       # offset beyond what was produced
    "4f 61626364 0400 ff", "4f 61626364 0400 05",   # match length extension ends the input
])
def test_corrupt(src):
    for lz4s in (False, True):
        for snappy in (False, True):
            assert U.convert(h(src), BIG, lz4s, snappy)[0] == U.CORRUPT, (src, lz4s, snappy)


def test_match_length_extension():
    assert body(h("4f 61626364 0400 05 00")) == (h("0c61626364 5e0400"), 28)


def test_capacity_edges():
    src = U.block([], b"abc")                     # d + ll > dLimit before the literals; the last run is not checked after
    assert U.convert(src, 13)[0] == 4 and U.convert(src, 12)[0] == U.DST_SMALL
    src = U.block([(ABCD, 4, 4)], b"x")           # after the copy: d = 7 must be <= dLimit = avail - 10
    for snappy in (False, True):
        assert U.convert(src, 18, snappy=snappy)[0] == 9 and U.convert(src, 17, snappy=snappy)[0] == U.DST_SMALL
    # the decision depends only on cap(dst) - len(dst)
    assert U.convert(src, 18, prefix=b"p" * 100)[0] == 109 and U.convert(src, 17, prefix=b"p" * 100)[0] == U.DST_SMALL


def test_inlined_emitter_room_is_dst_too_small():
    # 3000 literals (3-byte header) end exactly at dLimit and leave 7 bytes; the copy needs 8 (copy2 of 60 + a 5-byte
    # repeat).  The reference's inlined emitter only checks for 5 bytes of room and writes past cap(dst) (a panic in Go).
    lits = (bytes(range(256)) * 12)[:3000]
    src = U.block([(lits, 3000, 70000)], b"x")
    assert U.convert(src, 3010)[0] == U.DST_SMALL
    r, b, n = U.convert(src, 4000)
    assert r == 3000 + 3 + 8 + 2 and b.endswith(h("eeb80b 1d003011 00 0078"))
    # the smallest slot: dLimit = slot - 5 - 10 must hold the last literal run's start (3003 + 8 + 1)
    assert U.min_cap(src) == 3000 + 3 + 8 + 1 + 10 + 5


def test_record_bound():
    for lz4s in (False, True):
        rc = 2 if lz4s else 3
        for src in U.pool(seed=3, lz4s=lz4s):
            if U.convert(src, BIG, lz4s)[0] >= 0:
                assert U.record_count(src, lz4s) <= len(src) // rc + 1
        # densest blocks: back to back 3-byte sequences, and LZ4s literal-only tokens of one byte
        dense = U.block([(b"a", 1, 4)] + [(b"", 1, 4)] * 1000, b"z")
        assert U.record_count(dense) == 1002 and 1002 <= len(dense) // 3 + 1
        dense_s = U.block([(b"a", None, None)] * 1000, lz4s=True)
        assert U.record_count(dense_s, True) == 1000 and 1000 <= len(dense_s) // 2 + 1


def _fuzz_one(data):
    """FuzzLZ4Block's body (s2/lz4convert_test.go:365-447) with the oracle."""
    lzN, lz4Decoded = U.uncompress(data, len(data) * 2 + 65536)
    size = len(data) * 2 + 4096
    hdr = U.uvarint(lzN) if lzN >= 0 else b""
    r, cV, cN = U.convert(data, size - len(hdr), prefix=hdr)
    if lzN >= 0 and r >= 0:
        assert cN == lzN
        n, dec = s2_decode(hdr + cV, lzN)
        assert n == lzN and dec == lz4Decoded
    elif lzN >= 0:
        pytest.fail("lz4 decoded %d bytes, the conversion failed with %d" % (lzN, r))
    elif r >= 0:
        lzN, lz4Decoded = U.uncompress(data, cN)
        assert lzN >= 0
        n, dec = s2_decode(U.uvarint(cN) + cV, cN)
        assert n == cN and dec == lz4Decoded
    hdr = U.uvarint(lzN) if lzN >= 0 else U.uvarint(0)
    r, cV, cN = U.convert(data, size - len(hdr), snappy=True, prefix=hdr)
    if lzN >= 0 and r >= 0:
        assert cN == lzN
        n, dec = s2_decode(hdr + cV, lzN)
        assert n == lzN and dec == lz4Decoded and not has_repeat(cV)
        return
    if lzN >= 0:
        assert r == U.DST_SMALL                   # Snappy can expand a lot (64-byte match pieces)
    else:
        assert r < 0


def has_repeat(body_):
    """Whether an S2 body holds a repeat tag (copy1 with offset 0), which Snappy decoders refuse."""
    s = 0
    while s < len(body_):
        t = body_[s]
        if t & 3 == 0:
            x = t >> 2
            nb = 0 if x < 60 else x - 59
            ln = (x if nb == 0 else int.from_bytes(body_[s + 1:s + 1 + nb], "little")) + 1
            s += 1 + nb + ln
        elif t & 3 == 1:
            if ((t & 0xE0) << 3 | body_[s + 1]) == 0:
                return True
            s += 2
        else:
            s += 3 if t & 3 == 2 else 5
    return False


def test_reference_fuzz_seeds():
    seeds = U.fuzz_seeds()
    assert len(seeds) == 108 + 244
    for name, data in seeds:
        if 0 < len(data) <= (1 << 20):
            _fuzz_one(data)


@pytest.mark.parametrize("lz4s", [False, True])
def test_pool_round_trips(lz4s):
    for src in U.pool(seed=5, lz4s=lz4s):
        for snappy in (False, True):
            r, b, n = U.convert(src, 4 * len(src) + 64, lz4s, snappy)
            if r < 0:
                continue
            dn, dec = s2_decode(U.uvarint(n) + b, n)
            assert dn == n
            if not lz4s and src:
                assert U.uncompress(src, n) == (n, dec)


def test_lz4ref_round_trip_and_zeros():
    import helpers as H
    tw = H.golden("twain.txt")
    for lz4s in (False, True):
        blk = U.compress(tw, lz4s)
        r, b, n = U.convert(blk, 2 * len(tw), lz4s)
        assert n == len(tw) and s2_decode(U.uvarint(n) + b, n)[1] == tw
    blk = U.compress(tw)
    assert U.uncompress(blk, len(tw)) == (len(tw), tw)
    assert U.uncompress(blk, len(tw) - 1)[0] < 0
    z = bytes(17 << 20)                           # one match of ~17 MiB: the S2 repeat is split
    blk = U.compress(z)
    r, b, n = U.convert(blk, 1 << 16)
    assert n == len(z) and len(b) < 64 and s2_decode(U.uvarint(n) + b, n)[1] == z
