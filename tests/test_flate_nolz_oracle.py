"""The HuffmanOnly / NoCompression oracle (oracle/orc_flate_nolz.c: init's two branches, store, storeHuff, the
compressor's write / close, the zlib and gzip framing over orc_deflate.c's bit writer): the reference's test vectors and
size limits, read-back by Python's zlib / gzip and by the inflate oracle on the seeded pool and the encoder fuzz corpus,
the Writes' boundaries, and every decision path."""
import gzip
import os
import random
import zlib

import pytest

import flate_nolz_util as D
import flate_util as F

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _read_back(data, level, fmt, out):
    if fmt == D.RAW:
        assert zlib.decompress(out, -15) == data
    elif fmt == D.ZLIB:
        assert out[:2] == b"\x78\x01" and zlib.decompress(out) == data
    else:
        assert out[:10] == D.GZIP_HDR and gzip.decompress(out) == data
    assert len(out) <= D.bound(level, len(data)) + D.container(fmt)
    r, back = F.orc_decode(fmt, out, len(data) + 1)
    assert r == len(data) and back == data


def test_reference_vectors():
    # deflate_test.go:36-45, deflateTests rows 0 and 4-6 (level 0)
    assert D.nolz(b"", 0) == b"\x03\x00"
    assert D.nolz(b"\x11", 0) == bytes([0x0, 0x1, 0x0, 0xfe, 0xff, 0x11, 0x3, 0x0])
    assert D.nolz(b"\x11\x12", 0) == bytes([0x0, 0x2, 0x0, 0xfd, 0xff, 0x11, 0x12, 0x3, 0x0])
    assert D.nolz(b"\x11" * 8, 0) == bytes([0x0, 0x8, 0x0, 0xf7, 0xff]) + b"\x11" * 8 + b"\x03\x00"
    # an empty input writes only Close's block at -2 as well
    assert D.nolz(b"", -2) == b"\x03\x00"
    assert D.nolz(b"", -2, D.ZLIB) == b"\x78\x01\x03\x00\x00\x00\x00\x01"


@pytest.mark.parametrize("name,limits", [("e.txt", (100018, 43683 + 100)), ("twain.txt", (387999, 233460 + 100))])
def test_size_limits(name, limits):
    # deflate_test.go:403-414, deflateInflateStringTests: limit[0] is level 0, limit[10] ConstantCompression
    with open(os.path.join(GOLDEN, name), "rb") as f:
        data = f.read().replace(b"\r", b"")
    for level, limit in zip((0, -2), limits):
        out = D.nolz(data, level)
        assert len(out) <= limit, (name, level, len(out))
        _read_back(data, level, D.RAW, out)


def test_container_headers():
    for level in D.LEVELS:
        z, ck = D.nolz(b"hello", level, D.ZLIB, check=True)
        assert z[:2] == b"\x78\x01" and z[-4:] == zlib.adler32(b"hello").to_bytes(4, "big") and ck == zlib.adler32(b"hello")
        out, ck = D.nolz(b"hello", level, D.GZIP, check=True)
        assert out[8] == 0 and ck == zlib.crc32(b"hello")
        assert out[-8:] == zlib.crc32(b"hello").to_bytes(4, "little") + (5).to_bytes(4, "little")
    from compress_b200 import gzip as g
    for level in (g.HuffmanOnly, g.NoCompression):
        assert g.header_bytes(level=level) == D.GZIP_HDR          # XFL 0, Go's zero ModTime, OS 255


@pytest.mark.parametrize("level", D.LEVELS)
@pytest.mark.parametrize("fmt", D.FORMATS)
def test_pool_reads_back(level, fmt):
    for label, data in D.pool():
        _read_back(data, level, fmt, D.nolz(data, level, fmt))


@pytest.mark.parametrize("level", D.LEVELS)
def test_fuzz_corpus_reads_back(level):
    for i, data in enumerate(D.fuzz_inputs()):
        fmt = D.FORMATS[i % 3]
        _read_back(data, level, fmt, D.nolz(data, level, fmt))


@pytest.mark.parametrize("level", D.LEVELS)
def test_writes_boundaries_do_not_matter(level):
    # a window is written only when it is full and more bytes arrive, so any split of the input into Writes (empty ones
    # included) writes the same member
    rng = random.Random(5)
    w = D.WINDOW[level]
    for n in (0, 100, w, 3 * w + 5, 4 * w):
        data = D.text(rng, n)
        one = D.nolz(data, level, D.GZIP)
        for _ in range(3):
            cuts = sorted([rng.randint(0, n) for _ in range(rng.randint(0, 6))] + [w * k for k in (1, 2) if w * k <= n])
            writes = [b - a for a, b in zip([0] + cuts, cuts + [n])] + [0]
            assert D.nolz(data, level, D.GZIP, writes=writes) == one


@pytest.mark.parametrize("level", D.LEVELS)
def test_dst_small_and_cap(level):
    data = D.text(random.Random(1), 100000)
    out = D.nolz(data, level)
    assert D.nolz(data, level, cap=len(out) - 1) == -4
    assert D.nolz(data, level, cap=len(out)) == out


def test_bound_holds_on_adversarial_windows():
    # a window with few distinct bytes leaves a short header in force; a skewed window over all 256 values after it
    # replaces that table, and its real header is far longer than the lastHeader estBits counted
    rng = random.Random(2)
    few = (b"ab" * 16384)
    for data in (few + D.skewed(rng, 32768) + few + D.skewed(rng, 40000), rng.randbytes(5 * 32768 + 9),
                 D.huff_runs(3 * 32768), D.equal256(4 * 32768 + 3)):
        assert len(D.nolz(data, -2)) <= D.bound(-2, len(data))


def test_decision_paths():
    D.paths_reset()
    for _, data in D.pool():
        D.nolz(data, -2)
    for data in D.fuzz_inputs():
        D.nolz(data, -2)
    rng = random.Random(4)
    few = b"ab" * 16384
    D.nolz(few + D.skewed(rng, 32768) + D.skewed(rng, 20000), -2)
    p = D.paths()
    # writeBlockHuff: stored by the float64 test, stored by the estimate at <= 1 024 and > 1 024 bytes, a new table,
    # reuse, a new table that first writes the owed EOB, and a stored window that first writes the owed EOB
    for k in ("huff_stored_test", "est_stored_small", "est_stored_large", "huff_new", "huff_reuse", "new_owes_eob",
              "eob_before_stored"):
        assert p[k] > 0, (k, p)
    # the last window: full (its block written with sync at Close) and tiny; and the empty input
    for k in ("final_full", "final_tiny", "empty"):
        assert p[k] > 0, (k, p)
