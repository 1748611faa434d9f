"""The BestSpeed oracle (oracle/orc_deflate.c: fastEncL1, the compressor's write / storeFast / close, the zlib and gzip
writers' framing): the reference's test vector, read-back by Python's zlib / gzip and by the inflate oracle on the seeded
pool, the reference's encoder fuzz corpus and its huffman-*.in inputs, the Writes' boundaries, and every decision path."""
import gzip
import random
import zlib

import pytest

import flate_best_speed_util as D
import flate_util as F


def _read_back(data, fmt, out):
    if fmt == D.RAW:
        assert zlib.decompress(out, -15) == data
    elif fmt == D.ZLIB:
        assert out[:2] == b"\x78\x01" and zlib.decompress(out) == data
    else:
        assert out[:10] == D.GZIP_HDR_BEST_SPEED and gzip.decompress(out) == data
    r, back = F.orc_decode(fmt, out, len(data) + 1)
    assert r == len(data) and back == data


def test_empty_input_vector():
    # deflate_test.go:46, deflateTests row 7: level 1 on empty input writes 03 00
    assert D.best_speed(b"") == b"\x03\x00"
    assert D.best_speed(b"", D.ZLIB) == b"\x78\x01\x03\x00\x00\x00\x00\x01"


def test_container_headers():
    z = D.best_speed(b"hello", D.ZLIB)
    assert z[:2] == b"\x78\x01" and z[-4:] == zlib.adler32(b"hello").to_bytes(4, "big")
    from compress_b200 import gzip as g
    hdr = g.header_bytes(level=g.BestSpeed)
    assert hdr[8] == 4 and g.header_bytes()[8] == 0 and hdr == D.GZIP_HDR_BEST_SPEED
    out, ck = D.best_speed(b"hello", D.GZIP, hdr, check=True)
    assert out[8] == 4 and ck == zlib.crc32(b"hello")
    assert out[-8:] == zlib.crc32(b"hello").to_bytes(4, "little") + (5).to_bytes(4, "little")


@pytest.mark.parametrize("fmt", [D.RAW, D.ZLIB, D.GZIP])
def test_pool_reads_back(fmt):
    for label, data in D.pool():
        _read_back(data, fmt, D.best_speed(data, fmt))


def test_fuzz_corpus_reads_back():
    for i, data in enumerate(D.fuzz_inputs()):
        _read_back(data, (D.RAW, D.ZLIB, D.GZIP)[i % 3], D.best_speed(data, (D.RAW, D.ZLIB, D.GZIP)[i % 3]))


def test_huffman_inputs_read_back():
    names = [n for n in D.testdata_names() if n.startswith("flate/huffman-") and n.endswith(".in")]
    assert len(names) >= 9
    for n in names:
        data = D.testdata(n)
        for fmt in (D.RAW, D.ZLIB, D.GZIP):
            _read_back(data, fmt, D.best_speed(data, fmt))


def test_writes_boundaries_do_not_matter():
    # the compressor stores a window only when it is full and more bytes arrive, so any split of the input into Writes
    # (empty ones included) writes the same member
    rng = random.Random(3)
    for n in (0, 100, D.WINDOW, 3 * D.WINDOW + 5, 6 * D.WINDOW + 1):
        data = D.text(rng, n)
        one = D.best_speed(data, D.GZIP)
        for _ in range(3):
            cuts = sorted(rng.randint(0, n) for _ in range(rng.randint(0, 6))) + [D.WINDOW * k for k in range(1, 3) if D.WINDOW * k <= n]
            cuts = sorted(cuts)
            writes = [b - a for a, b in zip([0] + cuts, cuts + [n])] + [0]
            assert D.best_speed(data, D.GZIP, writes=writes) == one


def test_dst_small_and_cap():
    data = D.text(random.Random(1), 100000)
    out = D.best_speed(data)
    assert D.best_speed(data, cap=len(out) - 1) == -4
    assert D.best_speed(data, cap=len(out)) == out
    assert len(out) <= D.bound(len(data))


def test_bound_holds_on_incompressible_and_skewed_input():
    rng = random.Random(2)
    for data in (rng.randbytes(5 * D.WINDOW + 9), D.skewed(rng, 4 * D.WINDOW), D.huff_runs(3 * D.WINDOW), bytes(range(256)) * 300):
        assert len(D.best_speed(data)) <= D.bound(len(data))


def test_decision_paths():
    D.paths_reset()
    for _, data in D.pool():
        D.best_speed(data)
    for data in D.fuzz_inputs():
        D.best_speed(data)
    for n in D.testdata_names():
        if n.startswith("flate/huffman-") and n.endswith(".in"):
            D.best_speed(D.testdata(n))
    p = D.paths()
    # storeFast: stored (no tokens), Huffman-only, dynamic, and the short last window stored (<= 32) or Huffman-only
    for k in ("sf_stored", "sf_huff", "sf_dyn", "sf_final_stored", "sf_final_huff"):
        assert p[k] > 0, (k, p)
    # writeBlockDynamic: new table, reuse, fixed, stored; writeBlockHuff: a new table
    for k in ("dyn_new", "dyn_reuse", "dyn_fixed", "dyn_stored", "huff_new"):
        assert p[k] > 0, (k, p)
    # fastEncL1: matches into earlier windows, the history move before the sixth window, a length split above 258, and
    # backward extension stopped by the start of e.hist
    for k in ("l1_prev_window", "l1_hist_move", "long_match", "l1_back_stop"):
        assert p[k] > 0, (k, p)
    # After a move e.hist starts 32 768 bytes before the window, and a match reaches at most 32 768 back: its source is at
    # e.hist's start only when the match starts at the window's start, where nextEmit already stops the extension.  So the
    # moved start never stops one -- it bounds the extension exactly where the window start does.
    assert p["l1_back_stop_moved"] == 0, p
