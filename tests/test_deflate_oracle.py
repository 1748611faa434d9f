"""The StatelessDeflate oracle (oracle/orc_deflate.c) against the reference's golden outputs, Python's zlib and gzip, and
the inflate oracle."""
import ctypes
import gzip as pygzip
import json
import os
import struct
import zlib

import numpy as np

import deflate_util as D
import flate_util as F


def _inflate(s):
    return zlib.decompress(s, -15)


def test_block_huff_golden():
    # huffman_bit_writer_test.go testBlockHuff: writeBlockHuff(false, in, false) with logNewTablePenalty = 8
    names = [n for n in D.testdata_names() if n.endswith(".golden") and n.startswith("flate/huffman-")]
    assert len(names) >= 9
    for g in names:
        data = D.testdata(g[:-len(".golden")] + ".in")
        out = ctypes.create_string_buffer(len(data) * 2 + 1024)
        r = D.oracle().orc_deflate_block_huff(data, len(data), 8, out, len(out))
        assert out.raw[:r] == D.testdata(g), g


def test_block_dynamic_golden():
    # testBlock "dyn" and "sync": writeBlockDynamic(&tok, false, input, sync) with and without the input
    tests = json.load(open(os.path.join(D.GOLDEN, "flate_block_tokens.json")))
    n = 0
    for t in tests:
        toks = np.array(t["tokens"], dtype=np.uint32)
        for kind, sync in (("dyn", 0), ("sync", 1)):
            cases = [(None, t["wantNoInput"])]
            if t["input"]:
                cases.append((D.testdata("flate/" + os.path.basename(t["input"])), t["want"]))
            for data, want in cases:
                out = ctypes.create_string_buffer(1 << 17)
                r = D.oracle().orc_deflate_block_dynamic(toks.ctypes.data, len(toks), data, len(data) if data else 0, sync,
                                                         out, len(out))
                assert out.raw[:r] == D.testdata("flate/" + os.path.basename(want % kind)), (want, kind)
                n += 1
    assert n == 34


def test_pool_round_trip():
    for label, data in D.pool():
        for eof in (True, False):
            s = D.stateless(data, eof)
            assert _inflate(s + (b"" if eof else b"\x03\x00")) == data, (label, len(data), eof)
            if eof:
                r, back = F.orc_decode(F.RAW, s, len(data) + 16)
                assert r == len(data) and back == data, (label, len(data))
            else:
                assert s.endswith(b"\x00\x00\xff\xff")


def test_empty_calls():
    assert D.stateless(b"", True) == b"\x03\x00"
    assert D.stateless(b"", False) == b"\x00\x00\x00\xff\xff"


def test_dict_round_trip():
    for data, d in D.dict_cases():
        s = D.stateless(data, True, d)
        dd = d[-8192:]
        z = zlib.decompressobj(-15, zdict=dd) if dd else zlib.decompressobj(-15)
        assert z.decompress(s) + z.flush() == data, (len(data), len(d))


def test_fuzz_corpus():
    ins = D.fuzz_inputs()
    assert len(ins) == 1995
    for data in ins:
        s = b"".join(D.stateless(p, eof, dc) for p, eof, dc in D.fuzz_split(data))
        assert _inflate(s) == data


def test_gzip_members():
    data = D.text(__import__("random").Random(2), 90000)
    hdr = b"\x1f\x8b\x08" + bytes([8 | 16]) + struct.pack("<I", 1234567) + b"\x00\x03" + b"name.txt\x00" + b"a comment\x00"
    m = D.gzip_member(data, hdr)
    assert pygzip.decompress(m) == data
    assert m[:len(hdr)] == hdr
    assert m[len(hdr):-8] == D.stateless(data, False) + D.stateless(b"", True)
    assert struct.unpack("<II", m[-8:]) == (zlib.crc32(data), len(data))
    assert pygzip.decompress(D.gzip_member(b"")) == b""


def test_every_decision_path():
    D.oracle().orc_deflate_paths_reset()
    for label, data in D.pool():
        D.stateless(data, True)
    for data, d in D.dict_cases():
        D.stateless(data, True, d)
    for n in (3 * D.STEP + 7, 4 * D.STEP):
        D.stateless(D.huff_runs(n), False)
    p = D.paths()
    for k in ("stored_empty_tokens", "huff_stored_test", "huff_stored_est", "huff_new", "huff_reuse", "dyn_new",
              "dyn_reuse", "dyn_fixed", "eob_before_stored", "long_match"):
        assert p[k] > 0, (k, p)


def test_huffman_reuse_runs():
    # consecutive non-final Huffman-only blocks keep the first one's table; the stream reads back
    for n in (3 * D.STEP + 7, 4 * D.STEP, 5 * D.STEP):
        data = D.huff_runs(n)
        D.oracle().orc_deflate_paths_reset()
        s = D.stateless(data, False)
        assert D.paths()["huff_reuse"] >= 1
        assert _inflate(s + b"\x03\x00") == data


def test_huffman_reuse_final_block_is_not_final():
    # writeBlockHuff (huffman_bit_writer.go:1055-1068) reuses the table in force without checking eof, unlike
    # writeBlockDynamic (:631): when the final block reuses, no header is written, so no BFINAL bit is set and the
    # reference's stream holds every byte but has no final block.  The oracle keeps that.
    data = D.huff_runs(4 * D.STEP)
    s = D.stateless(data, True)
    z = zlib.decompressobj(-15)
    assert z.decompress(s) == data and not z.eof
    assert F.orc_decode(F.RAW, s, len(data) + 16)[0] == -12     # io.ErrUnexpectedEOF from the reference's reader
