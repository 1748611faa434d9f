"""StatelessDeflate and gzip members at StatelessCompression on the device: bytes equal to the oracle's (and so to the
reference's) through both entry points, at several batch shapes, across scratch passes, with dicts, and read back by the
device inflate and by Python's zlib / gzip."""
import gzip as pygzip
import io
import random
import zlib

import numpy as np
import pytest
import torch

import deflate_util as D

pytestmark = pytest.mark.gpu

HDR = b"\x1f\x8b\x08\x00\x00\x00\x00\x00\x00\xff"


@pytest.fixture(scope="module")
def enc():
    from compress_b200 import flate
    e = flate.Encoder()
    yield e
    e.close()


def _want(data, fmt, eof=True, dict=None, header=HDR):
    return D.gzip_member(data, header) if fmt == 2 else D.stateless(data, eof, dict)


def _device(enc, inputs, fmt, eofs=None, dicts=None, header=HDR, offsets=False, stream=None, cap=None):
    """encode_device over a packed (offsets) or strided batch; returns (outputs, codes)."""
    n = len(inputs)
    stride = max(1, max(len(b) for b in inputs))
    hdr = header if fmt == 2 else b""
    if offsets:
        offs, buf, pos = [], bytearray(), 0
        for b in inputs:
            pos += 1 + (len(buf) % 3)                    # unaligned starts
            buf += bytes(pos - len(buf)) if pos > len(buf) else b""
            offs.append(len(buf)); buf += b
            pos = len(buf)
        src = torch.frombuffer(bytearray(buf) + bytearray(8), dtype=torch.uint8).cuda()
        so = torch.tensor(offs, dtype=torch.int64).cuda()
    else:
        a = np.zeros((n, stride), dtype=np.uint8)
        for i, b in enumerate(inputs):
            a[i, :len(b)] = np.frombuffer(b, dtype=np.uint8)
        src, so = torch.from_numpy(a).cuda().reshape(-1), None
    sizes = torch.tensor([len(b) for b in inputs], dtype=torch.int32).cuda()
    kw = {}
    if eofs is not None:
        kw["eof"] = torch.tensor([1 if e else 0 for e in eofs], dtype=torch.uint8).cuda()
    if dicts is not None:
        dl = [d or b"" for d in dicts]
        kw["dict"] = torch.frombuffer(bytearray(b"".join(dl) + b"\0"), dtype=torch.uint8).cuda()
        kw["dict_offsets"] = torch.tensor(np.cumsum([0] + [len(d) for d in dl])[:-1], dtype=torch.int64).cuda()
        kw["dict_sizes"] = torch.tensor([len(d) for d in dl], dtype=torch.int32).cuda()
    with torch.cuda.stream(stream or torch.cuda.current_stream()):
        dst, out = enc.encode_device(src, sizes, stride, dst_cap=cap, format=fmt, header=hdr, src_offsets=so, **kw)
    torch.cuda.synchronize()
    out = out.cpu().numpy()
    d = dst.cpu().numpy()
    return [d[i, :out[i]].tobytes() if out[i] >= 0 else None for i in range(n)], [int(x) for x in out]


@pytest.mark.parametrize("fmt", [0, 2])
def test_pool_both_entry_points(enc, fmt):
    pool = [d for _, d in D.pool()]
    want = [_want(d, fmt) for d in pool]
    outs, codes, crcs = enc.encode_chunks(pool, format=fmt, header=HDR if fmt == 2 else b"")
    assert outs == want
    assert crcs == [zlib.crc32(d) for d in pool]
    got, _ = _device(enc, pool, fmt)
    assert got == want
    got, _ = _device(enc, pool, fmt, offsets=True)
    assert got == want


def test_eof_false_and_dicts(enc):
    cases = D.dict_cases()
    ins = [c[0] for c in cases]
    dicts = [c[1] for c in cases]
    eofs = [i % 2 == 0 for i in range(len(ins))]
    want = [D.stateless(d, e, dc) for d, e, dc in zip(ins, eofs, dicts)]
    assert enc.encode_chunks(ins, eof=eofs, dicts=dicts)[0] == want
    assert _device(enc, ins, 0, eofs=eofs, dicts=dicts)[0] == want


def test_fuzz_corpus(enc):
    items = [p for data in D.fuzz_inputs() for p in D.fuzz_split(data)]
    ins, eofs, dicts = [p[0] for p in items], [p[1] for p in items], [p[2] for p in items]
    want = [D.stateless(d, e, dc) for d, e, dc in items]
    assert enc.encode_chunks(ins, eof=eofs, dicts=dicts)[0] == want
    assert _device(enc, ins, 0, eofs=eofs, dicts=dicts, offsets=True)[0] == want


@pytest.mark.parametrize("n", [1, 31, 32, 33, 4097])
def test_batch_shapes(enc, n):
    rng = random.Random(n)
    ins = [D.text(rng, rng.randint(0, 3 * D.STEP)) if i % 3 else rng.randbytes(rng.randint(0, 40000)) for i in range(n)]
    if n == 4097:
        ins = [b[:rng.randint(0, 3000)] for b in ins]
    for fmt in (0, 2):
        want = [_want(d, fmt) for d in ins]
        assert _device(enc, ins, fmt, offsets=n != 32)[0] == want, (n, fmt)


PASS_SLOTS = 8192                                     # kDflPassSlots: block slots per scratch pass


def test_long_inputs_across_passes(enc):
    # 4 x 64 MiB: 2 731 blocks each at slots i * 2 731 + k.  Input 2's blocks are slots 5 462 .. 8 192 and a pass holds
    # 8 192 slots, so its last block is parsed and encoded in the second pass, from the writer state the first one saved
    rng = random.Random(9)
    unit = D.text(rng, 1 << 20) + rng.randbytes(1 << 18)
    n = 64 << 20
    big = [(unit * 64)[:n]] + [bytes(x ^ k for x in unit[:4096]) * (n // 4096) for k in (1, 2, 3)]
    assert all(len(b) == n for b in big)
    mb = D.blocks(n)
    spans = [(i * mb, i * mb + D.blocks(len(b)) - 1) for i, b in enumerate(big)]
    assert any(a < PASS_SLOTS <= b for a, b in spans), spans
    want = [D.stateless(b) for b in big]
    got, codes = _device(enc, big, 0)
    assert codes == [len(w) for w in want]
    assert got == want
    assert zlib.decompress(got[0], -15) == big[0]


def test_huffman_reuse_runs(enc):
    runs = [D.huff_runs(n) for n in (3 * D.STEP + 7, 4 * D.STEP, 5 * D.STEP)]
    for eof in (False, True):
        want = [D.stateless(r, eof) for r in runs]
        assert enc.encode_chunks(runs, eof=[eof] * 3)[0] == want
        assert _device(enc, runs, 0, eofs=[eof] * 3)[0] == want


def test_input_larger_than_stride(enc):
    # the device call sizes its block slots from src_stride: a larger input is B2C_ERR_ARG and its neighbours are intact
    rng = random.Random(12)
    ins = [D.text(rng, 30000), D.text(rng, 40000), D.text(rng, 30000)]
    stride = 30000
    a = np.zeros(3 * stride + 10000, dtype=np.uint8)
    offs = [0, stride, 2 * stride]
    for o, b in zip(offs, ins):
        a[o:o + len(b)] = np.frombuffer(b, dtype=np.uint8)
    src = torch.from_numpy(a).cuda()
    sizes = torch.tensor([len(b) for b in ins], dtype=torch.int32).cuda()
    so = torch.tensor(offs, dtype=torch.int64).cuda()
    dst, out = enc.encode_device(src, sizes, stride, src_offsets=so)
    torch.cuda.synchronize()
    out = out.cpu().tolist()
    assert out[1] == -102
    for i in (0, 2):
        assert dst[i, :out[i]].cpu().numpy().tobytes() == D.stateless(ins[i])


def test_gzip_refuses_dicts_and_eof(enc):
    from compress_b200._lib import B2CError
    with pytest.raises(B2CError):
        enc.encode_chunks([b"abc"], format=2, header=HDR, dicts=[b"x"])
    with pytest.raises(B2CError):
        enc.encode_chunks([b"abc"], format=2, header=HDR, eof=[True])


def test_dst_one_byte_short(enc):
    rng = random.Random(4)
    ins = [D.text(rng, 50000), rng.randbytes(3000), b"", D.text(rng, 100)]
    for fmt in (0, 2):
        want = [_want(d, fmt) for d in ins]
        caps = [len(w) - 1 for w in want]
        outs, codes, _ = enc.encode_chunks(ins, format=fmt, header=HDR if fmt == 2 else b"", caps=caps)
        assert codes == [-4] * len(ins)
        # the device form: rows one byte shorter than each output, and a guard column that must stay untouched
        for i, d in enumerate(ins):
            cap = len(want[i]) - 1
            src = torch.frombuffer(bytearray(d + b"\0"), dtype=torch.uint8).cuda()
            dst = torch.full((1, cap + 64), 0xA5, dtype=torch.uint8, device="cuda")
            _, out = enc.encode_device(src, torch.tensor([len(d)], dtype=torch.int32).cuda(), max(len(d), 1), dst=dst,
                                       dst_cap=cap, format=fmt, header=HDR if fmt == 2 else b"")
            torch.cuda.synchronize()
            assert int(out[0]) == -4
            assert bool((dst[0, cap:] == 0xA5).all())


def test_two_streams(enc):
    rng = random.Random(6)
    a = [D.text(rng, 30000 + i) for i in range(40)]
    b = [rng.randbytes(20000 + i) for i in range(40)]
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    ga, _ = _device(enc, a, 0, stream=s1)
    gb, _ = _device(enc, b, 2, stream=s2)
    assert ga == [D.stateless(x) for x in a] and gb == [D.gzip_member(x) for x in b]


def test_round_trip_through_device_inflate(enc):
    from compress_b200 import flate
    rng = random.Random(8)
    ins = [d for _, d in D.pool()] + [D.text(rng, 200000)]
    raw = enc.encode_chunks(ins)[0]
    gz = enc.encode_chunks(ins, format=2, header=HDR)[0]
    dec = flate.Decoder()
    try:
        back, codes = dec.decode_chunks(raw, [len(d) + 16 for d in ins], flate.RAW)
        assert back == ins
        back, codes = dec.decode_chunks(gz, [len(d) + 16 for d in ins], flate.GZIP)
        assert back == ins
    finally:
        dec.close()
    assert [zlib.decompress(r, -15) for r in raw] == ins
    assert [pygzip.decompress(g) for g in gz] == ins


def test_writers_match_oracle():
    from compress_b200 import flate, gzip
    rng = random.Random(10)
    writes = [D.text(rng, 70000), b"", rng.randbytes(5000), D.text(rng, 13), bytes(40000)]
    buf = io.BytesIO()
    w = flate.NewStatelessWriter(buf)
    for p in writes:
        w.Write(p)
    w.Close()
    assert buf.getvalue() == b"".join(D.stateless(p, False) for p in writes) + D.stateless(b"", True)
    g = io.BytesIO()
    z = gzip.NewWriterLevel(g, gzip.StatelessCompression)
    z.Name, z.Comment, z.ModTime, z.OS, z.Extra = "a.txt", "note", 1700000000, 3, b"xy"
    for p in writes:
        z.Write(p)
    z.Close()
    data = b"".join(writes)
    hdr = gzip.header_bytes("a.txt", "note", b"xy", 1700000000, 3)
    body = b"".join(D.stateless(p, False) for p in writes) + D.stateless(b"", True)
    assert g.getvalue() == hdr + body + zlib.crc32(data).to_bytes(4, "little") + len(data).to_bytes(4, "little")
    assert pygzip.decompress(g.getvalue()) == data
    assert D.gzip_member(writes[0], hdr) == gzip.header_bytes("a.txt", "note", b"xy", 1700000000, 3) + D.stateless(
        writes[0], False) + D.stateless(b"", True) + zlib.crc32(writes[0]).to_bytes(4, "little") + len(writes[0]).to_bytes(4, "little")
    with pytest.raises(ValueError):
        gzip.NewWriterLevel(io.BytesIO(), 6)


def test_gzip_writer_defaults_and_reset():
    # an unset ModTime is Go's zero time: MTIME uint32(time.Time{}.Unix()) = 0x886e0900; Reset clears the header fields
    from compress_b200 import gzip
    g = io.BytesIO()
    z = gzip.NewWriterLevel(g, gzip.StatelessCompression)
    z.Name = "x"
    z.Write(b"hello")
    z.Close()
    assert g.getvalue()[:10] == b"\x1f\x8b\x08\x08\x00\x09\x6e\x88\x00\xff"
    g2 = io.BytesIO()
    z.Reset(g2)
    z.Write(b"hello")
    z.Close()
    assert g2.getvalue() == HDR[:4] + b"\x00\x09\x6e\x88\x00\xff" + D.stateless(b"hello", False) + D.stateless(b"", True) + \
        zlib.crc32(b"hello").to_bytes(4, "little") + (5).to_bytes(4, "little")
