"""DEFLATE at BestSpeed on the device: raw, zlib and gzip members byte-identical to the oracle's (and so to the
reference's) through both entry points, at several batch shapes, across the history move and scratch passes, at the input
cap and the destination's end, on two streams; read back by the device inflate; and the flate / zlib / gzip writers."""
import gzip as pygzip
import io
import random
import zlib

import numpy as np
import pytest
import torch

import flate_best_speed_util as D

pytestmark = pytest.mark.gpu

FMTS = (D.RAW, D.ZLIB, D.GZIP)
HDR = D.GZIP_HDR_BEST_SPEED


@pytest.fixture(scope="module")
def enc():
    from compress_b200 import flate
    e = flate.Encoder()
    yield e
    e.close()


def _hdr(fmt):
    return HDR if fmt == D.GZIP else b""


def _device(enc, inputs, fmt, offsets=False, stream=None):
    """best_speed_device over a packed batch with unaligned offsets, or a strided one; returns (outputs, codes, checks)."""
    n = len(inputs)
    stride = max(1, max(len(b) for b in inputs))
    if offsets:
        offs, buf = [], bytearray()
        for b in inputs:
            buf += bytes(1 + len(buf) % 3)               # unaligned starts
            offs.append(len(buf))
            buf += b
        src = torch.frombuffer(buf + bytearray(8), dtype=torch.uint8).cuda()
        so = torch.tensor(offs, dtype=torch.int64).cuda()
    else:
        a = np.zeros((n, stride), dtype=np.uint8)
        for i, b in enumerate(inputs):
            a[i, :len(b)] = np.frombuffer(b, dtype=np.uint8)
        src, so = torch.from_numpy(a).cuda().reshape(-1), None
    sizes = torch.tensor([len(b) for b in inputs], dtype=torch.int32).cuda()
    chk = torch.zeros(n, dtype=torch.int32, device="cuda")
    with torch.cuda.stream(stream or torch.cuda.current_stream()):
        dst, out = enc.best_speed_device(src, sizes, stride, format=fmt, header=_hdr(fmt), check_out=chk, src_offsets=so)
    torch.cuda.synchronize()
    out = out.cpu().numpy()
    d = dst.cpu().numpy()
    return ([d[i, :out[i]].tobytes() if out[i] >= 0 else None for i in range(n)], [int(x) for x in out],
            [int(x) & 0xffffffff for x in chk.cpu().tolist()])


def _frame(raw, data, fmt):
    if fmt == D.ZLIB:
        return b"\x78\x01" + raw + zlib.adler32(data).to_bytes(4, "big")
    if fmt == D.GZIP:
        return HDR + raw + zlib.crc32(data).to_bytes(4, "little") + len(data).to_bytes(4, "little")
    return raw


def _checks(inputs, fmt):
    return [zlib.adler32(b) if fmt == D.ZLIB else zlib.crc32(b) for b in inputs]


@pytest.mark.parametrize("fmt", FMTS)
def test_pool_both_entry_points(enc, fmt):
    pool = [d for _, d in D.pool()]
    want = [D.best_speed(d, fmt) for d in pool]
    outs, codes, chks = enc.best_speed_chunks(pool, format=fmt, header=_hdr(fmt))
    assert outs == want and chks == _checks(pool, fmt)
    for offsets in (False, True):
        got, _, chks = _device(enc, pool, fmt, offsets=offsets)
        assert got == want and chks == _checks(pool, fmt)


def test_fuzz_corpus(enc):
    items = D.fuzz_inputs()
    for fmt in FMTS:
        want = [D.best_speed(d, fmt) for d in items]
        assert enc.best_speed_chunks(items, format=fmt, header=_hdr(fmt))[0] == want
        assert _device(enc, items, fmt, offsets=True)[0] == want


@pytest.mark.parametrize("n", [1, 31, 32, 33, 4097])
def test_batch_shapes(enc, n):
    rng = random.Random(n)
    ins = [D.text(rng, rng.randint(0, 3 * D.WINDOW)) if i % 3 else rng.randbytes(rng.randint(0, 40000)) for i in range(n)]
    if n == 4097:
        ins = [b[:rng.randint(0, 3000)] for b in ins]
    for fmt in FMTS:
        want = [D.best_speed(d, fmt) for d in ins]
        assert _device(enc, ins, fmt, offsets=n != 32)[0] == want, (n, fmt)


def test_many_windows_and_scratch_passes(enc):
    # 16 384 x 64 KiB: about 385 KiB of scratch per input, so the batch runs in two 4 GiB passes
    rng = random.Random(5)
    unit = D.text(rng, 1 << 20)
    ins = [unit[(i * 7919) % (1 << 19):][:65536] for i in range(16384)]
    raw = [D.best_speed(d) for d in ins]
    for fmt in FMTS:                                 # the containers around the oracle's raw stream, as its framing writes them
        want = [_frame(r, d, fmt) for r, d in zip(raw, ins)]
        got, codes, chks = _device(enc, ins, fmt)
        assert got == want, fmt
        assert chks == _checks(ins, fmt)


def test_long_inputs_across_history_moves(enc):
    # 2 x 8 MiB: 129 windows each, the history moving down every four windows after the fifth
    rng = random.Random(9)
    big = [(D.text(rng, 1 << 20) + rng.randbytes(1 << 17)) * 8, bytes(x % 251 for x in range(8 << 20))]
    big = [b[:8 << 20] for b in big]
    for fmt in FMTS:
        want = [D.best_speed(b, fmt) for b in big]
        got, codes, _ = _device(enc, big, fmt)
        assert got == want, fmt
    # window counts on both sides of every move up to the twelfth window
    ins = [D.text(rng, k * D.WINDOW + d) for k in range(4, 13) for d in (-1, 1)]
    assert _device(enc, ins, D.RAW, offsets=True)[0] == [D.best_speed(b) for b in ins]


def test_dst_one_byte_short(enc):
    rng = random.Random(4)
    ins = [D.text(rng, 150000), rng.randbytes(3000), b"", D.text(rng, 100), D.text(rng, 20)]
    for fmt in FMTS:
        want = [D.best_speed(d, fmt) for d in ins]
        caps = [len(w) - 1 for w in want]
        outs, codes, _ = enc.best_speed_chunks(ins, format=fmt, header=_hdr(fmt), caps=caps)
        assert codes == [-4] * len(ins)
        for i, d in enumerate(ins):                  # the device form: a guard region after each row must stay untouched
            cap = len(want[i]) - 1
            src = torch.frombuffer(bytearray(d + b"\0"), dtype=torch.uint8).cuda()
            dst = torch.full((1, cap + 64), 0xA5, dtype=torch.uint8, device="cuda")
            _, out = enc.best_speed_device(src, torch.tensor([len(d)], dtype=torch.int32).cuda(), max(len(d), 1), dst=dst,
                                           dst_cap=cap, format=fmt, header=_hdr(fmt))
            torch.cuda.synchronize()
            assert int(out[0]) == -4
            assert bool((dst[0, cap:] == 0xA5).all())


def test_input_over_the_cap(enc):
    # an input one byte over 1 GiB, in real device memory, is B2C_ERR_ARG; its neighbours are encoded as usual
    rng = random.Random(12)
    a, c = D.text(rng, 70000), D.text(rng, 5000)
    big = (1 << 30) + 1
    src = torch.zeros(big + 2 * 70000, dtype=torch.uint8, device="cuda")
    src[:len(a)] = torch.frombuffer(bytearray(a), dtype=torch.uint8).cuda()
    src[big + 70000:big + 70000 + len(c)] = torch.frombuffer(bytearray(c), dtype=torch.uint8).cuda()
    offs = torch.tensor([0, 70000, big + 70000], dtype=torch.int64).cuda()
    sizes = torch.tensor([len(a), big, len(c)], dtype=torch.int32).cuda()
    for fmt in FMTS:
        dst, out = enc.best_speed_device(src, sizes, big, dst_cap=D.bound(70000) + 64, format=fmt,
                                         header=_hdr(fmt), src_offsets=offs)
        torch.cuda.synchronize()
        out = out.cpu().tolist()
        assert out[1] == -102
        assert dst[0, :out[0]].cpu().numpy().tobytes() == D.best_speed(a, fmt)
        assert dst[2, :out[2]].cpu().numpy().tobytes() == D.best_speed(c, fmt)
    del src
    # an input larger than src_stride is refused the same way
    ins = [D.text(rng, 30000), D.text(rng, 40000), D.text(rng, 30000)]
    buf = np.zeros(3 * 30000 + 10000, dtype=np.uint8)
    for k, b in enumerate(ins):
        buf[k * 30000:k * 30000 + len(b)] = np.frombuffer(b, dtype=np.uint8)
    dst, out = enc.best_speed_device(torch.from_numpy(buf).cuda(), torch.tensor([len(b) for b in ins], dtype=torch.int32).cuda(),
                                     30000, src_offsets=torch.tensor([0, 30000, 60000], dtype=torch.int64).cuda())
    torch.cuda.synchronize()
    out = out.cpu().tolist()
    assert out[1] == -102
    for k in (0, 2):
        assert dst[k, :out[k]].cpu().numpy().tobytes() == D.best_speed(ins[k])


def test_two_streams(enc):
    rng = random.Random(6)
    a = [D.text(rng, 70000 + i) for i in range(40)]
    b = [rng.randbytes(20000 + i) for i in range(40)]
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    ga = _device(enc, a, D.ZLIB, stream=s1)[0]
    gb = _device(enc, b, D.GZIP, stream=s2)[0]
    assert ga == [D.best_speed(x, D.ZLIB) for x in a] and gb == [D.best_speed(x, D.GZIP) for x in b]


def test_round_trip_through_device_inflate(enc):
    from compress_b200 import flate
    rng = random.Random(8)
    ins = [d for _, d in D.pool()] + [D.text(rng, 400000)]
    dec = flate.Decoder()
    try:
        for fmt in FMTS:
            outs = enc.best_speed_chunks(ins, format=fmt, header=_hdr(fmt))[0]
            back, codes = dec.decode_chunks(outs, [len(d) + 16 for d in ins], fmt)
            assert back == ins, fmt
    finally:
        dec.close()


def test_writers_match_oracle():
    from compress_b200 import flate, gzip, zlib as bzlib
    rng = random.Random(10)
    writes = [D.text(rng, 70000), b"", rng.randbytes(5000), D.text(rng, 13), bytes(140000)]
    data = b"".join(writes)
    sizes = [len(p) for p in writes]
    for mod_writer, fmt in ((lambda o: flate.NewWriter(o, flate.BestSpeed), D.RAW),
                            (lambda o: bzlib.NewWriterLevel(o, bzlib.BestSpeed), D.ZLIB)):
        buf = io.BytesIO()
        w = mod_writer(buf)
        for p in writes:
            assert w.Write(p) == len(p)
        w.Close()
        assert buf.getvalue() == D.best_speed(data, fmt, writes=sizes)
        with pytest.raises(NotImplementedError):
            w.Flush()
        buf2 = io.BytesIO()                          # Reset starts a new member
        w.Reset(buf2)
        w.Write(b"hello")
        w.Close()
        assert buf2.getvalue() == D.best_speed(b"hello", fmt)
    g = io.BytesIO()
    z = gzip.NewWriterLevel(g, gzip.BestSpeed)
    z.Name, z.Comment, z.ModTime, z.OS, z.Extra = "a.txt", "note", 1700000000, 3, b"xy"
    for p in writes:
        z.Write(p)
    with pytest.raises(NotImplementedError):
        z.Flush()
    z.Close()
    hdr = gzip.header_bytes("a.txt", "note", b"xy", 1700000000, 3, level=gzip.BestSpeed)
    assert hdr[8] == 4
    assert g.getvalue() == D.best_speed(data, D.GZIP, hdr, writes=sizes)
    assert pygzip.decompress(g.getvalue()) == data
    g2 = io.BytesIO()
    z.Reset(g2)
    z.Write(b"hello")
    z.Close()
    assert g2.getvalue() == D.best_speed(b"hello", D.GZIP, HDR)
    # the levels not built keep raising
    for bad in (0, 2, 6, 9, -1, -2):
        with pytest.raises(ValueError):
            flate.NewWriter(io.BytesIO(), bad)
        with pytest.raises(ValueError):
            bzlib.NewWriterLevel(io.BytesIO(), bad)
    with pytest.raises(ValueError):
        bzlib.NewWriter(io.BytesIO())
    with pytest.raises(ValueError):
        gzip.NewWriterLevel(io.BytesIO(), 6)
