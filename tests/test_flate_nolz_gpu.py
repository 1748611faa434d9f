"""DEFLATE at HuffmanOnly and NoCompression on the device: raw, zlib and gzip members byte-identical to the oracle's (and
so to the reference's) through both entry points, at several batch shapes, for one 1 GiB member alone and among 4 096
small ones (record passes), at the destination's end, past src_stride and on two streams; read back by the device
inflate and Python's zlib / gzip; and the gzip writer at both levels."""
import ctypes
import gzip as pygzip
import io
import random
import zlib

import numpy as np
import pytest
import torch

import flate_nolz_util as D

pytestmark = pytest.mark.gpu

FMTS = D.FORMATS
LEVELS = D.LEVELS


@pytest.fixture(scope="module")
def enc():
    from compress_b200 import flate
    e = flate.Encoder()
    yield e
    e.close()


def _hdr(fmt):
    return D.GZIP_HDR if fmt == D.GZIP else b""


def _frame(raw, data, fmt):
    """The zlib / gzip framing the writers put around the oracle's raw stream."""
    if fmt == D.ZLIB:
        return b"\x78\x01" + raw + zlib.adler32(data).to_bytes(4, "big")
    if fmt == D.GZIP:
        return D.GZIP_HDR + raw + zlib.crc32(data).to_bytes(4, "little") + len(data).to_bytes(4, "little")
    return raw


def _checks(inputs, fmt):
    return [zlib.adler32(b) if fmt == D.ZLIB else zlib.crc32(b) for b in inputs]


def _device(enc, level, inputs, fmt, offsets=False, stream=None):
    """nolz_device over a packed batch with unaligned offsets, or a strided one; returns (outputs, codes, checks)."""
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
        dst, out = enc.nolz_device(level, src, sizes, stride, format=fmt, header=_hdr(fmt), check_out=chk, src_offsets=so)
    torch.cuda.synchronize()
    out = out.cpu().numpy()
    d = dst.cpu().numpy()
    return ([d[i, :out[i]].tobytes() if out[i] >= 0 else None for i in range(n)], [int(x) for x in out],
            [int(x) & 0xffffffff for x in chk.cpu().tolist()])


@pytest.mark.parametrize("level", LEVELS)
@pytest.mark.parametrize("fmt", FMTS)
def test_pool_both_entry_points(enc, level, fmt):
    pool = [d for _, d in D.pool()]
    want = [D.nolz(d, level, fmt) for d in pool]
    outs, codes, chks = enc.nolz_chunks(level, pool, format=fmt, header=_hdr(fmt))
    assert outs == want and chks == _checks(pool, fmt)
    for offsets in (False, True):
        got, _, chks = _device(enc, level, pool, fmt, offsets=offsets)
        assert got == want and chks == _checks(pool, fmt)


@pytest.mark.parametrize("level", LEVELS)
def test_fuzz_corpus(enc, level):
    items = D.fuzz_inputs()
    for fmt in FMTS:
        want = [D.nolz(d, level, fmt) for d in items]
        assert enc.nolz_chunks(level, items, format=fmt, header=_hdr(fmt))[0] == want
        assert _device(enc, level, items, fmt, offsets=True)[0] == want


@pytest.mark.parametrize("n", [1, 31, 32, 33, 4097])
def test_batch_shapes(enc, n):
    rng = random.Random(n)
    ins = [D.text(rng, rng.randint(0, 5 * 32768)) if i % 3 else D.skewed(rng, rng.randint(0, 70000)) for i in range(n)]
    if n == 4097:
        ins = [b[:rng.randint(0, 3000)] for b in ins]
    for level in LEVELS:
        raw = [D.nolz(d, level) for d in ins]
        for fmt in FMTS:
            want = [_frame(r, d, fmt) for r, d in zip(raw, ins)]
            assert _device(enc, level, ins, fmt, offsets=n != 32)[0] == want, (n, level, fmt)
            assert enc.nolz_chunks(level, ins, format=fmt, header=_hdr(fmt))[0] == want, (n, level, fmt)


def test_many_inputs(enc):
    # 16 384 x 64 KiB of text
    rng = random.Random(5)
    unit = D.text(rng, 1 << 20)
    ins = [unit[(i * 7919) % (1 << 19):][:65536] for i in range(16384)]
    for level in LEVELS:
        raw = [D.nolz(d, level) for d in ins]
        for fmt in FMTS:
            want = [_frame(r, d, fmt) for r, d in zip(raw, ins)]
            got, codes, chks = _device(enc, level, ins, fmt)
            assert got == want, (level, fmt)
            assert chks == _checks(ins, fmt)
        assert enc.nolz_chunks(level, ins[:4096])[0] == raw[:4096]


def _big(rng):
    """1 GiB: text with skewed, random and repeated stretches, so every outcome of the walk occurs along it."""
    units = [D.text(rng, 1 << 22), D.skewed(rng, 1 << 22), rng.randbytes(1 << 22), b"ab" * (1 << 21)]
    parts, n = [], 0
    while n < 1 << 30:
        u = units[rng.randrange(4)]
        o = rng.randrange(1 << 21)
        parts.append(u[o:o + rng.randint(1 << 16, 1 << 21)])
        n += len(parts[-1])
    return b"".join(parts)[:1 << 30]


def _dst_offsets(caps):
    offs, pos = [], 0
    for c in caps:
        offs.append(pos)
        pos += c
    return offs, pos


def test_one_gib_alone_and_among_small_ones(enc):
    rng = random.Random(21)
    big = _big(rng)
    small = [D.text(rng, rng.randint(0, 3000)) for _ in range(4096)]
    for level in LEVELS:
        raw_big = D.nolz(big, level)
        raw_small = [D.nolz(d, level) for d in small]
        for fmt in FMTS:
            # alone: one member is the whole device's work
            src = torch.frombuffer(bytearray(big), dtype=torch.uint8).cuda()
            sizes = torch.tensor([len(big)], dtype=torch.int32).cuda()
            chk = torch.zeros(1, dtype=torch.int32, device="cuda")
            dst, out = enc.nolz_device(level, src, sizes, len(big), format=fmt, header=_hdr(fmt), check_out=chk)
            torch.cuda.synchronize()
            want = _frame(raw_big, big, fmt)
            assert int(out[0]) == len(want) and dst[0, :len(want)].cpu().numpy().tobytes() == want, (level, fmt)
            assert int(chk[0]) & 0xffffffff == _checks([big], fmt)[0]
            del dst, src
            # among 4 096 small ones, in one call with src_stride 1 GiB: the records of a pass hold only some inputs
            ins = small[:2048] + [big] + small[2048:]
            offs, pos = [], 0
            for b in ins:
                offs.append(pos)
                pos += len(b) + 1
            buf = torch.empty(pos, dtype=torch.uint8, device="cuda")
            for o, b in zip(offs, ins):
                if b:
                    buf[o:o + len(b)] = torch.frombuffer(bytearray(b), dtype=torch.uint8).cuda()
            caps = [D.bound(level, len(b)) + D.container(fmt) for b in ins]
            doffs, dpos = _dst_offsets(caps)
            dst = torch.full((dpos,), 0xA5, dtype=torch.uint8, device="cuda")
            out = torch.empty(len(ins), dtype=torch.int64, device="cuda")
            so = torch.tensor(offs, dtype=torch.int64).cuda()
            sz = torch.tensor([len(b) for b in ins], dtype=torch.int32).cuda()
            do = torch.tensor(doffs, dtype=torch.int64).cuda()
            from compress_b200 import _lib
            stream = torch.cuda.current_stream().cuda_stream
            _lib.check(_lib.lib.b2c_flate_nolz_device(
                enc._ctx, level, fmt, 0, buf.data_ptr(), 1 << 30, so.data_ptr(), sz.data_ptr(), _hdr(fmt), len(_hdr(fmt)),
                dst.data_ptr(), 0, do.data_ptr(), max(caps), out.data_ptr(), None, len(ins), ctypes.c_void_p(stream)),
                enc._ctx)
            torch.cuda.synchronize()
            out = out.cpu().tolist()
            d = dst.cpu().numpy()
            wants = [_frame(r, b, fmt) for r, b in zip(raw_small[:2048] + [raw_big] + raw_small[2048:], ins)]
            for k, (o, w) in enumerate(zip(doffs, wants)):
                assert out[k] == len(w) and d[o:o + len(w)].tobytes() == w, (level, fmt, k)
            del buf, dst
        assert enc.nolz_chunks(level, [big])[0] == [raw_big]


@pytest.mark.parametrize("level", LEVELS)
def test_dst_one_byte_short(enc, level):
    rng = random.Random(4)
    ins = [D.text(rng, 150000), rng.randbytes(3000), b"", D.text(rng, 100), D.skewed(rng, 33000)]
    for fmt in FMTS:
        want = [D.nolz(d, level, fmt) for d in ins]
        caps = [len(w) - 1 for w in want]
        outs, codes, _ = enc.nolz_chunks(level, ins, format=fmt, header=_hdr(fmt), caps=caps)
        assert codes == [-4] * len(ins)
        for i, d in enumerate(ins):                  # the device form: the row and a guard after it stay untouched
            cap = len(want[i]) - 1
            src = torch.frombuffer(bytearray(d + b"\0"), dtype=torch.uint8).cuda()
            dst = torch.full((1, cap + 64), 0xA5, dtype=torch.uint8, device="cuda")
            _, out = enc.nolz_device(level, src, torch.tensor([len(d)], dtype=torch.int32).cuda(), max(len(d), 1), dst=dst,
                                     dst_cap=cap, format=fmt, header=_hdr(fmt))
            torch.cuda.synchronize()
            assert int(out[0]) == -4
            assert bool((dst[0] == 0xA5).all())


@pytest.mark.parametrize("level", LEVELS)
def test_input_over_src_stride(enc, level):
    rng = random.Random(12)
    ins = [D.text(rng, 30000), D.text(rng, 40000), D.text(rng, 30000)]
    buf = np.zeros(3 * 30000 + 10000, dtype=np.uint8)
    for k, b in enumerate(ins):
        buf[k * 30000:k * 30000 + len(b)] = np.frombuffer(b, dtype=np.uint8)
    for fmt in FMTS:
        dst, out = enc.nolz_device(level, torch.from_numpy(buf).cuda(),
                                   torch.tensor([len(b) for b in ins], dtype=torch.int32).cuda(), 30000, format=fmt,
                                   header=_hdr(fmt), src_offsets=torch.tensor([0, 30000, 60000], dtype=torch.int64).cuda())
        torch.cuda.synchronize()
        out = out.cpu().tolist()
        assert out[1] == -102
        for k in (0, 2):
            assert dst[k, :out[k]].cpu().numpy().tobytes() == D.nolz(ins[k], level, fmt)


def test_bad_level_is_refused(enc):
    from compress_b200 import _lib
    with pytest.raises(_lib.B2CError):
        enc.nolz_chunks(1, [b"abc"])
    assert _lib.lib.b2c_flate_nolz_bound(1, 100) == 0


def test_two_streams(enc):
    rng = random.Random(6)
    a = [D.text(rng, 70000 + i) for i in range(40)]
    b = [D.skewed(rng, 40000 + i) for i in range(40)]
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    ga = _device(enc, -2, a, D.ZLIB, stream=s1)[0]
    gb = _device(enc, 0, b, D.GZIP, stream=s2)[0]
    assert ga == [D.nolz(x, -2, D.ZLIB) for x in a] and gb == [D.nolz(x, 0, D.GZIP) for x in b]


def test_round_trip_through_device_inflate(enc):
    from compress_b200 import flate
    rng = random.Random(8)
    ins = [d for _, d in D.pool()] + [D.text(rng, 400000)]
    dec = flate.Decoder()
    try:
        for level in LEVELS:
            for fmt in FMTS:
                outs = enc.nolz_chunks(level, ins, format=fmt, header=_hdr(fmt))[0]
                back, codes = dec.decode_chunks(outs, [len(d) + 16 for d in ins], fmt)[:2]
                assert back == ins, (level, fmt)
                if fmt == D.GZIP:
                    assert [pygzip.decompress(o) for o in outs] == ins
                else:
                    assert [zlib.decompress(o, 15 if fmt == D.ZLIB else -15) for o in outs] == ins
    finally:
        dec.close()


@pytest.mark.parametrize("level", LEVELS)
def test_gzip_writer(level):
    from compress_b200 import gzip
    rng = random.Random(3)
    data = D.text(rng, 3 * 32768 + 100) + D.skewed(rng, 50000)
    sizes = [1, 0, 40000, 70000, len(data) - 110001]
    g = io.BytesIO()
    z = gzip.NewWriterLevel(g, level)
    z.Name, z.Comment, z.ModTime, z.OS, z.Extra = "a.txt", "note", 1700000000, 3, b"xy"
    pos = 0
    for s in sizes:
        z.Write(data[pos:pos + s])
        pos += s
    with pytest.raises(NotImplementedError):
        z.Flush()
    z.Close()
    hdr = gzip.header_bytes("a.txt", "note", b"xy", 1700000000, 3, level=level)
    assert hdr[8] == 0
    assert g.getvalue() == D.nolz(data, level, D.GZIP, hdr, writes=sizes)
    assert pygzip.decompress(g.getvalue()) == data
    g2 = io.BytesIO()
    z.Reset(g2)
    z.Write(b"hello")
    z.Write(b" world")
    z.Close()
    assert g2.getvalue() == D.nolz(b"hello world", level, D.GZIP, writes=[5, 6])
