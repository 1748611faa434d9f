"""Inflate on the device against the oracle (oracle/orc_flate.c) through both entry points: the seeded pool, invalid and
mutated streams, batch shapes and alignments, format extremes, two streams on one context, and the readers against
Python's gzip / zlib."""
import gzip as pygzip
import random
import zlib as pyzlib

import numpy as np
import pytest
import torch

import flate_util as F

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dec():
    from compress_b200 import flate
    d = flate.Decoder()
    yield d
    d.close()


def _device(dec, fmt, streams, caps, multistream=True, shift=(0, 0)):
    """The device call with packed, deliberately unaligned source and destination offsets."""
    so, do, s_off, d_off = shift[0], shift[1], [], []
    for s, c in zip(streams, caps):
        s_off.append(so); so += len(s) + 3
        d_off.append(do); do += c + 5
    src = np.zeros(so + 16, dtype=np.uint8)
    for s, o in zip(streams, s_off):
        src[o:o + len(s)] = np.frombuffer(s, dtype=np.uint8)
    d_src = torch.from_numpy(src).cuda()
    dst = torch.zeros(do + 16, dtype=torch.uint8, device="cuda")
    sizes = torch.tensor([len(s) for s in streams], dtype=torch.int32).cuda()
    so_t = torch.tensor(s_off, dtype=torch.int64).cuda()
    do_t = torch.tensor(d_off, dtype=torch.int64).cuda()
    out = torch.empty(len(streams), dtype=torch.int64, device="cuda")
    from compress_b200._lib import lib, check
    import ctypes
    stride = max([len(s) for s in streams] + [1])
    cap = max(caps + [0])
    assert all(c == cap for c in caps)
    check(lib.b2c_flate_decode_device(dec._ctx, fmt, 0 if multistream else 1, d_src.data_ptr(), stride, so_t.data_ptr(),
                                      sizes.data_ptr(), dst.data_ptr(), 0, do_t.data_ptr(), cap, out.data_ptr(),
                                      len(streams), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), dec._ctx)
    torch.cuda.synchronize()
    codes = out.cpu().tolist()
    host = dst.cpu().numpy()
    return [host[o:o + r].tobytes() if r >= 0 else None for o, r in zip(d_off, codes)], codes


def _check(dec, fmt, streams, cap, multistream=True, shift=(1, 3)):
    want = [F.orc_decode(fmt, s, cap, multistream) for s in streams]
    outs, codes = dec.decode_chunks(streams, [cap] * len(streams), fmt, multistream)
    for i, (r, w) in enumerate(want):
        assert codes[i] == r, (i, fmt, codes[i], r)
        if r >= 0:
            assert outs[i] == w, i
    outs, codes = _device(dec, fmt, streams, [cap] * len(streams), multistream, shift)
    for i, (r, w) in enumerate(want):
        assert codes[i] == r, (i, fmt, codes[i], r, "device")
        if r >= 0:
            assert outs[i] == w, (i, "device")


def test_pool(dec):
    for fmt in (F.RAW, F.ZLIB, F.GZIP):
        for multi in (True, False):
            items = [(s, d) for f, s, d, m in F.pool() if f == fmt and m == multi]
            if items:
                _check(dec, fmt, [s for s, _ in items], 110000, multi)


def test_invalid_streams(dec):
    for case in F.invalid_streams():
        fmt, s = case[0], case[1]
        multi = case[3] if len(case) > 3 else True
        _check(dec, fmt, [s], 1 << 16, multi)


def test_fixtures_and_stale_tables(dec):
    for fmt in (F.RAW, F.ZLIB, F.GZIP):
        streams = [s for _, f, s, _ in F.fixture_streams() if f == fmt] + [s for f, s, _ in F.stale_streams() if f == fmt]
        _check(dec, fmt, streams, 1 << 17)


@pytest.mark.parametrize("n", [1, 31, 32, 33, 4097])
def test_batch_shapes(dec, n):
    rng = random.Random(n)
    streams = []
    for i in range(n):
        data = F.text(rng, rng.choice([0, 10, 300, 5000, 20000]))
        streams.append(F.deflate(data, F.GZIP, rng.randint(0, 9)))
    _check(dec, F.GZIP, streams, 20000, shift=(n % 3, n % 5 + 1))


def test_format_extremes(dec):
    rng = random.Random(5)
    big = bytes(rng.getrandbits(8) for _ in range(3 * 65535 + 17))      # level 0: stored blocks of 65 535 bytes
    far = bytes(rng.getrandbits(8) for _ in range(32768)) * 3 + b"z" * 258   # distance 32 768, length 258
    members = b"".join(F.gzip_member(F.text(rng, rng.randint(0, 40)), 6) for _ in range(1200))
    cases = [(F.GZIP, F.deflate(big, F.GZIP, 0)), (F.ZLIB, F.deflate(far, F.ZLIB, 9)), (F.RAW, F.deflate(far, F.RAW, 1)),
             (F.GZIP, members)]
    for fmt, s in cases:
        r = F.orc_decode(fmt, s, 1 << 20)[0]
        assert r > 0
        _check(dec, fmt, [s], 1 << 20)
        _check(dec, fmt, [s], r - 1)                                        # one byte too small
        assert dec.decode_chunks([s], [r - 1], fmt)[1][0] == -4


def test_mutations(dec):
    rng = random.Random(17)
    base = {fmt: [F.deflate(F.text(rng, n), fmt, lv) for n, lv in ((3000, 1), (9000, 6), (700, 9), (2000, 0))] +
            [F.deflate(bytes(rng.getrandbits(8) for _ in range(1500)), fmt, 6)] for fmt in (F.RAW, F.ZLIB, F.GZIP)}
    for fmt in (F.RAW, F.ZLIB, F.GZIP):
        muts = [F.mutate(rng, rng.choice(base[fmt])) for _ in range(300)]
        _check(dec, fmt, muts, 12000)


def test_two_streams_one_context(dec):
    rng = random.Random(23)
    a = [F.deflate(F.text(rng, 20000), F.GZIP, 6) for _ in range(64)]
    b = [F.deflate(F.text(rng, 9000), F.GZIP, 1) for _ in range(64)]
    want_a = [F.orc_decode(F.GZIP, s, 20000) for s in a]
    want_b = [F.orc_decode(F.GZIP, s, 20000) for s in b]

    def prep(streams):
        stride = 32768
        src = torch.zeros(len(streams) * stride, dtype=torch.uint8)
        for i, s in enumerate(streams):
            src[i * stride:i * stride + len(s)] = torch.frombuffer(bytearray(s), dtype=torch.uint8)
        return src.cuda(), torch.tensor([len(s) for s in streams], dtype=torch.int32).cuda(), stride

    sa, za, st = prep(a)
    sb, zb, _ = prep(b)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    with torch.cuda.stream(s1):
        da, oa = dec.decode_device(sa, za, st, dst_cap=20000)
    with torch.cuda.stream(s2):
        db, ob = dec.decode_device(sb, zb, st, dst_cap=20000)
    torch.cuda.synchronize()
    for d, o, w in ((da, oa, want_a), (db, ob, want_b)):
        o = o.cpu().tolist()
        for i, (r, content) in enumerate(w):
            assert o[i] == r and bytes(d[i, :r].cpu().numpy()) == content


def test_readers():
    from compress_b200 import flate, gzip, zlib
    rng = random.Random(29)
    data = F.text(rng, 200000)
    g = pygzip.compress(data[:100000], 6) + pygzip.compress(data[100000:], 1)
    r = gzip.NewReader(g)
    assert r.read() == pygzip.decompress(g) == data
    r = gzip.NewReader(g)
    r.Multistream(False)
    assert r.read() == data[:100000]
    m = F.gzip_member(b"x" * 10, name=b"name.txt", comment=b"hi", extra=b"EX", fhcrc=True, mtime=1234, os_byte=7)
    h = gzip.NewReader(m).Header
    assert (h.Name, h.Comment, h.Extra, h.ModTime, h.OS) == ("name.txt", "hi", b"EX", 1234, 7)
    assert zlib.NewReader(pyzlib.compress(data, 9)).read() == data
    assert flate.NewReader(F.deflate(data, F.RAW, 3)).read() == data
    with pytest.raises(gzip.ErrChecksum):
        gzip.NewReader(g[:-5] + bytes([g[-5] ^ 1]) + g[-4:]).read()
    with pytest.raises(zlib.ErrHeader):
        zlib.NewReader(b"\x78\x9d" + pyzlib.compress(data)[2:])
    with pytest.raises(flate.ErrUnexpectedEOF):
        zlib.NewReader(pyzlib.compress(data)[:-9])
    with pytest.raises(flate.CorruptInputError):
        flate.NewReader(b"\x07")
