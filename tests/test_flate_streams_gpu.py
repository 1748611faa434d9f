"""Inflate on the device against the oracle (oracle/orc_flate.c), through both entry points, on the hand-built streams of
inflate_streams.py: code shapes, exec layouts, checksum sizes (up to 16 MiB), record-bound streams and header edges; every
truncation of a few streams; destinations of exactly the content and one byte less, with a guard after each row; and
batches whose record scratch takes several passes, with errors and multi-member inputs on both sides of each pass
boundary."""
import ctypes
import random
import struct
import zlib

import numpy as np
import pytest
import torch

import flate_util as F
import inflate_streams as S

pytestmark = pytest.mark.gpu

BIG_CAP = 1 << 21
REC_BYTES = 16                                  # sizeof(InfRec)
PASS_BYTES = 4 << 30                            # the record scratch of one pass


@pytest.fixture(scope="module")
def dec():
    from compress_b200 import flate
    d = flate.Decoder()
    yield d
    d.close()


def _device(dec, fmt, streams, caps, multistream=True, shift=(0, 0), guard=None):
    """The device call with packed, deliberately unaligned source and destination offsets.  guard: a byte value the
    destination is filled with first; the 5 bytes after each row must still hold it."""
    so, do, s_off, d_off = shift[0], shift[1], [], []
    for s, c in zip(streams, caps):
        s_off.append(so); so += len(s) + 3
        d_off.append(do); do += c + 5
    src = np.zeros(so + 16, dtype=np.uint8)
    for s, o in zip(streams, s_off):
        src[o:o + len(s)] = np.frombuffer(s, dtype=np.uint8)
    d_src = torch.from_numpy(src).cuda()
    dst = torch.full((do + 16,), 0 if guard is None else guard, dtype=torch.uint8, device="cuda")
    sizes = torch.tensor([len(s) for s in streams], dtype=torch.int32).cuda()
    so_t = torch.tensor(s_off, dtype=torch.int64).cuda()
    do_t = torch.tensor(d_off, dtype=torch.int64).cuda()
    out = torch.empty(len(streams), dtype=torch.int64, device="cuda")
    from compress_b200._lib import lib, check
    stride = max([len(s) for s in streams] + [1])
    cap = max(caps + [0])
    assert all(c == cap for c in caps)
    check(lib.b2c_flate_decode_device(dec._ctx, fmt, 0 if multistream else 1, d_src.data_ptr(), stride, so_t.data_ptr(),
                                      sizes.data_ptr(), dst.data_ptr(), 0, do_t.data_ptr(), cap, out.data_ptr(),
                                      len(streams), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), dec._ctx)
    torch.cuda.synchronize()
    codes = out.cpu().tolist()
    host = dst.cpu().numpy()
    if guard is not None:
        for o in d_off:
            assert (host[o + cap:o + cap + 5] == guard).all(), "a write past the row's end"
    return [host[o:o + r].tobytes() if r >= 0 else None for o, r in zip(d_off, codes)], codes


def _caps(streams):
    return [s.cap if s.cap is not None else max(F.orc_decode(s.fmt, s.data, BIG_CAP)[0], 0) + 64 for s in streams]


def _expect(got, fmt, data, cap, what):
    outs, codes = got
    for i, s in enumerate(data):
        r, want = F.orc_decode(fmt, s, cap[i] if isinstance(cap, list) else cap)
        assert codes[i] == r, (what[i], codes[i], r)
        if r >= 0:
            assert outs[i] == want, what[i]


def _check(dec, streams, alone=False, shift=(1, 3)):
    """streams through decode_chunks (each at its own cap) and the device entry point (a batch per format at the largest
    cap; streams over 1 MiB of content, or all of them with alone, in a call of their own at their own cap)."""
    for fmt in (S.RAW, S.ZLIB, S.GZIP):
        part = [s for s in streams if s.fmt == fmt]
        if not part:
            continue
        caps = _caps(part)
        data, names = [s.data for s in part], [s.name for s in part]
        _expect(dec.decode_chunks(data, caps, fmt), fmt, data, caps, names)
        small = [i for i, c in enumerate(caps) if c <= (1 << 20) and not alone]
        if small:
            cap = max(caps[i] for i in small)
            sd = [data[i] for i in small]
            _expect(_device(dec, fmt, sd, [cap] * len(sd), shift=shift), fmt, sd, cap, [names[i] for i in small])
        for i in range(len(part)):
            if i not in small:
                _expect(_device(dec, fmt, [data[i]], [caps[i]], shift=shift), fmt, [data[i]], caps[i], [names[i]])


def test_code_shapes(dec):
    _check(dec, S.code_shapes())


def test_exec_layouts(dec):
    _check(dec, S.exec_layouts(), shift=(2, 7))
    _check(dec, S.exec_layouts(), shift=(3, 0))


def test_checksum_sizes(dec):
    _check(dec, S.checksum_sizes(big=True))


def test_record_bound(dec):
    streams = S.record_bound(big=True)
    for s in streams:
        records, want = S.record_term(s)
        assert records >= want, s.name
    _check(dec, streams, alone=True)


def test_header_edges(dec):
    _check(dec, S.header_edges())


def test_truncations(dec):
    by_fmt = {}
    for fmt, s in S.truncation_set():
        by_fmt.setdefault(fmt, []).extend(s[:i] for i in range(len(s) + 1))
    for fmt, cuts in by_fmt.items():
        names = ["cut %d" % i for i in range(len(cuts))]
        _expect(dec.decode_chunks(cuts, [8192] * len(cuts), fmt), fmt, cuts, 8192, names)
        _expect(_device(dec, fmt, cuts, [8192] * len(cuts), shift=(1, 1)), fmt, cuts, 8192, names)


def _last_item_streams(n):
    """Raw streams of exactly n content bytes whose last output item is a literal, a match and a stored run."""
    rng = random.Random(n)
    head = F.text(rng, n - 40)
    lit = S.Writer().fixed(list(head) + list(b"x" * 39) + [0x79, S.EOB], final=True)
    mat = S.Writer().fixed(list(head) + list(b"ab") + [S.match(38, 2), S.EOB], final=True)
    sto = S.Writer().fixed(list(head) + [S.EOB], final=False).stored(rng.randbytes(40), final=True)
    for w in (lit, mat, sto):
        assert w.d == n
    return [lit.data(), mat.data(), sto.data()]


@pytest.mark.parametrize("n", [41, 64, 1000, 4099])
def test_exact_caps(dec, n):
    raw = _last_item_streams(n)
    for fmt in (S.RAW, S.GZIP):
        streams = raw if fmt == S.RAW else [S.gzip_wrap(r, F.orc_decode(S.RAW, r, n)[1]) for r in raw]
        names = ["last item: literal", "last item: match", "last item: stored run"]
        for cap in (n, n - 1):
            want = [F.orc_decode(fmt, s, cap)[0] for s in streams]
            assert want == ([n] * 3 if cap == n else [-4] * 3)
            _expect(dec.decode_chunks(streams, [cap] * 3, fmt), fmt, streams, cap, names)
            for shift in ((0, 0), (1, 3), (2, 13)):
                _expect(_device(dec, fmt, streams, [cap] * 3, shift=shift, guard=0xA5), fmt, streams, cap, names)


def _rec_cap(slen, cap):
    """inf_rec_cap (b2c_inflate.cuh)."""
    return min(cap // 3, 4 * slen) + slen // 5 + slen // 18 + 2


def _passes(per_item):
    """next_pass (b2c_api.cu) over items of the given record counts: the list of [c0, c1) passes."""
    out, c0, n = [], 0, len(per_item)
    base = np.concatenate([[0], np.cumsum(per_item)])
    while c0 < n:
        e = c0 + 1
        while e < n and (base[e + 1] - base[c0]) * REC_BYTES <= PASS_BYTES:
            e += 1
        out.append((c0, e))
        c0 = e
    return out


def _kinds(rng):
    """The inputs placed around pass boundaries: a walk error, a CRC failure, a content over the cap (-4), an empty gzip
    input (-12) and three gzip members."""
    walk = S.gzip_wrap(S.Writer().fixed([0x41, S.match(3, 9), S.EOB], final=True).data(), b"")
    good = F.gzip_member(b"crc " * 5)
    crc = good[:-8] + struct.pack("<I", zlib.crc32(b"crc " * 5) ^ 4) + good[-4:]
    over = F.gzip_member(b"o" * 300000, 9)
    multi = b"".join(F.gzip_member(F.text(rng, k), 6) for k in (5, 17, 3))
    return [walk, crc, over, b"", multi]


def test_scratch_passes_device(dec):
    # src_stride 65 536 into dst_cap 262 144: 104 130 records of 16 bytes per input, 2 577 inputs per 4 GiB pass
    stride, cap, n = 65536, 262144, 6000
    per = _rec_cap(stride, cap)
    assert per == 104130 and PASS_BYTES // (per * REC_BYTES) == 2577
    assert _passes([per] * n) == [(0, 2577), (2577, 5154), (5154, 6000)]
    rng = random.Random(41)
    plain = [F.gzip_member(b"%d:" % c + F.text(rng, rng.randrange(0, 30)), rng.choice((0, 1, 6))) for c in range(n)]
    kinds = _kinds(rng)
    where = [2576, 2577, 2578, 5153, 5154, 5155]
    dst = torch.empty((n, cap), dtype=torch.uint8, device="cuda")
    for rot in range(len(kinds)):
        streams = list(plain)
        for p, c in enumerate(where):
            streams[c] = kinds[(rot + p) % len(kinds)]
        offs, pos = [], 5
        for s in streams:
            offs.append(pos)
            pos += len(s) + 1 + (pos % 3)
        src = np.zeros(pos + 16, dtype=np.uint8)
        for s, o in zip(streams, offs):
            src[o:o + len(s)] = np.frombuffer(s, dtype=np.uint8)
        sizes = torch.tensor([len(s) for s in streams], dtype=torch.int32).cuda()
        before = dec.launches
        _, out = dec.decode_device(torch.from_numpy(src).cuda(), sizes, stride, dst=dst, dst_cap=cap, format=S.GZIP,
                                   src_offsets=torch.tensor(offs, dtype=torch.int64).cuda())
        torch.cuda.synchronize()
        assert dec.launches - before == 3 * 3
        codes = out.cpu().tolist()
        head = dst[:, :256].cpu().numpy()
        for c, s in enumerate(streams):
            r, want = F.orc_decode(S.GZIP, s, cap)
            assert codes[c] == r, (rot, c, codes[c], r)
            if r >= 0:
                assert r <= 256 and head[c, :r].tobytes() == want, (rot, c)
        assert {codes[c] for c in where} >= {-5, -9, -4, -12}


def test_scratch_passes_chunks(dec):
    # stored inputs of 8 MiB into 100 MiB caps: about 35.7 M records each (the 4 * slen term), 7 per 4 GiB pass; small
    # inputs between them move the break to item 11.  Item 10, the last of the first pass, has a bad CRC; item 11, the
    # first of the second, ends in a block of type 3.
    rng = random.Random(43)
    big_n, big_cap = 8 << 20, 100 << 20
    items = []
    for k in range(12):
        if k in (1, 4, 5, 9):
            content = F.text(rng, rng.randrange(10, 4000))
            items.append((F.gzip_member(content, 6), 8192))
            continue
        content = rng.randbytes(big_n - k)
        w = S.Writer()
        for i in range(0, len(content), 65535):
            w.stored(content[i:i + 65535], final=k != 11 and i + 65535 >= len(content))
        if k == 11:
            w.bits(1, 1).bits(3, 2)
        items.append((S.gzip_wrap(w.data(), content, crc=zlib.crc32(content) ^ (k == 10)), big_cap))
    data, caps = [s for s, _ in items], [c for _, c in items]
    passes = _passes([_rec_cap(len(s), c) for s, c in items])
    assert passes == [(0, 11), (11, 12)], passes
    before = dec.launches
    got = dec.decode_chunks(data, caps, S.GZIP)
    assert dec.launches - before == 3 * len(passes)
    _expect(got, S.GZIP, data, caps, ["item %d" % i for i in range(len(items))])
    assert got[1][10] == -9 and got[1][11] == -5
