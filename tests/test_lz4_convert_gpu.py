"""LZ4 / LZ4s -> S2 / Snappy conversion on the device (b2c_s2_convert_lz4_*): bytes, decoded sizes and error codes equal the
oracle's (oracle/orc_lz4.c) for the seeded pool and the reference's fuzz seeds, in both formats and both outputs, at each
sampled block's smallest accepted slot and one byte below; every output decodes with the library's own S2 decoder."""
import numpy as np
import pytest
import torch

import helpers as H
import lz4_util as U
from compress_b200 import s2

pytestmark = pytest.mark.gpu
MODES = [(False, False), (False, True), (True, False), (True, True)]   # (lz4s, snappy)


@pytest.fixture(scope="module")
def codec():
    c = s2.Codec()
    yield c
    c.close()


@pytest.fixture(scope="module")
def pools():
    return {lz4s: U.pool(seed=11, lz4s=lz4s) for lz4s in (False, True)}


def _cap(src):
    return 2 * len(src) + 64


def _expect(cache, src, cap, lz4s, snappy):
    k = (src, cap, lz4s, snappy)
    if k not in cache:
        cache[k] = U.slot_result(src, cap, lz4s, snappy)
    return cache[k]


def _check(codec, blocks, caps, outs, codes, ns, lz4s, snappy, cache):
    for i, (b, cap) in enumerate(zip(blocks, caps)):
        want = _expect(cache, b, cap, lz4s, snappy)
        got = (codes[i], outs[i], ns[i] if codes[i] >= 0 or codes[i] == U.TOO_BIG else 0)
        assert got == want, (i, len(b), cap, lz4s, snappy, got[0], want[0])
    ok = [i for i in range(len(blocks)) if codes[i] >= 0]
    back, dcodes = codec.decode_blocks([outs[i] for i in ok], [max(ns[i], 1) for i in ok])
    assert dcodes == [ns[i] for i in ok]


@pytest.mark.parametrize("lz4s,snappy", MODES)
def test_pool_and_capacity_thresholds(codec, pools, lz4s, snappy):
    cache = {}
    blocks = pools[lz4s]
    outs, codes, ns = codec.convert_lz4_blocks(blocks, [_cap(b) for b in blocks], lz4s=lz4s, snappy=snappy)
    _check(codec, blocks, [_cap(b) for b in blocks], outs, codes, ns, lz4s, snappy, cache)
    rng = np.random.default_rng(3)
    sample, caps = [], []
    for i in rng.choice(len(blocks), size=min(40, len(blocks)), replace=False):
        m = U.min_cap(blocks[i], lz4s, snappy)
        if m is None:
            continue
        sample += [blocks[i], blocks[i]]
        caps += [m, m - 1]
    outs, codes, ns = codec.convert_lz4_blocks(sample, caps, lz4s=lz4s, snappy=snappy)
    _check(codec, sample, caps, outs, codes, ns, lz4s, snappy, cache)
    assert all(codes[k] >= 0 and codes[k + 1] < 0 for k in range(0, len(sample), 2))


def test_fuzz_seeds(codec):
    seeds = [s for _, s in U.fuzz_seeds() if len(s) <= (1 << 20)]
    for lz4s, snappy in MODES:
        caps = [_cap(b) for b in seeds]
        outs, codes, ns = codec.convert_lz4_blocks(seeds, caps, lz4s=lz4s, snappy=snappy)
        _check(codec, seeds, caps, outs, codes, ns, lz4s, snappy, {})


@pytest.mark.parametrize("n", [1, 33, 4097, 16397])
def test_device_batches_unaligned_with_sentinels(codec, pools, n):
    """The device form with per-block source and slot offsets (odd alignments), 0xA5 sentinels between the slots."""
    cache = {}
    for lz4s, snappy in MODES:
        pool = pools[lz4s]
        blocks = [pool[(i * 7 + n) % len(pool)] for i in range(n)]
        smax = max(len(b) for b in blocks)
        cap = 2 * smax + 64
        src_off, pos = [], 3
        for b in blocks:
            src_off.append(pos)
            pos += len(b) + (pos % 5)
        src = np.zeros(pos + 16, dtype=np.uint8)
        for o, b in zip(src_off, blocks):
            src[o:o + len(b)] = np.frombuffer(b, dtype=np.uint8)
        dst_off = [1 + i * (cap + 9) for i in range(n)]
        dst = torch.full((dst_off[-1] + cap + 9,), 0xA5, dtype=torch.uint8, device="cuda")
        d_src = torch.from_numpy(src).cuda()
        sizes = torch.tensor([len(b) for b in blocks], dtype=torch.int32).cuda()
        so = torch.tensor(src_off, dtype=torch.int64).cuda()
        do = torch.tensor(dst_off, dtype=torch.int64).cuda()
        _, out_sizes, dec = codec.convert_lz4_device(d_src, sizes, smax, lz4s=lz4s, snappy=snappy, dst=dst, dst_cap=cap,
                                                     src_offsets=so, dst_offsets=do, dst_stride=0)
        torch.cuda.synchronize()
        host = dst.cpu().numpy()
        codes, ns = out_sizes.cpu().tolist(), dec.cpu().tolist()
        outs = [host[o:o + c].tobytes() if c >= 0 else None for o, c in zip(dst_off, codes)]
        _check(codec, blocks, [cap] * n, outs, codes, ns, lz4s, snappy, cache)
        for i, o in enumerate(dst_off):                 # the bytes between slots are untouched
            assert (host[o + cap:o + cap + 9] == 0xA5).all(), i
        assert host[0] == 0xA5


def test_host_and_device_forms_agree(codec, pools):
    for lz4s, snappy in MODES:
        blocks = pools[lz4s][:200]
        stride = (max(len(b) for b in blocks) + 15) // 16 * 16
        cap = 2 * stride + 64
        src = torch.zeros(len(blocks) * stride, dtype=torch.uint8)
        for i, b in enumerate(blocks):
            if b:
                src[i * stride:i * stride + len(b)] = torch.frombuffer(bytearray(b), dtype=torch.uint8)
        sizes = torch.tensor([len(b) for b in blocks], dtype=torch.int32).cuda()
        dst, out_sizes, dec = codec.convert_lz4_device(src.cuda(), sizes, stride, lz4s=lz4s, snappy=snappy, dst_cap=cap)
        torch.cuda.synchronize()
        codes, ns = out_sizes.cpu().tolist(), dec.cpu().tolist()
        outs_h, codes_h, ns_h = codec.convert_lz4_blocks(blocks, [cap] * len(blocks), lz4s=lz4s, snappy=snappy)
        assert codes == codes_h and ns == ns_h
        d = dst.cpu().numpy()
        assert [d[i, :c].tobytes() if c >= 0 else None for i, c in enumerate(codes)] == outs_h


def test_large_blocks(codec):
    text = H.synth_text(4 << 20)
    zeros = bytes((16 << 20) + 12345)                   # one match far above 2^24: the S2 repeat is split
    for lz4s in (False, True):
        blocks = [U.compress(text, lz4s), U.compress(zeros, lz4s)]
        for snappy in (False, True):
            caps = [len(text) + (len(text) >> 1), 3 * (len(zeros) // 64) + 4096]
            outs, codes, ns = codec.convert_lz4_blocks(blocks, caps, lz4s=lz4s, snappy=snappy)
            _check(codec, blocks, caps, outs, codes, ns, lz4s, snappy, {})
            assert ns == [len(text), len(zeros)]
            if not snappy:
                assert codes[1] < 64
    # the device form with a block larger than src_stride is refused for that block alone
    src = torch.zeros(64, dtype=torch.uint8, device="cuda")
    sizes = torch.tensor([40, 8], dtype=torch.int32, device="cuda")
    _, o, _ = codec.convert_lz4_device(src, sizes, 32, dst_cap=256)
    assert o.cpu().tolist()[0] == -102


def test_two_streams_alternating_with_s2_decode(codec, pools):
    blocks = [b for b in pools[False] if b][:64]
    stride = (max(len(b) for b in blocks) + 15) // 16 * 16
    cap = 2 * stride + 64
    src = torch.zeros(len(blocks) * stride, dtype=torch.uint8)
    for i, b in enumerate(blocks):
        src[i * stride:i * stride + len(b)] = torch.frombuffer(bytearray(b), dtype=torch.uint8)
    src = src.cuda()
    sizes = torch.tensor([len(b) for b in blocks], dtype=torch.int32).cuda()
    want, wcodes, wns = codec.convert_lz4_blocks(blocks, [cap] * len(blocks))
    ok = [i for i, c in enumerate(wcodes) if c >= 0]
    s2blocks = [want[i] for i in ok]
    s2stride = (max(len(b) for b in s2blocks) + 15) // 16 * 16
    s2src = torch.zeros(len(ok) * s2stride, dtype=torch.uint8)
    for k, b in enumerate(s2blocks):
        s2src[k * s2stride:k * s2stride + len(b)] = torch.frombuffer(bytearray(b), dtype=torch.uint8)
    s2src = s2src.cuda()
    s2sizes = torch.tensor([len(b) for b in s2blocks], dtype=torch.int32).cuda()
    dcap = max(wns[i] for i in ok) + 16
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    results = []
    for it in range(6):
        with torch.cuda.stream(streams[it & 1]):
            if it % 3 == 2:
                d, o = codec.decode_device(s2src, s2sizes, s2stride, dst_cap=dcap)
                results.append(("dec", d, o))
            else:
                d, o, n = codec.convert_lz4_device(src, sizes, stride, dst_cap=cap)
                results.append(("cvt", d, o, n))
    torch.cuda.synchronize()
    for r in results:
        if r[0] == "cvt":
            codes = r[2].cpu().tolist()
            assert codes == wcodes and r[3].cpu().tolist() == wns
            d = r[1].cpu().numpy()
            assert [d[i, :c].tobytes() for i, c in enumerate(codes) if c >= 0] == s2blocks
        else:
            assert r[2].cpu().tolist() == [wns[i] for i in ok]


def test_converter_mirror(codec):
    tw = H.golden("twain.txt")[:50000]
    for cls, lz4s in ((s2.LZ4Converter, False), (s2.LZ4sConverter, True)):
        conv = cls(codec=codec)
        blk = U.compress(tw, lz4s)
        for snappy, fn in ((False, conv.ConvertBlock), (True, conv.ConvertBlockSnappy)):
            r, body, n = U.convert(blk, 100000, lz4s, snappy, prefix=b"head")
            out, got_n = fn(b"head", blk, 100004)
            assert out == b"head" + body and got_n == n == len(tw)
            assert codec.Decode(U.uvarint(n) + out[4:]) == tw
            m = U.min_cap(blk, lz4s, snappy) - 5
            assert fn(b"", blk, m)[1] == n
            with pytest.raises(s2.ErrDstTooSmall):
                fn(b"", blk, m - 1)
        with pytest.raises(s2.ErrCorrupt):
            conv.ConvertBlock(b"", blk[:-3], 100000)
        assert conv.ConvertBlock(b"xy", b"", 2) == (b"xy", 0)


def test_pyarrow_lz4_raw_blocks(codec):
    pa = pytest.importorskip("pyarrow")
    tw = H.golden("twain.txt")
    datas = [tw[:65536], tw[100000:100000 + 3000], bytes(100000), H.golden("html.txt")[:65536]]
    blocks = [pa.compress(d, codec="lz4_raw", asbytes=True) for d in datas]
    for snappy in (False, True):
        caps = [2 * len(d) + 64 for d in datas]
        outs, codes, ns = codec.convert_lz4_blocks(blocks, caps, snappy=snappy)
        _check(codec, blocks, caps, outs, codes, ns, False, snappy, {})
        assert ns == [len(d) for d in datas]
        for d, o in zip(datas, outs):
            if snappy:
                assert pa.decompress(o, decompressed_size=len(d), codec="snappy", asbytes=True) == d
            assert codec.Decode(o) == d
