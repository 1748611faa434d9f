"""GPU tests of the S2 best level (B2C_S2_BEST: s2.EncodeBest / EncodeSnappyBest) through the C ABI and the Python
interface: the device's bytes equal the emulated kernels', everything decodes with the oracle, the device's staged
decoder and pyarrow's Snappy, edge sizes and batch shapes, 256 MiB device-resident, the stored-or-tags decision, and
streams / Writer output with the chunk types s2.Writer would choose."""
import io

import numpy as np
import pytest
import torch

import helpers as H
import s2_stream_ref as R
import s2best_util as U
from test_s2_best_oracle import _blocks

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def codec():
    from compress_b200 import s2
    c = s2.Codec()
    yield c
    c.close()


@pytest.fixture(scope="module")
def E():
    return U.emu()


def _mode(snappy):
    return U.SNAPPY_BEST if snappy else U.BEST


@pytest.mark.parametrize("snappy", [False, True])
def test_best_equals_emulator_and_decodes(codec, E, snappy):
    blocks = [b for b in _blocks() + U.fuzz_seeds() if len(b) <= 65536]
    dev = codec.encode_blocks(blocks, snappy=snappy, best=True)
    emu, _ = U.emu_encode(E, blocks, snappy=snappy)
    assert dev == emu
    for i, (b, c) in enumerate(zip(blocks, dev)):
        r, got = U.decode(c, len(b))
        assert r == len(b) and got == b, i
    outs, codes = codec.decode_blocks(dev, [len(b) for b in blocks])
    assert outs == blocks, codes
    if snappy:
        pa = pytest.importorskip("pyarrow")
        pc = pa.Codec("snappy")
        for b, c in zip(blocks, dev):
            if b:
                assert pc.decompress(c, decompressed_size=len(b)).to_pybytes() == b


def test_best_staged_decode_covers_text(codec):
    tw = H.golden("twain.txt")
    blocks = [tw[i:i + 65536] for i in range(0, 5 * 65536, 65536)] + [b"ab" * 20000, bytes(50000), tw[:1000]]
    for snappy in (False, True):
        comps = codec.encode_blocks(blocks, snappy=snappy, best=True)
        outs, codes = codec.decode_blocks(comps, [len(b) for b in blocks])
        assert outs == blocks, codes
        assert codec.staged_count(len(blocks)) == len(blocks)


def test_best_edge_sizes_and_python_entry_points(codec, E):
    from compress_b200 import s2
    tw = H.golden("twain.txt")
    for n in (0, 1, 31, 32, 33, 65535, 65536):
        b = tw[:n]
        for snappy in (False, True):
            c = codec.encode_blocks([b], snappy=snappy, best=True)[0]
            assert c == U.emu_encode(E, [b], snappy=snappy)[0][0]
            assert len(c) <= s2.MaxEncodedLen(n) and U.decode(c, n)[1] == b
    big = tw[:200000]
    for fn, snappy in ((codec.EncodeBest, False), (codec.EncodeSnappyBest, True)):
        c = fn(big)
        assert codec.Decode(c) == big and U.decode(c, len(big))[1] == big
        assert c == s2.ConcatBlocks(codec.encode_blocks([big[o:o + 65536] for o in range(0, len(big), 65536)], snappy=snappy, best=True))
    with pytest.raises(ValueError):
        codec.encode_blocks([b"x" * 100], better=True, best=True)


def test_best_ratio_per_corpus(codec):
    """Per corpus (the corpora of test_s2_ratio_per_corpus) the device's best output is within +5 % of the serial
    EncodeBest / EncodeSnappyBest and smaller than its better output."""
    tw = H.golden("twain.txt")
    corp = {"twain": [tw[i:i + 65536] for i in range(0, len(tw), 65536)], "html": [H.golden("html.txt")],
            "e": [H.golden("e.txt")[:65536], H.golden("e.txt")[65536:]], "synth": H.synth_chunks("text", 8, seed=5)}
    for name, chunks in corp.items():
        for snappy in (False, True):
            ours = sum(len(x) for x in codec.encode_blocks(chunks, snappy=snappy, best=True))
            better = sum(len(x) for x in codec.encode_blocks(chunks, snappy=snappy, better=True))
            ref = sum(len(U.encode(c, _mode(snappy))) for c in chunks)
            assert ours <= 1.05 * ref and ours < better, (name, snappy, ours, ref, better)


@pytest.mark.parametrize("nblocks", [1, 7, 4097, 16384])
def test_best_batches_device_resident(codec, nblocks):
    src = H.synth_text_torch(nblocks * 65536, "cuda", seed=nblocks)
    sizes = torch.full((nblocks,), 65536, dtype=torch.int32, device="cuda")
    sizes[::3] = torch.arange(0, nblocks, 3, dtype=torch.int32, device="cuda") % 65537
    dst_a, out_a = codec.encode_device(src, best=True)
    dst_b, out_b = codec.encode_device(src, sizes=sizes, best=True)
    torch.cuda.synchronize()
    oa, ob = out_a.cpu().numpy(), out_b.cpu().numpy()
    assert (oa > 0).all() and (ob > 0).all()
    host = src.cpu().numpy()
    szs = sizes.cpu().numpy()
    pick = sorted(set([0, nblocks - 1] + list(range(0, nblocks, max(1, nblocks // 5)))))
    for i in pick:
        blk = host[i * 65536:(i + 1) * 65536].tobytes()
        ca = dst_a[i, :int(oa[i])].cpu().numpy().tobytes()
        assert U.decode(ca, 65536)[1] == blk
        cb = dst_b[i, :int(ob[i])].cpu().numpy().tobytes()
        assert U.decode(cb, int(szs[i]))[1] == blk[:int(szs[i])]
    if nblocks >= 4097:
        # the host-buffer call gives the same bytes as the device-resident one
        assert codec.encode_blocks([host[i * 65536:(i + 1) * 65536].tobytes() for i in pick], best=True) == \
            [dst_a[i, :int(oa[i])].cpu().numpy().tobytes() for i in pick]


def test_best_256mib_with_zero_and_random_blocks(codec):
    n = 4096
    src = H.synth_text_torch(n * 65536, "cuda", seed=3)
    src[5 * 65536:6 * 65536] = 0
    g = torch.Generator(device="cuda").manual_seed(9)
    src[9 * 65536:10 * 65536] = torch.randint(0, 256, (65536,), dtype=torch.uint8, device="cuda", generator=g)
    dst, outs = codec.encode_device(src, best=True)
    torch.cuda.synchronize()
    o = outs.cpu().numpy()
    assert (o > 0).all()
    assert o[9] == 3 + 3 + 65536 and o[5] < 64
    ratio = float(o.sum()) / src.numel()
    assert ratio < 0.8, ratio
    host = src.cpu().numpy()
    for i in (0, 5, 9, 1234, n - 1):
        assert U.decode(dst[i, :int(o[i])].cpu().numpy().tobytes(), 65536)[1] == host[i * 65536:(i + 1) * 65536].tobytes()


@pytest.mark.parametrize("snappy", [False, True])
def test_best_random_with_repeat_is_tags(codec, snappy):
    b = U.random_with_repeat()
    c = codec.encode_blocks([b], snappy=snappy, best=True)[0]
    ref = U.encode(b, _mode(snappy))
    assert len(ref) < 65536 and len(c) < 65536 - 900 and U.decode(c, len(b))[1] == b
    better = codec.encode_blocks([b], snappy=snappy, better=True)[0]
    assert len(better) == 3 + 3 + 65536


def _orc_decode_block(body, n):
    r, got = U.decode(body, n)
    return got if r == n else None


@pytest.mark.parametrize("snappy", [False, True])
def test_best_stream_and_writer(codec, snappy):
    """EncodeStream(best=True) and Writer(best=True): compressed chunks exactly where the block encoder returns tags
    (the random block with one repeat included), read back by DecodeStream and the reference reader model."""
    from compress_b200 import s2
    tw = H.golden("twain.txt")
    rng = np.random.default_rng(1)
    # blocks: two of text, the random block with one repeat, a random block, then a short tail
    data = tw[:131072] + U.random_with_repeat() + rng.integers(0, 256, 65536, dtype=np.uint8).tobytes() + bytes(20) + tw[:31]
    st = codec.EncodeStream(data, snappy=snappy, best=True)
    assert codec.DecodeStream(st, max_size=len(data) + 64) == data
    assert R.read_stream(st, _orc_decode_block) == data

    def enc_block(blk):         # encodeBlock of the device: b'' when the block is stored
        c = codec.encode_blocks([blk], snappy=snappy, best=True)[0]
        n = len(blk)
        hdr = 1 if n < 128 else (2 if n < 16384 else 3)
        lh = 0 if n == 0 else (1 if n <= 60 else (2 if n <= 256 else 3))
        return b"" if len(c) == hdr + lh + n else c[hdr:]
    assert st == R.write_stream(data, enc_block, snappy=snappy)
    # the chunk of the random-with-repeat block is compressed (type 0), the random block's is not (type 1)
    types, o = [], 10
    while o < len(st):
        types.append(st[o])
        o += 4 + (st[o + 1] | (st[o + 2] << 8) | (st[o + 3] << 16))
    assert types[:4] == [0x00, 0x00, 0x00, 0x01], types
    out = io.BytesIO()
    w = s2.Writer(out, codec=codec, best=True, snappy=snappy, batch_bytes=1 << 17)
    w.Write(data)
    w.Close()
    assert codec.DecodeStream(out.getvalue(), max_size=len(data) + 64) == data
    assert R.read_stream(out.getvalue(), _orc_decode_block) == data
    dst, total, err = codec.encode_stream_device(torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda(), snappy=snappy, best=True)
    torch.cuda.synchronize()
    assert int(err.item()) == 0 and dst[:int(total.item())].cpu().numpy().tobytes() == st


def test_level_4_unsupported_and_queue(codec):
    import ctypes
    from compress_b200._lib import lib
    src = np.frombuffer(b"x" * 1000, dtype=np.uint8)
    dst = np.zeros(2000, dtype=np.uint8)
    srcs = (ctypes.c_void_p * 1)(src.ctypes.data)
    dsts = (ctypes.c_void_p * 1)(dst.ctypes.data)
    ss = (ctypes.c_size_t * 1)(1000)
    dc = (ctypes.c_size_t * 1)(2000)
    res = (ctypes.c_int64 * 1)(0)
    assert lib.b2c_s2_encode_chunks(codec._ctx, 4, 0, srcs, ss, dsts, dc, res, 1) == -11      # B2C_ERR_UNSUPPORTED
    assert lib.b2c_s2_encode_chunks(codec._ctx, 3, 0, srcs, ss, dsts, dc, res, 1) == 0 and res[0] > 0
    from compress_b200 import zstd
    q = zstd.Queue(max_batch=64, linger_us=300)
    tw = H.golden("twain.txt")[:65536]
    for snappy in (False, True):
        assert q.S2Encode(tw, snappy=snappy, best=True) == codec.encode_blocks([tw], snappy=snappy, best=True)[0]
    q.close()
