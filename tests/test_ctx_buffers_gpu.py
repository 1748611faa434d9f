"""The buffers a library context owns grow on demand and are shared between call kinds: the host-batch buffers by the zstd
decode, S2 block and huff0 host calls, the staged decoder's records by zstd decode and huff0 decompress, the S2 stream
buffers by stream encode and decode, the work pool by every encode call.  One context created through the C ABI runs every
call kind interleaved, at sizes that go small -> large -> small, so that each buffer grows while other kinds still use it;
every result must equal the same call on a fresh context, byte for byte, and decode back.  Run on an H100: python -m
pytest tests -m gpu."""
import ctypes

import numpy as np
import pytest
import torch

import helpers as H

pytestmark = pytest.mark.gpu

ZSTD_FLAGS = 3          # B2C_ZSTD_CRC | B2C_ZSTD_FRAME
S2_FAST = 1
HUF_4X = 1
BLOCK = 65536


def _lib():
    from compress_b200._lib import lib, check
    return lib, check


def _arr(t, vals):
    return (t * len(vals))(*vals)


def _table(fn, ctx, pre, blobs, caps, with_caps=True, rows=False):
    """A pointer-table call: blobs[i] -> (output bytes, code) per element (rows: the whole output buffer)."""
    lib, check = _lib()
    n = len(blobs)
    bufs = [np.frombuffer(bytes(b) or b"\0", dtype=np.uint8) for b in blobs]
    outs = [np.zeros(max(int(c), 1), dtype=np.uint8) for c in caps]
    res = (ctypes.c_int64 * n)()
    args = [ctx, *pre, _arr(ctypes.c_void_p, [b.ctypes.data for b in bufs]), _arr(ctypes.c_size_t, [len(b) for b in blobs]),
            _arr(ctypes.c_void_p, [o.ctypes.data for o in outs])]
    if with_caps:
        args.append(_arr(ctypes.c_size_t, [int(c) for c in caps]))
    check(fn(*args, res, n), ctx)
    return [(outs[i].tobytes() if rows else outs[i][:max(int(res[i]), 0)].tobytes(), int(res[i])) for i in range(n)]


def zstd_encode_chunks(ctx, chunks):
    lib, _ = _lib()
    return _table(lib.b2c_zstd_encode_chunks, ctx, (1, ZSTD_FLAGS), chunks, [lib.b2c_zstd_bound(len(c), 1) + 16 for c in chunks])


def zstd_encode_frames(ctx, inputs):
    lib, _ = _lib()
    return _table(lib.b2c_zstd_encode_frames, ctx, (1, 1), inputs, [lib.b2c_zstd_frame_bound(len(c), 1) + 16 for c in inputs])


def zstd_encode_frames_device(ctx, inputs):
    lib, check = _lib()
    n = len(inputs)
    padded = [x + bytes(-len(x) % 16) for x in inputs]        # frames at 16-byte aligned offsets, as the host-buffer call places them
    offs = np.cumsum([0] + [len(x) for x in padded[:-1]]).astype(np.uint64)
    lens = np.array([len(x) for x in inputs], dtype=np.uint64)
    src = torch.frombuffer(bytearray(b"".join(padded) or b"\0"), dtype=torch.uint8).cuda()
    cap = sum(int(lib.b2c_zstd_frame_bound(len(x), 1)) for x in inputs) + 64
    dst = torch.empty(cap, dtype=torch.uint8, device="cuda")
    foff = torch.empty(n, dtype=torch.int64, device="cuda")
    fsz = torch.empty(n, dtype=torch.int64, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    check(lib.b2c_zstd_encode_frames_device(ctx, 1, 1, src.data_ptr(), offs.ctypes.data, lens.ctypes.data, n, dst.data_ptr(), cap,
                                            foff.data_ptr(), fsz.data_ptr(), ctypes.c_void_p(stream)), ctx)
    torch.cuda.synchronize()
    d = dst.cpu().numpy()
    return [(d[o:o + s].tobytes(), s) for o, s in zip(foff.cpu().tolist(), fsz.cpu().tolist())]


def zstd_encode_packed(ctx, data):
    """Pageable source and destination: the call stages both through the context's pinned buffers."""
    lib, check = _lib()
    src = np.frombuffer(data, dtype=np.uint8)
    nchunks = max(1, (len(data) + BLOCK - 1) // BLOCK)
    dst = np.zeros(len(data) + nchunks * 32 + 64, dtype=np.uint8)
    sizes = np.zeros(nchunks, dtype=np.int64)
    offs = np.zeros(nchunks, dtype=np.uint64)
    total = ctypes.c_size_t(0)
    check(lib.b2c_zstd_encode_packed(ctx, 1, ZSTD_FLAGS, src.ctypes.data, len(data), BLOCK, dst.ctypes.data, dst.size,
                                     sizes.ctypes.data, offs.ctypes.data, ctypes.byref(total)), ctx)
    return dst[:total.value].tobytes(), sizes.tolist(), offs.tolist()


def zstd_decode_chunks(ctx, frames, caps):
    lib, _ = _lib()
    return _table(lib.b2c_zstd_decode_chunks, ctx, (), frames, caps)


def s2_encode_chunks(ctx, blocks):
    lib, _ = _lib()
    return _table(lib.b2c_s2_encode_chunks, ctx, (S2_FAST, 0), blocks, [lib.b2c_s2_bound(len(b)) + 16 for b in blocks])


def s2_decode_chunks(ctx, blocks, caps):
    lib, _ = _lib()
    return _table(lib.b2c_s2_decode_chunks, ctx, (), blocks, caps)


def s2_encode_stream(ctx, data):
    lib, check = _lib()
    src = np.frombuffer(data, dtype=np.uint8)
    out = np.zeros(int(lib.b2c_s2_stream_bound(len(data), BLOCK)) + 16, dtype=np.uint8)
    n = ctypes.c_size_t(0)
    check(lib.b2c_s2_encode_stream(ctx, S2_FAST, 0, src.ctypes.data, len(data), BLOCK, out.ctypes.data, out.size, ctypes.byref(n)), ctx)
    return out[:n.value].tobytes()


def s2_decode_stream(ctx, stream, size):
    lib, check = _lib()
    src = np.frombuffer(stream, dtype=np.uint8)
    out = np.zeros(size + 64, dtype=np.uint8)
    n = ctypes.c_size_t(0)
    check(lib.b2c_s2_decode_stream(ctx, src.ctypes.data, len(stream), out.ctypes.data, out.size, ctypes.byref(n)), ctx)
    return out[:n.value].tobytes()


def huf_compress_chunks(ctx, blocks):
    lib, _ = _lib()
    return _table(lib.b2c_huf_compress_chunks, ctx, (HUF_4X,), blocks, [len(b) + 16 for b in blocks])


def huf_decompress_chunks(ctx, comp, sizes):
    lib, _ = _lib()
    return _table(lib.b2c_huf_decompress_chunks, ctx, (HUF_4X,), comp, sizes)


def huf_read_table(ctx, comp):
    lib, _ = _lib()
    return _table(lib.b2c_huf_read_table, ctx, (), comp, [260] * len(comp), with_caps=False, rows=True)


def decode_staged_flags(ctx, n):
    lib, check = _lib()
    f = np.zeros(n, dtype=np.uint8)
    check(lib.b2c_decode_staged_flags(ctx, n, f.ctypes.data), ctx)
    return f


class _Ctx:
    def __init__(self):
        lib, _ = _lib()
        self.h = lib.b2c_ctx_create(0, 64)
        assert self.h

    def close(self):
        lib, _ = _lib()
        lib.b2c_ctx_destroy(self.h)


def _workload(big, seed):
    text = H.synth_text(12 << 20 if big else 1 << 20, seed)
    k = lambda small, large: large if big else small
    return dict(
        chunks=[text[i * BLOCK:(i + 1) * BLOCK - (i * 977) % 5000] for i in range(k(3, 40))],
        inputs=[text[:k(150_000, 3_000_000)], text[5:5 + k(5000, 1_000_000)], b""],
        packed=text[:k(2, 150) * BLOCK - 777],      # 150 chunks: three batches, both pipeline slots
        blocks=[text[i * 30000:i * 30000 + BLOCK - 13 * i] for i in range(k(3, 60))],
        stream=text[:k(100_000, 6_000_000)],
        hblocks=[text[i * 50000:i * 50000 + k(10_000, 120_000)] for i in range(k(3, 30))])


def test_one_context_every_call_kind_sizes_grow_and_shrink(oracle_lib):
    from test_oracle_s2 import s2_decode as orc_s2_decode
    shared = _Ctx()

    def both(fn, *args):
        got = fn(shared.h, *args)
        fresh = _Ctx()
        try:
            want = fn(fresh.h, *args)
        finally:
            fresh.close()
        assert got == want, "%s: the shared context differs from a fresh one" % fn.__name__
        return got

    try:
        for r, big in enumerate((False, True, False)):
            w = _workload(big, seed=100 + r)
            frames = both(zstd_encode_chunks, w["chunks"])
            for (f, code), c in zip(frames, w["chunks"]):
                assert code > 0 and H.libzstd_decode(f, len(c)) == c
            s2b = both(s2_encode_chunks, w["blocks"])
            for (e, code), b in zip(s2b, w["blocks"]):
                assert code > 0 and orc_s2_decode(e, len(b)) == (len(b), b)
            # a stream of several frames per input, and single frames
            streams = [b"".join(f for f, _ in frames[i:i + 3]) for i in range(0, len(frames), 3)] + [f for f, _ in frames]
            wants = [b"".join(w["chunks"][i:i + 3]) for i in range(0, len(frames), 3)] + w["chunks"]
            assert both(zstd_decode_chunks, streams, [len(x) + 64 for x in wants]) == [(x, len(x)) for x in wants]
            fr = both(zstd_encode_frames, w["inputs"])
            for (f, code), x in zip(fr, w["inputs"]):
                assert code > 0 and H.libzstd_decode(f, len(x)) == x
            hc = both(huf_compress_chunks, w["hblocks"])
            assert all(code > 0 for _, code in hc)
            st = both(s2_encode_stream, w["stream"])
            assert both(s2_decode_chunks, [e for e, _ in s2b], [len(b) + 64 for b in w["blocks"]]) == \
                [(b, len(b)) for b in w["blocks"]]
            assert both(zstd_encode_frames_device, w["inputs"]) == fr
            assert both(huf_decompress_chunks, [c for c, _ in hc], [len(b) for b in w["hblocks"]]) == \
                [(b, len(b)) for b in w["hblocks"]]
            packed, sizes, offs = both(zstd_encode_packed, w["packed"])
            assert H.libzstd_decode(packed, len(w["packed"])) == w["packed"]
            assert both(s2_decode_stream, st, len(w["stream"])) == w["stream"]
            rows = both(huf_read_table, [c for c, _ in hc])
            assert all(code > 0 for _, code in rows)
            assert both(zstd_decode_chunks, [packed], [len(w["packed"]) + 64]) == [(w["packed"], len(w["packed"]))]
    finally:
        shared.close()


def test_staged_flags_zero_after_staged_huff0_decompress():
    """The staged huff0 decompress writes its records where the staged zstd decoder keeps its own: afterwards no input of
    the earlier zstd decode is reported as staged."""
    text = H.synth_text(1 << 20, 7)
    chunks = [text[i * BLOCK:(i + 1) * BLOCK] for i in range(8)]
    hblocks = [text[i * 40000:(i + 1) * 40000] for i in range(8)]
    c = _Ctx()
    try:
        frames = [f for f, _ in zstd_encode_chunks(c.h, chunks)]
        assert zstd_decode_chunks(c.h, frames, [BLOCK + 64] * 8) == [(x, BLOCK) for x in chunks]
        assert decode_staged_flags(c.h, 8).any(), "the zstd decode did not run the staged kernels"
        comp = [x for x, _ in huf_compress_chunks(c.h, hblocks)]
        assert huf_decompress_chunks(c.h, comp, [len(b) for b in hblocks]) == [(b, len(b)) for b in hblocks]
        assert not decode_staged_flags(c.h, 8).any()
    finally:
        c.close()
