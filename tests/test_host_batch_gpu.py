"""The contract the pointer-table calls share (HostBatch in b2c_api.cu), for each of them: zstd decode, S2 block encode and
decode, LZ4 -> S2 conversion, inflate, stateless deflate, huff0 compress and decompress.  Empty batches, empty pieces, sizes
around every 16-byte boundary, the per-call size limit, a capacity one byte short, sparse results (the per-piece scatter)
and, for inflate, a batch whose packed input passes the 1 GiB staging limit (the per-piece gather).  Every result is checked
against the oracle or a round trip.  Run on an H100: python -m pytest tests -m gpu."""
import ctypes
import zlib

import pytest

import helpers as H

pytestmark = pytest.mark.gpu

ERR_DST_SMALL, ERR_ARG = -4, -102
SIZES = [0, 1, 15, 16, 17, 31, 32, 33, 255, 256, 257, 4095, 4096, 4097, 65519, 65520, 65521, 65535, 65536]


def _gzip(data, level=6):
    c = zlib.compressobj(level, zlib.DEFLATED, 31)
    return c.compress(data) + c.flush()


class Call:
    """One pointer-table call: `args` puts the table into the call's argument order; `inp` is the input blob for content
    `data`, `cap` a capacity it fits; `verify` asserts a full-capacity result; `short` gives (capacity, expected code) one
    byte short of a result of `code` bytes, the code None where only its class (an error) is fixed."""
    encoder = False
    limit = 0xffffffff

    def run(self, ctx, blobs, caps, fake=None):
        """-> (call rc, outputs, codes); fake = (i, size): a size piece i does not have, passed to the call."""
        from compress_b200._lib import lib, PointerTable
        t = PointerTable(blobs, caps)
        if fake:
            t.ssz[fake[0]] = fake[1]
        rc = getattr(lib, self.fn)(*self.args(ctx, t))
        outs, codes = t.results()
        return rc, outs, codes

    def cap(self, data, blob):
        return len(data)

    def short(self, data, blob, code):
        return (code - 1, ERR_DST_SMALL) if self.encoder and code > 0 else None

    def sparse_cap(self, data, blob):
        return 64 * self.cap(data, blob) + 4096


class ZstdDecode(Call):
    fn = "b2c_zstd_decode_chunks"

    def args(self, ctx, t):
        return ctx, t.srcs, t.ssz, t.dsts, t.dcap, t.res, t.n

    def inp(self, data):
        return H.oracle_encode(data)[1]

    def verify(self, data, blob, cap, out, code):
        assert (code, out) == (len(data), data)

    def short(self, data, blob, code):
        return (len(data) - 1, H.oracle_decode(blob, len(data) - 1)[0]) if data else None


class S2Encode(Call):
    fn, encoder = "b2c_s2_encode_chunks", True

    def args(self, ctx, t):
        return ctx, 1, 0, t.srcs, t.ssz, t.dsts, t.dcap, t.res, t.n

    def inp(self, data):
        return data

    def cap(self, data, blob):
        from compress_b200._lib import lib
        return int(lib.b2c_s2_bound(len(data)))

    def verify(self, data, blob, cap, out, code):
        from test_oracle_s2 import s2_decode
        assert code > 0 and s2_decode(out, len(data)) == (len(data), data)


class S2Decode(Call):
    fn = "b2c_s2_decode_chunks"

    def args(self, ctx, t):
        return ctx, t.srcs, t.ssz, t.dsts, t.dcap, t.res, t.n

    def inp(self, data):
        _, outs, _ = S2Encode().run(_ctx(), [data], [len(data) + len(data) // 6 + 32])
        return outs[0]

    def verify(self, data, blob, cap, out, code):
        assert (code, out) == (len(data), data)

    def short(self, data, blob, code):
        from test_oracle_s2 import s2_decode
        return (len(data) - 1, s2_decode(blob, len(data) - 1)[0]) if data else None


class Lz4Convert(Call):
    fn = "b2c_s2_convert_lz4_chunks"

    def args(self, ctx, t):
        self.dec = (ctypes.c_int64 * t.n)()
        return ctx, 0, 0, t.srcs, t.ssz, t.dsts, t.dcap, t.res, self.dec, t.n

    def inp(self, data):
        import lz4_util
        return lz4_util.compress(data)

    def cap(self, data, blob):
        return len(data) + len(data) // 6 + 32

    def verify(self, data, blob, cap, out, code):
        import lz4_util
        assert (code, out) == lz4_util.slot_result(blob, cap)[:2]

    def short(self, data, blob, code):
        import lz4_util
        return (code - 1, lz4_util.slot_result(blob, code - 1)[0]) if code > 0 else None


class Inflate(Call):
    fn = "b2c_flate_decode_chunks"

    def args(self, ctx, t):
        return ctx, 2, 0, t.srcs, t.ssz, t.dsts, t.dcap, t.res, t.n

    def inp(self, data):
        return _gzip(data)

    def verify(self, data, blob, cap, out, code):
        assert (code, out) == (len(data), data)

    def short(self, data, blob, code):
        return (len(data) - 1, ERR_DST_SMALL) if data else None


class StatelessDeflate(Call):
    fn, encoder = "b2c_flate_stateless_chunks", True

    def args(self, ctx, t):
        return ctx, 0, 0, t.srcs, t.ssz, None, None, None, None, 0, t.dsts, t.dcap, t.res, None, None, t.n

    def inp(self, data):
        return data

    def cap(self, data, blob):
        import deflate_util
        return deflate_util.bound(len(data))

    def verify(self, data, blob, cap, out, code):
        import deflate_util
        want = deflate_util.stateless(data)
        assert (code, out) == (len(want), want) and zlib.decompress(out, -15) == data


class HufCompress(Call):
    fn, encoder, limit = "b2c_huf_compress_chunks", True, 0x7fffffff

    def args(self, ctx, t):
        return ctx, 1, t.srcs, t.ssz, t.dsts, t.dcap, t.res, t.n

    def inp(self, data):
        return data

    def cap(self, data, blob):
        return len(data) + 16

    def verify(self, data, blob, cap, out, code):
        from test_emu_huf0 import orc_compress
        want, wcode = orc_compress(data, True)
        assert code == wcode and (code < 0 or out == want)


class HufDecompress(Call):
    fn, limit = "b2c_huf_decompress_chunks", 0x7fffffff

    def args(self, ctx, t):
        return ctx, 1, t.srcs, t.ssz, t.dsts, t.dcap, t.res, t.n

    def inp(self, data):
        from test_emu_huf0 import orc_compress
        comp, code = orc_compress(data, True)
        return comp if code > 0 else None      # only compressible content has a huff0 block

    def verify(self, data, blob, cap, out, code):
        assert (code, out) == (len(data), data)

    def short(self, data, blob, code):
        return (len(data) - 1, None) if data else None

    def sparse_cap(self, data, blob):
        return len(data)         # exact sizes: the stride of the largest output leaves the smaller ones sparse


CALLS = [ZstdDecode(), S2Encode(), S2Decode(), Lz4Convert(), Inflate(), StatelessDeflate(), HufCompress(), HufDecompress()]
IDS = [type(c).__name__ for c in CALLS]
_CTX = []


def _ctx():
    if not _CTX:
        from compress_b200._lib import Context
        _CTX.append(Context())
    return _CTX[0]._ctx


def _pieces(call, sizes, seed):
    text = H.synth_text(sum(sizes) + 1, seed)
    datas, o = [], 0
    for s in sizes:
        datas.append(text[o:o + s])
        o += s
    blobs = [call.inp(d) for d in datas]
    keep = [i for i, b in enumerate(blobs) if b is not None]
    return [datas[i] for i in keep], [blobs[i] for i in keep]


def _check(call, datas, blobs, caps):
    rc, outs, codes = call.run(_ctx(), blobs, caps)
    assert rc == 0
    for d, b, c, o, code in zip(datas, blobs, caps, outs, codes):
        call.verify(d, b, c, o, code)
    return codes


@pytest.mark.parametrize("call", CALLS, ids=IDS)
def test_empty_batch(call):
    rc, outs, codes = call.run(_ctx(), [], [])
    assert (rc, outs, codes) == (0, [], [])


@pytest.mark.parametrize("call", CALLS, ids=IDS)
def test_empty_pieces_and_sizes_off_16_byte_boundaries(call):
    """Every size around a 16-byte boundary, with empty pieces between them: packed offsets of every alignment."""
    sizes = [s for x in SIZES for s in (x, 0)]
    datas, blobs = _pieces(call, sizes, seed=11)
    _check(call, datas, blobs, [call.cap(d, b) for d, b in zip(datas, blobs)])


@pytest.mark.parametrize("call", CALLS, ids=IDS)
def test_size_limit_is_an_argument_error(call):
    """A piece above the call's size limit fails the whole call before any of its bytes are read."""
    datas, blobs = _pieces(call, [1000, 2000, 3000], seed=12)
    caps = [call.cap(d, b) for d, b in zip(datas, blobs)]
    assert call.run(_ctx(), blobs, caps, fake=(1, call.limit + 1))[0] == ERR_ARG
    _check(call, datas, blobs, caps)           # the context still works


@pytest.mark.parametrize("call", CALLS, ids=IDS)
def test_capacity_one_byte_short(call):
    """An encoder's result one byte over its capacity is B2C_ERR_DST_SMALL; a decoder keeps its own code for it.  The last
    piece keeps its full capacity, so that the stride-addressed calls give every piece room on the device."""
    datas, blobs = _pieces(call, [17, 4096, 40000, 65536], seed=13)
    full = [call.cap(d, b) for d, b in zip(datas, blobs)]
    codes = _check(call, datas, blobs, full)
    short = [(b, call.short(d, b, code)) for d, b, code in zip(datas, blobs, codes)]
    short = [(b, s) for b, s in short if s is not None]
    assert short
    rc, outs, got = call.run(_ctx(), [b for b, _ in short] + blobs[-1:], [s[0] for _, s in short] + full[-1:])
    assert rc == 0
    for (_, (cap, want)), code in zip(short, got):
        assert code < 0 and want in (None, code), (cap, code, want)
    call.verify(datas[-1], blobs[-1], full[-1], outs[-1], got[-1])


@pytest.mark.parametrize("call", CALLS, ids=IDS)
def test_sparse_results_scatter_per_piece(call):
    """Capacities far above the results: the results fill under half the output range and are copied piece by piece."""
    datas, blobs = _pieces(call, [100, 300, 5000, 200, 60000, 7], seed=14)
    _check(call, datas, blobs, [call.sparse_cap(d, b) for d, b in zip(datas, blobs)])


def test_inflate_batch_over_the_staging_limit():
    """17 gzip members of 64 MiB of stored blocks: the packed input and output pass 1 GiB, so both the gather and the
    scatter copy piece by piece."""
    call = Inflate()
    data = H.synth_text(64 << 20, 15)
    member = _gzip(data, 0)
    n = 17
    assert n * len(member) > 1 << 30
    rc, outs, codes = call.run(_ctx(), [member] * n, [len(data)] * n)
    assert rc == 0 and codes == [len(data)] * n
    assert all(o == data for o in outs)
