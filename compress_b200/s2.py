"""Host-side mirror of the reference's S2 block interface for the accelerated path.

Names follow klauspost/compress/s2: ``Encode`` (s2/encode.go:29), ``EncodeBetter`` (:117), ``EncodeSnappy`` (:204),
``EncodeSnappyBetter`` (:248), ``Decode``
(s2/decode.go:58), ``MaxEncodedLen`` (s2/encode.go:389), ``ErrCorrupt`` / ``ErrTooLarge`` (s2/decode.go:17-26).
The work is done by libb200comp.so through the C ABI in include/b2c.h; device blocks are at most 64 KiB (the
``WriterBlockSize`` the GPU path is built for): ``encode_blocks`` raises ``ErrTooLarge`` beyond that, ``Encode*`` join
64 KiB pieces into one block with ``ConcatBlocks`` (s2/encode.go:322), ``EncodeStream`` / ``DecodeStream`` are the framing
format (s2.Writer / s2.Reader over a buffer), ``EncodeStream(index=True)`` / ``DecodeStreamRange`` the seek index on top of it
(``s2_index.py``).
"""
import ctypes

import numpy as np
import torch

from ._lib import lib, check, B2CError, Context, PointerTable
from . import s2_index
from .s2_index import Index, IndexStream, RemoveIndexHeaders, RestoreIndexHeaders   # noqa: F401  (s2/index.go)

BLOCK = 1 << 16
SLOT = BLOCK + 512
FAST = 1
BETTER = 2
BEST = 3
FLAG_SNAPPY = 1


def _level(better=False, best=False):
    """The block encoder class: FAST, BETTER (s2.EncodeBetter's) or BEST (s2.EncodeBest's); the last two exclude each other."""
    if better and best:
        raise ValueError("s2: better and best exclude each other")
    return BEST if best else (BETTER if better else FAST)


class ErrCorrupt(B2CError):
    pass


class ErrCRC(B2CError):
    """s2.ErrCRC (s2/decode.go:20)"""


class ErrUnsupported(B2CError):
    """s2.ErrUnsupported (s2/decode.go:24)"""


class ErrTooLarge(B2CError):
    pass


class ErrDstTooSmall(B2CError):
    """s2.ErrDstTooSmall (s2/lz4convert.go:19)"""


def MaxEncodedLen(n):
    r = int(lib.b2c_s2_bound(n))
    return r if (r or n == 0) and n <= 0xffffffff else -1


def _decoded_len(block):
    """decodedLen (s2/decode.go:36-49): (length, header bytes) of a block, ErrCorrupt on a bad varint."""
    v, shift = 0, 0
    for k in range(10):
        if k >= len(block):
            raise ErrCorrupt("s2: corrupt input")
        b = block[k]
        v |= (b & 0x7F) << shift
        if b < 0x80:
            if k + 1 > 5 or v > 0xFFFFFFFF:
                raise ErrCorrupt("s2: corrupt input")
            return v, k + 1
        shift += 7
    raise ErrCorrupt("s2: corrupt input")


def ConcatBlocks(blocks, dst=None):
    """s2.ConcatBlocks (s2/encode.go:322-361): the blocks' bodies behind one length header -- a single valid block.  Host-side
    byte work, as in the reference (the blocks are not validated)."""
    total, bodies = 0, []
    for b in blocks:
        n, hdr = _decoded_len(b)
        total += n
        bodies.append(bytes(b[hdr:]))
    out = bytearray() if dst is None else dst
    if total == 0:
        out.append(0)
        return bytes(out) if dst is None else out
    if total > 0xFFFFFFFF:
        raise ErrTooLarge("s2: decoded block is too large")
    v = total
    while v >= 0x80:
        out.append((v & 0x7F) | 0x80)
        v >>= 7
    out.append(v)
    for body in bodies:
        out += body
    return bytes(out) if dst is None else out


# class Codec: batches of S2 blocks on one GPU.  The helpers above need neither torch nor the library, and
# tests/test_s2_stream_model.py runs them on their own by cutting this file at this line's first words.
class Codec(Context):
    """Batch S2 block encoder/decoder on one GPU."""

    @property
    def launches(self):
        return int(lib.b2c_launch_count(self._ctx))

    # ---- device-resident batches --------------------------------------------------------------
    def encode_device(self, src, sizes=None, block=BLOCK, snappy=False, dst=None, out_sizes=None, better=False, best=False):
        """src: uint8 CUDA tensor, block i at i*block.  Returns (dst [n, SLOT], out_sizes int64).  Async."""
        assert src.is_cuda and src.dtype == torch.uint8
        level = _level(better, best)
        n = src.numel() // block if sizes is None else sizes.numel()
        if dst is None:
            dst = torch.empty((n, SLOT), dtype=torch.uint8, device=src.device)
        if out_sizes is None:
            out_sizes = torch.empty((n,), dtype=torch.int64, device=src.device)
        stream = torch.cuda.current_stream(src.device).cuda_stream
        check(lib.b2c_s2_encode_device(self._ctx, level, FLAG_SNAPPY if snappy else 0, src.data_ptr(), block,
                                       None if sizes is None else sizes.data_ptr(), block, dst.data_ptr(), SLOT,
                                       out_sizes.data_ptr(), n, ctypes.c_void_p(stream)), self._ctx)
        return dst, out_sizes

    def decode_device(self, src, src_sizes, src_stride, dst=None, dst_cap=BLOCK, out_sizes=None):
        assert src.is_cuda and src.dtype == torch.uint8
        n = src_sizes.numel()
        if dst is None:
            dst = torch.empty((n, dst_cap), dtype=torch.uint8, device=src.device)
        if out_sizes is None:
            out_sizes = torch.empty((n,), dtype=torch.int64, device=src.device)
        stream = torch.cuda.current_stream(src.device).cuda_stream
        check(lib.b2c_s2_decode_device(self._ctx, src.data_ptr(), src_stride, None, src_sizes.data_ptr(), dst.data_ptr(),
                                       dst_cap, None, dst_cap, out_sizes.data_ptr(), n, ctypes.c_void_p(stream)), self._ctx)
        return dst, out_sizes

    # ---- host buffers ------------------------------------------------------------------------------
    def staged_count(self, n):
        """How many of the first n blocks of the last decode launch were finished by the staged kernels (diagnostics)."""
        k = ctypes.c_uint32(0)
        check(lib.b2c_s2_decode_staged_count(self._ctx, n, ctypes.byref(k)), self._ctx)
        return int(k.value)

    def staged_flags(self, n):
        """Per block of the first n of the last decode launch: 1 if the staged kernels finished it, else 0 (uint8 ndarray)."""
        f = np.zeros(n, dtype=np.uint8)
        check(lib.b2c_s2_decode_staged_flags(self._ctx, n, f.ctypes.data), self._ctx)
        return f

    def _host(self, fn, blobs, caps, *pre):
        t = PointerTable(blobs, caps)
        check(fn(self._ctx, *pre, t.srcs, t.ssz, t.dsts, t.dcap, t.res, t.n), self._ctx)
        return t.results()

    def encode_blocks(self, blocks, snappy=False, better=False, best=False):
        level = _level(better, best)
        if not blocks:
            return []
        outs, codes = self._host(lib.b2c_s2_encode_chunks, blocks, [MaxEncodedLen(len(b)) + 16 for b in blocks], level,
                                 FLAG_SNAPPY if snappy else 0)
        for c in codes:
            if c == -3:
                raise ErrTooLarge("s2: block larger than the GPU path's 64 KiB block size")
            if c < 0:
                raise B2CError(lib.b2c_strerror(c).decode())
        return outs

    def decode_blocks(self, blocks, caps):
        if not blocks:
            return [], []
        return self._host(lib.b2c_s2_decode_chunks, blocks, caps)

    def _encode_any(self, src, snappy=False, better=False, best=False):
        """One block for an input of any size: pieces of 64 KiB are encoded as one device batch and joined with ConcatBlocks
        (every piece's copies stay inside the piece, so the joined bodies are one valid block)."""
        if len(src) <= BLOCK:
            return self.encode_blocks([src], snappy=snappy, better=better, best=best)[0]
        src = bytes(src)
        parts = self.encode_blocks([src[o:o + BLOCK] for o in range(0, len(src), BLOCK)], snappy=snappy, better=better, best=best)
        return ConcatBlocks(parts)

    def Encode(self, src):
        """s2.Encode(nil, src) (s2/encode.go:29)."""
        return self._encode_any(src)

    def EncodeBetter(self, src):
        """s2.EncodeBetter(nil, src) (s2/encode.go:117): the two-table match finder."""
        return self._encode_any(src, better=True)

    def EncodeSnappyBetter(self, src):
        """s2.EncodeSnappyBetter(nil, src) (s2/encode.go:248)."""
        return self._encode_any(src, snappy=True, better=True)

    def EncodeSnappy(self, src):
        """s2.EncodeSnappy(nil, src) (s2/encode.go:204): output any Snappy decoder accepts."""
        return self._encode_any(src, snappy=True)

    def EncodeBest(self, src):
        """s2.EncodeBest(nil, src) (s2/encode.go:161): the cost-scored match finder, for data written once and read often."""
        return self._encode_any(src, best=True)

    def EncodeSnappyBest(self, src):
        """s2.EncodeSnappyBest(nil, src) (s2/encode.go:292)."""
        return self._encode_any(src, snappy=True, best=True)

    def Decode(self, src, max_len=None):
        """s2.Decode(nil, src) (s2/decode.go:58); max_len defaults to the block's own declared length."""
        if max_len is None:
            max_len = max(_decoded_len(src)[0], 1)
        outs, codes = self.decode_blocks([src], [max_len])
        if codes[0] == -4:
            raise ErrTooLarge("s2: decoded block is too large")
        if codes[0] < 0:
            raise ErrCorrupt("s2: corrupt input")
        return outs[0]

    # ---- LZ4 / LZ4s -> S2 / Snappy blocks (s2.LZ4Converter / s2.LZ4sConverter, s2/lz4convert.go, s2/lz4sconvert.go) ----
    def convert_lz4_blocks(self, blocks, caps, lz4s=False, snappy=False):
        """Convert LZ4 (or LZ4s) blocks; caps[i] = slot capacity.  Returns (outs, codes, ns): outs[i] = uvarint(n) + the S2
        (Snappy) body or None, codes[i] = its size or a negative error, ns[i] = the decoded size."""
        if not blocks:
            return [], [], []
        t = PointerTable(blocks, caps)
        dec = (ctypes.c_int64 * t.n)()
        check(lib.b2c_s2_convert_lz4_chunks(self._ctx, 1 if lz4s else 0, FLAG_SNAPPY if snappy else 0, t.srcs, t.ssz, t.dsts,
                                            t.dcap, t.res, dec, t.n), self._ctx)
        return (*t.results(), [int(x) for x in dec])

    def convert_lz4_device(self, src, src_sizes, src_stride, lz4s=False, snappy=False, dst=None, dst_cap=None, out_sizes=None,
                           decoded=None, src_offsets=None, dst_offsets=None, dst_stride=None):
        """src: uint8 CUDA tensor, block i at i * src_stride (or src_offsets[i]; then every block is at most src_stride bytes).
        Slot i at i * dst_stride (or dst_offsets[i]) with dst_cap bytes.  Returns (dst, out_sizes int64, decoded int64).  Async."""
        assert src.is_cuda and src.dtype == torch.uint8
        n = src_sizes.numel()
        if dst_cap is None:
            dst_cap = src_stride + src_stride // 2 + 64
        if dst_stride is None:
            dst_stride = dst_cap
        if dst is None:
            dst = torch.empty((n, dst_stride), dtype=torch.uint8, device=src.device)
        if out_sizes is None:
            out_sizes = torch.empty((n,), dtype=torch.int64, device=src.device)
        if decoded is None:
            decoded = torch.empty((n,), dtype=torch.int64, device=src.device)
        stream = torch.cuda.current_stream(src.device).cuda_stream
        check(lib.b2c_s2_convert_lz4_device(self._ctx, 1 if lz4s else 0, FLAG_SNAPPY if snappy else 0, src.data_ptr(), src_stride,
                                            None if src_offsets is None else src_offsets.data_ptr(), src_sizes.data_ptr(),
                                            dst.data_ptr(), dst_stride, None if dst_offsets is None else dst_offsets.data_ptr(),
                                            dst_cap, out_sizes.data_ptr(), decoded.data_ptr(), n, ctypes.c_void_p(stream)),
              self._ctx)
        return dst, out_sizes, decoded

    # ---- streams: the framing format (s2.Writer.EncodeBuffer / s2.Reader, s2/writer.go:357-470, s2/reader.go:249-420) ----
    def EncodeStream(self, src, better=False, snappy=False, block_size=BLOCK, index=False, best=False):
        """Writer.EncodeBuffer(src) + Close(): a complete S2 (or Snappy) stream -- identifier, one checksummed chunk per
        block.  block_size <= 64 KiB (WriterBlockSize)."""
        level = _level(better, best)
        buf = np.frombuffer(src, dtype=np.uint8) if len(src) else np.zeros(0, dtype=np.uint8)
        cap = int(lib.b2c_s2_stream_bound(len(src), block_size)) + 16
        out = np.empty(cap, dtype=np.uint8)
        n = ctypes.c_size_t(0)
        rc = lib.b2c_s2_encode_stream(self._ctx, level, FLAG_SNAPPY if snappy else 0, buf.ctypes.data, len(src),
                                      block_size, out.ctypes.data, cap, ctypes.byref(n))
        check(rc, self._ctx)
        stream = out[: n.value].tobytes()
        if index:                          # WriterAddIndex(): the seek index as a trailing skippable chunk (s2/writer.go, s2/index.go)
            stream += s2_index.IndexStream(stream, est_block=block_size)
        return stream

    def DecodeStreamRange(self, stream, start, length=None, index=None):
        """Content bytes [start, start+length) of an indexed stream, decoding only the chunks that cover them (the
        ReadSeeker use of the index, s2/index_test.go:16-104).  index: separately stored index bytes; default: the one
        appended to the stream."""
        return s2_index.read_range(stream, start, length, self.DecodeStream, index)

    def encode_stream_device(self, src, better=False, snappy=False, block_size=BLOCK, dst=None, best=False):
        """src: uint8 CUDA tensor.  Returns (dst uint8 CUDA tensor, total uint64 CUDA tensor [1], err int32 CUDA tensor [1]).  Async."""
        assert src.is_cuda and src.dtype == torch.uint8
        level = _level(better, best)
        n = src.numel()
        if dst is None:
            dst = torch.empty(int(lib.b2c_s2_stream_bound(n, block_size)) + 16, dtype=torch.uint8, device=src.device)
        total = torch.zeros(1, dtype=torch.uint64, device=src.device)
        err = torch.zeros(1, dtype=torch.int32, device=src.device)
        stream = torch.cuda.current_stream(src.device).cuda_stream
        rc = lib.b2c_s2_encode_stream_device(self._ctx, level, FLAG_SNAPPY if snappy else 0, src.data_ptr(), n,
                                             block_size, dst.data_ptr(), dst.numel(), total.data_ptr(), err.data_ptr(),
                                             ctypes.c_void_p(stream))
        check(rc, self._ctx)
        return dst, total, err

    def DecodeStream(self, stream, max_size=None):
        """io.ReadAll(s2.NewReader(stream)): the stream's content; raises the reader's errors (ErrCorrupt, ErrCRC, ...)."""
        buf = np.frombuffer(stream, dtype=np.uint8) if len(stream) else np.zeros(0, dtype=np.uint8)
        cap = max_size if max_size is not None else max(64, 64 * len(stream))
        out = np.empty(cap, dtype=np.uint8)
        n = ctypes.c_size_t(0)
        rc = lib.b2c_s2_decode_stream(self._ctx, buf.ctypes.data, len(stream), out.ctypes.data, cap, ctypes.byref(n))
        if rc == -5:
            raise ErrCorrupt("s2: corrupt input")
        if rc == -9:
            raise ErrCRC("s2: corrupt input, crc mismatch")
        if rc == -11:
            raise ErrUnsupported("s2: unsupported input")
        check(rc, self._ctx)
        return out[: n.value].tobytes()


# ---- stream writer / reader over io objects (s2.NewWriter / s2.NewReader) --------------------------------------------------
MAGIC_S2 = b"\xff\x06\x00\x00S2sTwO"
MAGIC_SNAPPY = b"\xff\x06\x00\x00sNaPpY"
_CHUNK_PADDING = 0xFE


def calcSkippableFrame(written, want_multiple):
    """s2/writer.go:854-874: bytes to add (0, or >= the 4-byte chunk header) to reach a multiple."""
    if want_multiple <= 0 or written < 0:
        raise ValueError("calcSkippableFrame: bad arguments")
    left = written % want_multiple
    if left == 0:
        return 0
    add = want_multiple - left
    while add < 4:
        add += want_multiple
    return add


def skippableFrame(total, fill=None):
    """A padding chunk (type 0xfe) of `total` bytes in all (s2/writer.go:876-898); content from fill(n), default os.urandom."""
    if total == 0:
        return b""
    if total < 4:
        raise ValueError("s2: requested skippable frame (%d) < 4" % total)
    if total >= (4 << 20) + 4:
        raise ValueError("s2: requested skippable frame (%d) >= max 1<<24" % total)
    import os
    return bytes([_CHUNK_PADDING]) + (total - 4).to_bytes(3, "little") + (fill or os.urandom)(total - 4)


def _walk_chunks(buf, pos, end):
    """Yield (type, start, length incl. header, decoded length or None) for the complete chunks of buf[pos:end]."""
    while end - pos >= 4:
        typ = buf[pos]
        ln = buf[pos + 1] | buf[pos + 2] << 8 | buf[pos + 3] << 16
        if pos + 4 + ln > end:
            return
        d = None
        if typ == 0x00 and ln >= 5:
            d = _decoded_len(bytes(buf[pos + 8:pos + 4 + min(ln, 14)]))[0]
        elif typ == 0x01 and ln >= 4:
            d = ln - 4
        yield typ, pos, 4 + ln, d
        pos += 4 + ln


class Writer:
    """s2.Writer (NewWriter / Write / EncodeBuffer / ReadFrom / Flush / Close / CloseIndex / Reset, s2/writer.go:34-852) over
    the device stream encoder: input is gathered and leaves in batches of `batch_bytes` (a multiple of the block size) through
    ONE EncodeStream call each -- all blocks of the batch in parallel -- with the stream identifier kept on the first batch
    only.  add_index = WriterAddIndex, padding = WriterPadding (the padding chunk comes before the index so that the index
    stays at the end), better / best / snappy / block_size = WriterBetterCompression / WriterBestCompression /
    WriterSnappyCompat / WriterBlockSize."""

    def __init__(self, w, codec=None, device=0, block_size=BLOCK, better=False, snappy=False, add_index=False, padding=0,
                 batch_bytes=8 << 20, rand=None, flush_on_write=False, best=False):
        _level(better, best)
        if not 4096 <= block_size <= BLOCK:
            raise ErrUnsupported("s2: block size on the device path: 4 KiB .. 64 KiB")
        self._codec = codec if codec is not None else Codec(device=device)
        self._own = codec is None
        self._bs, self._better, self._snappy, self._best = block_size, better, snappy, best
        self._add_index, self._pad, self._rand = add_index, padding, rand
        self._flush_on_write = flush_on_write               # WriterFlushOnWrite: nothing stays buffered after Write
        self._batch = max(block_size, batch_bytes // block_size * block_size)
        self.Reset(w)

    def Reset(self, w):
        self._w = w
        self._buf = bytearray()
        self._wrote_header = False
        self.written = 0                 # compressed bytes handed to w
        self.uncomp_written = 0
        self._index = s2_index.Index()
        self._index.reset(self._bs)
        self._closed = False

    def _out(self, b):
        self._w.write(b)
        self.written += len(b)

    def _emit(self, data):
        # A Writer takes any codec with EncodeStream(data, better=, snappy=, block_size=); `best` is passed only when
        # that level is asked for, so a codec that knows the first two levels (such as a host model of the format)
        # still serves them.
        extra = {"best": True} if self._best else {}
        piece = self._codec.EncodeStream(bytes(data), better=self._better, snappy=self._snappy, block_size=self._bs, **extra)
        body = piece[10:]
        if not self._wrote_header:
            self._out(piece[:10])
            self._wrote_header = True
        base, u = self.written, self.uncomp_written
        for typ, start, ln, d in _walk_chunks(body, 0, len(body)):
            if d is not None:
                self._index.add(base + start, u)
                u += d
        if u - self.uncomp_written != len(data):
            raise ErrCorrupt("s2: stream encoder returned %d bytes of content for %d" % (u - self.uncomp_written, len(data)))
        self._out(body)
        self.uncomp_written = u

    def Write(self, p):
        if self._closed:
            raise B2CError("s2: Writer is closed")
        self._buf += p
        while len(self._buf) >= self._batch:
            self._emit(self._buf[:self._batch])
            del self._buf[:self._batch]
        if self._flush_on_write:
            self.Flush()
        return len(p)

    def EncodeBuffer(self, buf):
        """Encode a whole buffer (after whatever is pending): s2/writer.go:357-470."""
        self.Flush()
        view = memoryview(bytes(buf))
        for o in range(0, len(view), self._batch):
            self._emit(view[o:o + self._batch])

    def ReadFrom(self, r):
        """Encode everything r yields until EOF; returns the byte count (s2/writer.go:220-300)."""
        n = 0
        while True:
            chunk = r.read(self._batch)
            if not chunk:
                break
            n += len(chunk)
            self.Write(chunk)
        return n

    def Flush(self):
        if self._buf:
            self._emit(self._buf)
            self._buf = bytearray()

    def _close(self, want_index):
        if self._closed:
            raise B2CError("s2: Writer is closed")
        self.Flush()
        index = b""
        if want_index or self._add_index:
            if not self._wrote_header:                         # an index needs a stream to sit in
                self._out(MAGIC_SNAPPY if self._snappy else MAGIC_S2)
                self._wrote_header = True
            comp = self.written if self._pad <= 1 else -1
            index = self._index.appendTo(b"", self.uncomp_written, comp)
            if self._add_index:
                self.written += len(index)                     # counted for the padding; written last
        if self._pad > 1 and self._wrote_header:
            self._w.write(skippableFrame(calcSkippableFrame(self.written, self._pad), self._rand))
        if index and self._add_index:
            self._w.write(index)
        self._closed = True
        if self._own:
            self._codec.close()
        return index

    def Close(self):
        self._close(False)

    def CloseIndex(self):
        """Close and return the index for separate storage (s2/writer.go:787-796)."""
        return self._close(True)


class Reader:
    """s2.Reader (NewReader / Read / Skip / DecodeConcurrent / Reset, s2/reader.go:31-672) over the device stream decoder: the
    4-byte chunk headers are walked on the host to cut the input at chunk boundaries, complete chunks are gathered up to
    `batch_bytes` and decoded by ONE DecodeStream call (all blocks of the batch in parallel, checksums verified on the device).
    Skip drops whole chunks without decoding them where it can (as the reference does); what was decoded before a damaged chunk is
    delivered before the error."""

    def __init__(self, r, codec=None, device=0, batch_bytes=8 << 20, read_size=1 << 20, ignore_stream_identifier=False):
        self._codec = codec if codec is not None else Codec(device=device)
        self._own = codec is None
        self._batch, self._rs, self._ignore_id = batch_bytes, read_size, ignore_stream_identifier
        self.Reset(r)

    def Reset(self, r):
        self._r = r
        self._in = bytearray()
        self._out = bytearray()
        self._eof = False
        self._err = None
        self._seen_id = self._ignore_id
        self._magic = MAGIC_S2
        self._skip = 0
        self._pos = 0                      # content offset of the next byte read() returns
        self._index = None

    def _decode(self, pieces):
        """pieces: list of chunk byte strings.  Decode as one batch; on an error find the chunk it belongs to, keeping the
        output of the chunks before it."""
        try:
            return self._codec.DecodeStream(self._magic + b"".join(pieces)), None
        except (ErrCorrupt, ErrCRC, ErrUnsupported) as e:
            if len(pieces) == 1:
                return b"", e
        out = bytearray()
        for p in pieces:
            try:
                out += self._codec.DecodeStream(self._magic + p)
            except (ErrCorrupt, ErrCRC, ErrUnsupported) as e:
                return bytes(out), e
        return bytes(out), ErrCorrupt("s2: corrupt input")

    def _fill(self):
        if self._err:
            raise self._err
        pieces, pos, flushed = [], 0, bytearray()
        while True:
            got = None
            try:
                for got in _walk_chunks(self._in, pos, len(self._in)):
                    break
            except ErrCorrupt as e:                            # a block length that is not a valid uvarint
                self._err = e
                break
            if got is None:
                if self._eof:
                    if pos < len(self._in):
                        self._err = ErrCorrupt("s2: corrupt input (unexpected EOF)")
                    break
                if pieces and len(self._in) >= self._batch:
                    break
                chunk = self._r.read(self._rs)
                if chunk:
                    self._in += chunk
                else:
                    self._eof = True
                continue
            typ, start, ln, d = got
            if not self._seen_id:
                if typ != 0xFF:
                    self._err = ErrCorrupt("s2: corrupt input")
                    break
                self._seen_id = True
            piece = bytes(self._in[start:start + ln])
            pos = start + ln
            if typ == 0xFF:
                if pieces:                                     # a new stream: decode what precedes under the old identifier
                    pos = start
                    break
                if piece == MAGIC_SNAPPY:
                    self._magic = MAGIC_SNAPPY
                elif piece == MAGIC_S2:
                    self._magic = MAGIC_S2
                else:
                    self._err = ErrCorrupt("s2: corrupt input")
                    break
                continue
            if d is not None and self._skip >= d > 0 and typ in (0, 1):
                self._skip -= d                                # Skip: the whole block is not wanted, do not decode it
                continue
            if typ >= 0x80:
                continue                                       # padding, index and other skippable chunks
            pieces.append(piece)
            if pos >= self._batch:
                break
        if pieces:
            out, err = self._decode(pieces)
            if self._skip:
                k = min(self._skip, len(out))
                out = out[k:]
                self._skip -= k
            self._out += out
            if err is not None:
                self._err = err                                # (comes before any later structural error)
        del self._in[:pos]
        if self._err:
            if self._out:
                return True
            raise self._err
        return bool(pieces) or pos > 0 or not self._eof

    def read(self, size=-1):
        while size < 0 or len(self._out) < size:
            if self._err and self._out:
                break
            if not self._fill():
                break
        if size < 0 or size >= len(self._out):
            out = bytes(self._out)
            self._out.clear()
        else:
            out = bytes(self._out[:size])
            del self._out[:size]
        self._pos += len(out)
        return out

    Read = read

    def Skip(self, n):
        """Skip n bytes of content forward (s2/reader.go:674-800)."""
        if n < 0:
            raise ValueError("attempted negative skip")
        self._pos += n
        k = min(n, len(self._out))
        del self._out[:k]
        n -= k
        self._skip += n
        while self._skip:
            if not self._fill():
                raise ErrCorrupt("s2: corrupt input (unexpected EOF)")     # io.ErrUnexpectedEOF: skipped past the end
            if self._skip == 0:
                break
            if self._out:                      # (cannot happen: _fill consumes the skip first)
                break

    def DecodeConcurrent(self, w, concurrent=0):
        """Decode all that remains into w; returns the byte count (s2/reader.go:413-672; the concurrency is the device's)."""
        total = 0
        while True:
            if self._out:
                total += len(self._out)
                w.write(bytes(self._out))
                self._out.clear()
            if not self._fill():
                break
        if self._out:
            total += len(self._out)
            w.write(bytes(self._out))
            self._out.clear()
        return total

    def ReadSeeker(self, random=False, index=None):
        """-> ReadSeeker over this reader (s2/reader.go:855-920).  index: serialised index bytes; without one it is loaded from
        the end of a seekable input.  random=True needs a seekable input and an index; otherwise seeking is forward only."""
        if index:
            self._index = s2_index.Index()
            try:
                self._index.Load(index)
            except (ValueError, EOFError) as e:
                raise ErrCantSeek("loading index returned: %s" % e)
        seekable = hasattr(self._r, "seek") and (not hasattr(self._r, "seekable") or self._r.seekable())
        if not seekable:
            if random:
                raise ErrCantSeek("input stream isn't seekable")
            return ReadSeeker(self)
        if self._index is None:
            pos = self._r.tell()
            idx = s2_index.Index()
            try:
                idx.LoadStream(self._r)
                self._index = idx
            except s2_index.ErrUnsupported:
                if random:
                    raise ErrCantSeek("input stream does not contain an index")
            except (ValueError, EOFError) as e:
                raise ErrCantSeek("reading index returned: %s" % e)
            finally:
                self._r.seek(pos)
        return ReadSeeker(self)

    def Close(self):
        if self._own and self._codec is not None:
            self._codec.close()
        self._codec = None


class ErrCantSeek(B2CError):
    """s2.ErrCantSeek"""


class ReadSeeker:
    """s2.ReadSeeker (s2/reader.go:845-1060): Seek / ReadAt on the content of a stream.  With an index and a seekable input a
    seek goes to the chunk Index.Find names and skips forward inside it (whole blocks on the way are dropped undecoded);
    without them only forward seeks work, by skipping."""

    def __init__(self, reader):
        self.Reader = reader

    def read(self, size=-1):
        return self.Reader.read(size)

    Read = read

    def Seek(self, offset, whence=0):
        r = self.Reader
        if whence == 0:
            target = offset
        elif whence == 1:
            target = r._pos + offset
        elif whence == 2:
            if r._index is None:
                raise ErrUnsupported("s2: unsupported input")
            target = r._index.TotalUncompressed + offset
        else:
            raise ErrUnsupported("s2: unsupported input")
        if target < 0:
            raise ValueError("seek before start of file")
        if isinstance(r._err, (ErrCorrupt, ErrCRC, ErrUnsupported)):
            raise r._err
        buffered = len(r._out)
        if r._pos <= target <= r._pos + buffered and not r._skip:
            r.Skip(target - r._pos)                           # inside what is already decoded
            return target
        seekable = hasattr(r._r, "seek") and (not hasattr(r._r, "seekable") or r._r.seekable())
        if r._index is None or not seekable:
            if target >= r._pos:
                r.Skip(target - r._pos)
                return target
            raise ErrUnsupported("s2: unsupported input")
        try:
            c, u = r._index.Find(target)
        except EOFError:
            raise ErrCorrupt("s2: corrupt input (unexpected EOF)")
        magic, seen, idx = r._magic, r._seen_id, r._index
        r._r.seek(c)
        r.Reset(r._r)                                          # drop everything buffered; the next chunk read starts at c
        r._index = idx
        r._magic, r._seen_id = magic, True if c else seen      # (mid-stream there is no identifier in front)
        r._pos = u
        if target > u:
            r.Skip(target - u)
        return target

    def ReadAt(self, n, offset):
        """n bytes of content at `offset` (fewer only at the end of the stream)."""
        self.Seek(offset, 0)
        out = bytearray()
        while len(out) < n:
            part = self.Reader.read(n - len(out))
            if not part:
                break
            out += part
        return bytes(out)


# ---- LZ4 / LZ4s converters (s2/lz4convert.go:13-275, s2/lz4sconvert.go:23-284) ---------------------------------------------
class LZ4Converter:
    """s2.LZ4Converter on the device.  ConvertBlock(dst, src, cap) appends the S2 form of the LZ4 block src to dst, where cap is
    the Go slice's capacity (cap(dst) >= len(dst)); returns (dst + body, decoded size) or raises ErrCorrupt / ErrDstTooSmall
    as the reference does (ErrTooLarge for a decoded size above 2^32 - 1).  ConvertBlockSnappy writes Snappy instead."""
    _lz4s = False

    def __init__(self, codec=None, device=0):
        self._codec = codec if codec is not None else Codec(device=device)

    def _convert(self, dst, src, cap, snappy):
        dst = bytes(dst)
        if cap is None:
            cap = len(dst)
        if cap < len(dst):
            raise ValueError("cap below len(dst)")
        if len(src) == 0:
            return dst, 0
        outs, codes, ns = self._codec.convert_lz4_blocks([src], [cap - len(dst) + 5], lz4s=self._lz4s, snappy=snappy)
        if codes[0] == -5:
            raise ErrCorrupt("s2: corrupt input")
        if codes[0] == -4:
            raise ErrDstTooSmall("s2: destination too small")
        if codes[0] == -3:
            raise ErrTooLarge("s2: decoded block is too large")
        if codes[0] < 0:
            raise B2CError(lib.b2c_strerror(codes[0]).decode())
        return dst + outs[0][_decoded_len(outs[0])[1]:], ns[0]

    def ConvertBlock(self, dst, src, cap=None):
        return self._convert(dst, src, cap, False)

    def ConvertBlockSnappy(self, dst, src, cap=None):
        return self._convert(dst, src, cap, True)


class LZ4sConverter(LZ4Converter):
    """s2.LZ4sConverter: the same for LZ4s blocks (Intel QAT's LZ4 variant, where a match length of 3 means no match)."""
    _lz4s = True
