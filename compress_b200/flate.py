"""Inflate on the device: raw DEFLATE, zlib and gzip streams in batches (the reader side of the reference's flate, zlib and
gzip packages: flate/inflate.go, zlib/reader.go, gzip/gunzip.go).

Encoder.encode_chunks / encode_device write flate.StatelessDeflate output (flate/stateless.go) for a batch of inputs, raw
or as gzip members, byte-identical to the reference: every block of every input is parsed at once on the device.
StatelessDeflate and NewStatelessWriter are thin layers over one such call.

Encoder.best_speed_chunks / best_speed_device write what flate.NewWriter(w, BestSpeed) -- or zlib / gzip
.NewWriterLevel(w, BestSpeed) -- writes for Writes then Close, byte-identical to the reference: one lane per input parses
and writes its windows in order.  NewWriter(w, BestSpeed) buffers its Writes and makes one such call at Close.

Encoder.nolz_chunks / nolz_device write what the reference's writers write at HuffmanOnly (-2) and NoCompression (0):
neither level has a match finder, so every window of every input is analysed and written in parallel, and a single
large member is the whole device's work.  These methods are the way to raw and zlib streams at these levels: NewWriter
here and zlib.NewWriterLevel keep raising ValueError for them.  gzip.NewWriterLevel(w, HuffmanOnly | NoCompression)
buffers its Writes and makes one such call at Close.

Decoder.decode_chunks / decode_device decode a batch of whole streams in one call, one lane per stream; results are the
content's bytes or the reference's error class (B2C_ERR_* codes, see include/b2c.h).  NewReader and the readers of the gzip
and zlib modules are thin layers over one such call for a single input: a single stream is serial, so one long stream
decodes at the speed of one GPU lane -- batches of many streams are what the device is for.
"""
import ctypes
import io

import torch

from ._lib import lib, check, B2CError, Context, PointerTable

RAW, ZLIB, GZIP = 0, 1, 2                    # B2C_FLATE_RAW / _ZLIB / _GZIP
GZIP_SINGLE = 1                              # B2C_GZIP_SINGLE: gzip.Reader.Multistream(false)
ERR_DST_SMALL, ERR_CORRUPT, ERR_MAGIC, ERR_CRC, ERR_UNSUPPORTED, ERR_UNEXPECTED_EOF = -4, -5, -7, -9, -11, -12
MAX_CAP = (1 << 32) - 1                      # contents are under 4 GiB


MAX_STATELESS_DICT = 8 << 10                 # only the last 8 KiB of a dict are used
BestSpeed = 1
MAX_BEST_SPEED_INPUT = 1 << 30               # a larger input is B2C_ERR_ARG
NoCompression, HuffmanOnly = 0, -2
ConstantCompression = HuffmanOnly
MAX_NOLZ_INPUT = (1 << 32) - 1               # inputs are under 4 GiB at HuffmanOnly / NoCompression


class CorruptInputError(Exception):
    """flate.CorruptInputError: the DEFLATE data is invalid (the device does not report the offset)."""


class ErrUnexpectedEOF(EOFError):
    """io.ErrUnexpectedEOF: the input ends inside a stream, a header or a trailer."""


class Decoder(Context):
    """Batches of raw DEFLATE / zlib / gzip streams decoded on one GPU."""

    @property
    def launches(self):
        """Kernel launches on this context so far: a decode call launches 3 per pass over its record scratch."""
        return int(lib.b2c_launch_count(self._ctx))

    def decode_device(self, src, src_sizes, src_stride, dst=None, dst_cap=1 << 16, out_sizes=None, format=GZIP,
                      multistream=True, src_offsets=None):
        """Device-resident batch: input i is src_sizes[i] bytes at src + i * src_stride (or src + src_offsets[i], each at
        most src_stride bytes); its content goes to row i of dst ([n, dst_cap] uint8).  Asynchronous on the current stream.
        Returns (dst, out_sizes): out_sizes[i] = content bytes or a negative B2C_ERR_* code."""
        assert src.is_cuda and src.dtype == torch.uint8
        n = src_sizes.numel()
        if dst is None:
            dst = torch.empty((n, dst_cap), dtype=torch.uint8, device=src.device)
        if out_sizes is None:
            out_sizes = torch.empty((n,), dtype=torch.int64, device=src.device)
        stream = torch.cuda.current_stream(src.device).cuda_stream
        flags = 0 if multistream else GZIP_SINGLE
        check(lib.b2c_flate_decode_device(self._ctx, format, flags, src.data_ptr(), src_stride,
                                          None if src_offsets is None else src_offsets.data_ptr(), src_sizes.data_ptr(),
                                          dst.data_ptr(), dst.shape[1] if dst.dim() == 2 else dst_cap, None, dst_cap,
                                          out_sizes.data_ptr(), n, ctypes.c_void_p(stream)), self._ctx)
        return dst, out_sizes

    def decode_chunks(self, inputs, caps, format=GZIP, multistream=True):
        """Host buffers: inputs[i] decoded into at most caps[i] bytes.  Returns (outputs, codes): outputs[i] is the content
        (None on error), codes[i] its length or a negative B2C_ERR_* code."""
        if not inputs:
            return [], []
        t = PointerTable(inputs, caps)
        check(lib.b2c_flate_decode_chunks(self._ctx, format, 0 if multistream else GZIP_SINGLE, t.srcs, t.ssz, t.dsts, t.dcap,
                                          t.res, t.n), self._ctx)
        return t.results()

    def decode_all(self, data, format, multistream=True):
        """One input of unknown content size: the destination starts at 4x the input (at least 64 KiB) and doubles while it
        is too small.  Returns the content or raises the reference's error."""
        cap = min(max(4 * len(data), 1 << 16), MAX_CAP)
        while True:
            outs, codes = self.decode_chunks([data], [cap], format, multistream)
            if codes[0] != ERR_DST_SMALL or cap == MAX_CAP:
                break
            cap = min(2 * cap, MAX_CAP)
        return outs[0] if codes[0] >= 0 else raise_for(codes[0], format)


def raise_for(code, format):
    """Raises the reference's error for a negative result code of the given format."""
    if code == ERR_CORRUPT:
        raise CorruptInputError("flate: corrupt input")
    if code == ERR_UNEXPECTED_EOF:
        raise ErrUnexpectedEOF("unexpected EOF")
    if format == GZIP:
        from . import gzip as _g
        if code == ERR_MAGIC:
            raise _g.ErrHeader("gzip: invalid header")
        if code == ERR_CRC:
            raise _g.ErrChecksum("gzip: invalid checksum")
    if format == ZLIB:
        from . import zlib as _z
        if code == ERR_MAGIC:
            raise _z.ErrHeader("zlib: invalid header")
        if code == ERR_CRC:
            raise _z.ErrChecksum("zlib: invalid checksum")
        if code == ERR_UNSUPPORTED:
            raise _z.ErrDictionary("zlib: invalid dictionary")
    raise B2CError(f"libb200comp error {code}: {lib.b2c_strerror(code).decode()}")


_dec = None


def _decoder():
    global _dec
    if _dec is None:
        _dec = Decoder()
    return _dec


def NewReader(r):
    """flate.NewReader over a bytes-like object or a binary file: the whole raw DEFLATE stream is decoded in one device call
    (one GPU lane).  Returns an io.BytesIO of the content; errors are raised here."""
    data = r if isinstance(r, (bytes, bytearray, memoryview)) else r.read()
    return io.BytesIO(_decoder().decode_all(bytes(data), RAW))


def StatelessBound(n, dict_len=0):
    """The largest raw StatelessDeflate output of an n-byte input."""
    return int(lib.b2c_flate_stateless_bound(n, dict_len))


class Encoder(Context):
    """Batches of flate.StatelessDeflate calls (raw) or gzip members at StatelessCompression, encoded on one GPU."""

    def encode_device(self, src, src_sizes, src_stride, dst=None, dst_cap=None, out_sizes=None, format=RAW, eof=None,
                      dict=None, dict_offsets=None, dict_sizes=None, header=b"", crc_in=None, crc_out=None,
                      src_offsets=None):
        """Device-resident batch: input i is src_sizes[i] bytes at src + i * src_stride (or src + src_offsets[i]); its
        output goes to row i of dst ([n, dst_cap] uint8).  eof: optional uint8 per input (raw only, default all true);
        dict / dict_offsets / dict_sizes: optional per-input dicts (raw only); header: the gzip member header (format
        GZIP); crc_in / crc_out: optional uint32 (int32 tensors) CRC-32 seeds and results.  Asynchronous on the current
        stream.  Returns (dst, out_sizes): out_sizes[i] = bytes or a negative B2C_ERR_* code."""
        assert src.is_cuda and src.dtype == torch.uint8
        n = src_sizes.numel()
        if dst_cap is None:
            dst_cap = StatelessBound(src_stride, MAX_STATELESS_DICT) + len(header) + 10
        if dst is None:
            dst = torch.empty((n, dst_cap), dtype=torch.uint8, device=src.device)
        if out_sizes is None:
            out_sizes = torch.empty((n,), dtype=torch.int64, device=src.device)
        ptr = lambda t: None if t is None else t.data_ptr()  # noqa: E731
        stream = torch.cuda.current_stream(src.device).cuda_stream
        check(lib.b2c_flate_stateless_device(self._ctx, format, 0, src.data_ptr(), src_stride, ptr(src_offsets),
                                             src_sizes.data_ptr(), ptr(eof), ptr(dict), ptr(dict_offsets), ptr(dict_sizes),
                                             bytes(header), len(header), dst.data_ptr(),
                                             dst.shape[1] if dst.dim() == 2 else dst_cap, None, dst_cap,
                                             out_sizes.data_ptr(), ptr(crc_in), ptr(crc_out), n,
                                             ctypes.c_void_p(stream)), self._ctx)
        return dst, out_sizes

    def encode_chunks(self, inputs, format=RAW, eof=None, dicts=None, header=b"", caps=None, crc_in=None):
        """Host buffers: one StatelessDeflate call (raw) or one gzip member per input.  Returns (outputs, codes, crcs):
        outputs[i] the bytes (None on error), codes[i] their length or a negative B2C_ERR_* code, crcs[i] the CRC-32 of
        input i continued from crc_in[i]."""
        n = len(inputs)
        if n == 0:
            return [], [], []
        if caps is None:
            caps = [StatelessBound(len(b), MAX_STATELESS_DICT) + len(header) + 10 for b in inputs]
        t = PointerTable(inputs, caps)
        eofs = None if eof is None else (ctypes.c_uint8 * n)(*[1 if e else 0 for e in eof])
        dp = dsz = None
        if dicts is not None:
            dl = [d or b"" for d in dicts]
            dp = t.pointers(dl)
            dsz = (ctypes.c_size_t * n)(*[len(d) for d in dl])
        cin = None if crc_in is None else (ctypes.c_uint32 * n)(*crc_in)
        cout = (ctypes.c_uint32 * n)()
        check(lib.b2c_flate_stateless_chunks(self._ctx, format, 0, t.srcs, t.ssz, eofs, dp, dsz, bytes(header), len(header),
                                             t.dsts, t.dcap, t.res, cin, cout, n), self._ctx)
        return (*t.results(), [int(c) for c in cout])


    def best_speed_device(self, src, src_sizes, src_stride, dst=None, dst_cap=None, out_sizes=None, format=RAW, header=b"",
                          check_out=None, src_offsets=None):
        """Device-resident batch at BestSpeed: input i is src_sizes[i] bytes at src + i * src_stride (or src +
        src_offsets[i], each at most src_stride bytes), written as one member of `format` (RAW, ZLIB, or GZIP with this
        member header) into row i of dst ([n, dst_cap] uint8).  check_out: optional int32 tensor for each input's CRC-32
        (RAW, GZIP) or Adler-32 (ZLIB).  Asynchronous on the current stream.  Returns (dst, out_sizes): out_sizes[i] =
        bytes or a negative B2C_ERR_* code."""
        assert src.is_cuda and src.dtype == torch.uint8
        n = src_sizes.numel()
        if dst_cap is None:
            dst_cap = BestSpeedBound(src_stride) + _container_bytes(format, header)
        if dst is None:
            dst = torch.empty((n, dst_cap), dtype=torch.uint8, device=src.device)
        if out_sizes is None:
            out_sizes = torch.empty((n,), dtype=torch.int64, device=src.device)
        stream = torch.cuda.current_stream(src.device).cuda_stream
        check(lib.b2c_flate_best_speed_device(self._ctx, format, 0, src.data_ptr(), src_stride,
                                              None if src_offsets is None else src_offsets.data_ptr(), src_sizes.data_ptr(),
                                              bytes(header), len(header), dst.data_ptr(),
                                              dst.shape[1] if dst.dim() == 2 else dst_cap, None, dst_cap,
                                              out_sizes.data_ptr(), None if check_out is None else check_out.data_ptr(), n,
                                              ctypes.c_void_p(stream)), self._ctx)
        return dst, out_sizes

    def best_speed_chunks(self, inputs, format=RAW, header=b"", caps=None):
        """Host buffers at BestSpeed: one member of `format` per input.  Returns (outputs, codes, checks): outputs[i] the
        bytes (None on error), codes[i] their length or a negative B2C_ERR_* code, checks[i] the CRC-32 (RAW, GZIP) or
        Adler-32 (ZLIB) of input i."""
        n = len(inputs)
        if n == 0:
            return [], [], []
        if caps is None:
            caps = [BestSpeedBound(len(b)) + _container_bytes(format, header) for b in inputs]
        t = PointerTable(inputs, caps)
        chk = (ctypes.c_uint32 * n)()
        check(lib.b2c_flate_best_speed_chunks(self._ctx, format, 0, t.srcs, t.ssz, bytes(header), len(header), t.dsts,
                                              t.dcap, t.res, chk, n), self._ctx)
        return (*t.results(), [int(c) for c in chk])


    def nolz_device(self, level, src, src_sizes, src_stride, dst=None, dst_cap=None, out_sizes=None, format=RAW,
                    header=b"", check_out=None, src_offsets=None):
        """Device-resident batch at `level` (HuffmanOnly or NoCompression): input i is src_sizes[i] bytes at src + i *
        src_stride (or src + src_offsets[i], each at most src_stride bytes), written as one member of `format` (RAW, ZLIB,
        or GZIP with this member header) into row i of dst ([n, dst_cap] uint8).  check_out: optional int32 tensor for
        each input's CRC-32 (RAW, GZIP) or Adler-32 (ZLIB).  Asynchronous on the current stream.  Returns (dst,
        out_sizes): out_sizes[i] = bytes or a negative B2C_ERR_* code."""
        assert src.is_cuda and src.dtype == torch.uint8
        n = src_sizes.numel()
        if dst_cap is None:
            dst_cap = NoLZBound(level, src_stride) + _container_bytes(format, header)
        if dst is None:
            dst = torch.empty((n, dst_cap), dtype=torch.uint8, device=src.device)
        if out_sizes is None:
            out_sizes = torch.empty((n,), dtype=torch.int64, device=src.device)
        stream = torch.cuda.current_stream(src.device).cuda_stream
        check(lib.b2c_flate_nolz_device(self._ctx, level, format, 0, src.data_ptr(), src_stride,
                                        None if src_offsets is None else src_offsets.data_ptr(), src_sizes.data_ptr(),
                                        bytes(header), len(header), dst.data_ptr(),
                                        dst.shape[1] if dst.dim() == 2 else dst_cap, None, dst_cap, out_sizes.data_ptr(),
                                        None if check_out is None else check_out.data_ptr(), n, ctypes.c_void_p(stream)),
              self._ctx)
        return dst, out_sizes

    def nolz_chunks(self, level, inputs, format=RAW, header=b"", caps=None):
        """Host buffers at `level` (HuffmanOnly or NoCompression): one member of `format` per input.  Returns (outputs,
        codes, checks): outputs[i] the bytes (None on error), codes[i] their length or a negative B2C_ERR_* code,
        checks[i] the CRC-32 (RAW, GZIP) or Adler-32 (ZLIB) of input i."""
        n = len(inputs)
        if n == 0:
            return [], [], []
        if caps is None:
            caps = [NoLZBound(level, len(b)) + _container_bytes(format, header) for b in inputs]
        t = PointerTable(inputs, caps)
        chk = (ctypes.c_uint32 * n)()
        check(lib.b2c_flate_nolz_chunks(self._ctx, level, format, 0, t.srcs, t.ssz, bytes(header), len(header), t.dsts,
                                        t.dcap, t.res, chk, n), self._ctx)
        return (*t.results(), [int(c) for c in chk])


def NoLZBound(level, n):
    """The largest raw output of an n-byte input at HuffmanOnly or NoCompression (a zlib stream adds 6 bytes, a gzip
    member its header + 8); 0 for another level."""
    return int(lib.b2c_flate_nolz_bound(level, n))


def BestSpeedBound(n):
    """The largest raw output of an n-byte input at BestSpeed (a zlib stream adds 6 bytes, a gzip member its header + 8)."""
    return int(lib.b2c_flate_best_speed_bound(n))


def _container_bytes(format, header):
    return 6 if format == ZLIB else (len(header) + 8 if format == GZIP else 0)


_enc = None


def _encoder():
    global _enc
    if _enc is None:
        _enc = Encoder()
    return _enc


def StatelessDeflate(out, in_, eof, dict=None):
    """flate.StatelessDeflate: writes the stateless encoding of in_ to out (a binary file-like object), encoded on the
    device in one call.  Only the last 8 KiB of dict are used."""
    outs, codes, _ = _encoder().encode_chunks([bytes(in_)], RAW, eof=[eof], dicts=None if dict is None else [bytes(dict)])
    if codes[0] < 0:
        raise B2CError(f"libb200comp error {codes[0]}: {lib.b2c_strerror(codes[0]).decode()}")
    out.write(outs[0])


class _StatelessWriter:
    """flate.NewStatelessWriter (flate/stateless.go:20-55): every Write is one StatelessDeflate(p, false) call, Close
    writes the final empty block."""

    def __init__(self, dst):
        self._dst, self._closed = dst, False

    def Write(self, p):
        StatelessDeflate(self._dst, p, False)
        return len(p)

    write = Write

    def Close(self):
        if self._closed:
            return
        self._closed = True
        StatelessDeflate(self._dst, b"", True)

    close = Close

    def Reset(self, w):
        self._dst, self._closed = w, False


def NewStatelessWriter(dst):
    return _StatelessWriter(dst)


def best_speed_member(data, format, header=b""):
    """One member of `format` at BestSpeed for the bytes of all Writes, encoded in one device call; raises on error."""
    outs, codes, _ = _encoder().best_speed_chunks([data], format, header)
    if codes[0] < 0:
        raise B2CError(f"libb200comp error {codes[0]}: {lib.b2c_strerror(codes[0]).decode()}")
    return outs[0]


class BufferedWriter:
    """The Write / Close side of a writer at BestSpeed: Writes are buffered and Close encodes them in one device call --
    without Flush the reference's blocks depend on the byte count alone, so the Writes' boundaries do not matter.  Flush
    (a sync flush) is not built.  Subclasses give _member(data)."""

    def __init__(self, w):
        self.Reset(w)

    def Reset(self, w):
        """Discards the buffered bytes; the next Write starts a new member on w."""
        self._w, self._buf, self._closed = w, bytearray(), False

    def Write(self, p):
        if self._closed:
            raise ValueError("write after Close")
        p = bytes(p)
        if len(self._buf) + len(p) > MAX_BEST_SPEED_INPUT:
            raise ValueError("the device encodes at most 1 GiB per member at BestSpeed")
        self._buf += p
        return len(p)

    write = Write

    def Flush(self):
        raise NotImplementedError("Flush (a sync flush) is not built on the device at BestSpeed; Close ends the member")

    def Close(self):
        if self._closed:
            return
        self._closed = True
        self._w.write(self._member(bytes(self._buf)))
        self._buf = bytearray()

    close = Close


class Writer(BufferedWriter):
    """flate.Writer at BestSpeed (flate/deflate.go): a raw DEFLATE stream, encoded on the device at Close."""

    def __init__(self, w, level=BestSpeed):
        if level != BestSpeed:
            raise ValueError("flate: only BestSpeed (1) is built on the device for NewWriter; level %r is not" % (level,))
        super().__init__(w)

    def _member(self, data):
        return best_speed_member(data, RAW)


def nolz_member(data, level, format, header=b""):
    """One member of `format` at HuffmanOnly or NoCompression for the bytes of all Writes, encoded in one device call;
    raises on error."""
    outs, codes, _ = _encoder().nolz_chunks(level, [data], format, header)
    if codes[0] < 0:
        raise B2CError(f"libb200comp error {codes[0]}: {lib.b2c_strerror(codes[0]).decode()}")
    return outs[0]


def NewWriter(w, level):
    """flate.NewWriter; only BestSpeed is built.  Raw streams at HuffmanOnly and NoCompression come from
    Encoder.nolz_chunks / nolz_device (this still raises ValueError for them)."""
    return Writer(w, level)
