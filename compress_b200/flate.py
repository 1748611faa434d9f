"""Inflate on the device: raw DEFLATE, zlib and gzip streams in batches (the reader side of the reference's flate, zlib and
gzip packages: flate/inflate.go, zlib/reader.go, gzip/gunzip.go).

Decoder.decode_chunks / decode_device decode a batch of whole streams in one call, one lane per stream; results are the
content's bytes or the reference's error class (B2C_ERR_* codes, see include/b2c.h).  NewReader and the readers of the gzip
and zlib modules are thin layers over one such call for a single input: a single stream is serial, so one long stream
decodes at the speed of one GPU lane -- batches of many streams are what the device is for.
"""
import ctypes
import io

import numpy as np
import torch

from ._lib import lib, check, B2CError

RAW, ZLIB, GZIP = 0, 1, 2                    # B2C_FLATE_RAW / _ZLIB / _GZIP
GZIP_SINGLE = 1                              # B2C_GZIP_SINGLE: gzip.Reader.Multistream(false)
ERR_DST_SMALL, ERR_CORRUPT, ERR_MAGIC, ERR_CRC, ERR_UNSUPPORTED, ERR_UNEXPECTED_EOF = -4, -5, -7, -9, -11, -12
MAX_CAP = (1 << 32) - 1                      # contents are under 4 GiB


class CorruptInputError(Exception):
    """flate.CorruptInputError: the DEFLATE data is invalid (the device does not report the offset)."""


class ErrUnexpectedEOF(EOFError):
    """io.ErrUnexpectedEOF: the input ends inside a stream, a header or a trailer."""


class Decoder:
    """Batches of raw DEFLATE / zlib / gzip streams decoded on one GPU."""

    def __init__(self, device=0):
        if lib.b2c_device_count() <= 0:
            raise B2CError("no CUDA device")
        self._ctx = lib.b2c_ctx_create(device, 0)
        if not self._ctx:
            raise B2CError("b2c_ctx_create failed")

    def close(self):
        if self._ctx:
            lib.b2c_ctx_destroy(self._ctx)
            self._ctx = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

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
        n = len(inputs)
        if n == 0:
            return [], []
        bufs = [np.frombuffer(bytes(b), dtype=np.uint8) if len(b) else np.zeros(1, dtype=np.uint8) for b in inputs]
        outs = [np.empty(max(int(c), 1), dtype=np.uint8) for c in caps]
        srcs = (ctypes.c_void_p * n)(*[b.ctypes.data for b in bufs])
        ssz = (ctypes.c_size_t * n)(*[len(b) for b in inputs])
        dsts = (ctypes.c_void_p * n)(*[o.ctypes.data for o in outs])
        dcap = (ctypes.c_size_t * n)(*[int(c) for c in caps])
        res = (ctypes.c_int64 * n)()
        check(lib.b2c_flate_decode_chunks(self._ctx, format, 0 if multistream else GZIP_SINGLE, srcs, ssz, dsts, dcap, res, n),
              self._ctx)
        codes = [int(r) for r in res]
        return [outs[i][:codes[i]].tobytes() if codes[i] >= 0 else None for i in range(n)], codes

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
