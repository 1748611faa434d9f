"""zlib.NewReader on the device (zlib/reader.go): the whole zlib stream is decoded in one device call, on one GPU lane
(a single stream is serial; see flate.Decoder for batches).

zlib.NewWriterLevel(w, BestSpeed) (zlib/writer.go): a Writer that buffers its Writes and encodes the stream in one device
call at Close.  Other levels, and so NewWriter's DefaultCompression, are not built.  zlib streams at HuffmanOnly and
NoCompression come from flate.Encoder.nolz_chunks / nolz_device with format ZLIB; NewWriterLevel raises ValueError for
them."""
import io

from . import flate
from .flate import ErrUnexpectedEOF  # noqa: F401

NoCompression, BestSpeed, BestCompression, DefaultCompression, HuffmanOnly = 0, 1, 9, -1, -2


class ErrHeader(Exception):
    """zlib.ErrHeader"""


class ErrChecksum(Exception):
    """zlib.ErrChecksum"""


class ErrDictionary(Exception):
    """zlib.ErrDictionary: the stream names a preset dictionary (NewReaderDict is not offered)."""


def NewReader(r):
    """Decodes the zlib stream in r (bytes-like or a binary file) and returns an io.BytesIO of its content; the reference's
    errors are raised here."""
    data = r if isinstance(r, (bytes, bytearray, memoryview)) else r.read()
    return io.BytesIO(flate._decoder().decode_all(bytes(data), flate.ZLIB))


class Writer(flate.BufferedWriter):
    """zlib.Writer at BestSpeed: header 78 01, the DEFLATE stream and the Adler-32, written at Close."""

    def __init__(self, w, level=DefaultCompression):
        if level != BestSpeed:
            raise ValueError("zlib: only BestSpeed (1) is built on the device; level %r is not" % (level,))
        super().__init__(w)

    def _member(self, data):
        return flate.best_speed_member(data, flate.ZLIB)


def NewWriter(w):
    """zlib.NewWriter: DefaultCompression, which is not built, so this raises ValueError; use NewWriterLevel(w,
    BestSpeed)."""
    return Writer(w)


def NewWriterLevel(w, level):
    """zlib.NewWriterLevel; only BestSpeed is built (HuffmanOnly and NoCompression: flate.Encoder.nolz_chunks /
    nolz_device)."""
    return Writer(w, level)
