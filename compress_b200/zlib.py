"""zlib.NewReader on the device (zlib/reader.go): the whole zlib stream is decoded in one device call, on one GPU lane
(a single stream is serial; see flate.Decoder for batches)."""
import io

from . import flate
from .flate import ErrUnexpectedEOF  # noqa: F401


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
