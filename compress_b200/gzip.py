"""gzip.NewReader on the device (gzip/gunzip.go): the members are decoded in one device call, on one GPU lane (a single
input is serial; see flate.Decoder for batches).  The first member's Header is parsed on the host."""
import io
import struct
from dataclasses import dataclass

from . import flate
from .flate import ErrUnexpectedEOF  # noqa: F401


class ErrHeader(Exception):
    """gzip.ErrHeader"""


class ErrChecksum(Exception):
    """gzip.ErrChecksum"""


@dataclass
class Header:
    """gzip.Header of the first member (ModTime in Unix seconds; strings decoded as ISO 8859-1)."""
    Name: str = ""
    Comment: str = ""
    Extra: bytes = None
    ModTime: int = 0
    OS: int = 255


def _header(data):
    try:
        return _parse_header(data)
    except (ValueError, struct.error):
        return Header()


def _parse_header(data):
    if len(data) < 10 or data[:3] != b"\x1f\x8b\x08":
        return Header()
    flg = data[3]
    h = Header(ModTime=struct.unpack_from("<I", data, 4)[0], OS=data[9])
    p = 10
    if flg & 4:
        n = struct.unpack_from("<H", data, p)[0]
        h.Extra = bytes(data[p + 2:p + 2 + n])
        p += 2 + n
    for bit, field in ((8, "Name"), (16, "Comment")):
        if flg & bit:
            e = data.index(0, p)
            setattr(h, field, bytes(data[p:e]).decode("latin-1"))
            p = e + 1
    return h


class Reader:
    """gzip.Reader over a whole input: Multistream(True) by default.  The content is decoded at the first read (or by
    decode()); every error, a bad first header included, is raised then.  Header is the first member's, read on the host
    (left empty when that header is invalid)."""

    def __init__(self, r):
        self._data = bytes(r if isinstance(r, (bytes, bytearray, memoryview)) else r.read())
        self._multi = True
        self._buf = None
        self.Header = Header()
        if len(self._data) == 0:
            raise ErrUnexpectedEOF("EOF")   # gzip.NewReader returns io.EOF for an empty input
        self.Header = _header(self._data)

    def Multistream(self, ok):
        self._multi = bool(ok)

    def decode(self):
        if self._buf is None:
            self._buf = io.BytesIO(flate._decoder().decode_all(self._data, flate.GZIP, self._multi))
        return self._buf.getvalue()

    def read(self, n=-1):
        self.decode()
        return self._buf.read(n)

    Read = read

    def close(self):
        pass

    Close = close


def NewReader(r):
    """gzip.NewReader: a Reader over r (bytes-like or a binary file)."""
    return Reader(r)
