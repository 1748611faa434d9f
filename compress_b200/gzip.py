"""gzip.NewReader on the device (gzip/gunzip.go): the members are decoded in one device call, on one GPU lane (a single
input is serial; see flate.Decoder for batches).  The first member's Header is parsed on the host.

gzip.NewWriterLevel(w, StatelessCompression) (gzip/gzip.go): a Writer whose every Write is one device call of
flate.StatelessDeflate; the CRC-32 is continued on the device.  gzip.NewWriterLevel(w, BestSpeed | HuffmanOnly |
NoCompression): a Writer that buffers its Writes and encodes the member in one device call at Close.  Other levels are not
built."""
import io
import struct
from dataclasses import dataclass

from . import flate
from .flate import ErrUnexpectedEOF  # noqa: F401


StatelessCompression = -3
BestSpeed, BestCompression = 1, 9
NoCompression, HuffmanOnly = 0, -2
ConstantCompression = HuffmanOnly
_BUFFERED = {BestSpeed: (flate.MAX_BEST_SPEED_INPUT, "1 GiB"), HuffmanOnly: (flate.MAX_NOLZ_INPUT, "4 GiB - 1"),
             NoCompression: (flate.MAX_NOLZ_INPUT, "4 GiB - 1")}   # the levels whose member is one call at Close
# time.Time{}.Unix(): the reference writes uint32(ModTime.Unix()) without a zero check, so an unset ModTime is this
ZERO_MODTIME = -62135596800


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


class Writer:
    """gzip.Writer at StatelessCompression, BestSpeed, HuffmanOnly or NoCompression: Name / Comment / Extra / ModTime
    (Unix seconds; unset is Go's zero time) / OS set before the first Write (at the other levels: before Close) go into
    the header.
    StatelessCompression: each Write(p) is StatelessDeflate(p, false), Close writes StatelessDeflate(nil, true), the
    CRC-32 and ISIZE; Flush writes nothing (the stateless writer keeps no pending data).
    BestSpeed, HuffmanOnly, NoCompression: the Writes are buffered and Close writes the whole member (header with XFL 4
    at BestSpeed, else 0, the stream, CRC-32 and ISIZE) from one device call; Flush (a sync flush) is not built and
    raises."""

    def __init__(self, w, level=StatelessCompression):
        if level != StatelessCompression and level not in _BUFFERED:
            raise ValueError("gzip: only StatelessCompression (-3), HuffmanOnly (-2), NoCompression (0) and BestSpeed (1) "
                             "are built on the device; level %r is not" % (level,))
        self._level = level
        self.Reset(w)

    def Reset(self, w):
        """As the reference's Reset (gzip/gzip.go:98-114): the header fields go back to their zero values too."""
        self.Name, self.Comment, self.Extra, self.ModTime, self.OS = "", "", None, ZERO_MODTIME, 255
        self._w, self._wrote, self._closed, self._crc, self._size = w, False, False, 0, 0
        self._buf = bytearray()

    def _header(self):
        flg = (4 if self.Extra is not None else 0) | (8 if self.Name else 0) | (16 if self.Comment else 0)
        xfl = 4 if self._level == BestSpeed else (2 if self._level == BestCompression else 0)   # gzip/gzip.go:193-198
        h = b"\x1f\x8b\x08" + bytes([flg]) + struct.pack("<I", int(self.ModTime) & 0xffffffff) + bytes([xfl, self.OS])
        if self.Extra is not None:
            h += struct.pack("<H", len(self.Extra)) + bytes(self.Extra)
        if self.Name:
            h += self.Name.encode("latin-1") + b"\x00"
        if self.Comment:
            h += self.Comment.encode("latin-1") + b"\x00"
        return h

    def Write(self, p):
        p = bytes(p)
        if self._level in _BUFFERED:
            if self._closed:
                raise ValueError("write after Close")
            limit, text = _BUFFERED[self._level]
            if len(self._buf) + len(p) > limit:
                raise ValueError("the device encodes at most %s per member at level %d" % (text, self._level))
            self._buf += p
            return len(p)
        if not self._wrote:
            self._wrote = True
            self._w.write(self._header())
        outs, codes, crcs = flate._encoder().encode_chunks([p], flate.RAW, eof=[False], crc_in=[self._crc])
        if codes[0] < 0:
            flate.raise_for(codes[0], flate.RAW)
        self._w.write(outs[0])
        self._crc = crcs[0]
        self._size = (self._size + len(p)) & 0xffffffff
        return len(p)

    write = Write

    def Flush(self):
        if self._level in _BUFFERED:
            raise NotImplementedError("Flush (a sync flush) is not built on the device at level %d; Close ends the member"
                                      % self._level)

    def Close(self):
        if self._closed:
            return
        self._closed = True
        if self._level in _BUFFERED:
            data = bytes(self._buf)
            if self._level == BestSpeed:
                self._w.write(flate.best_speed_member(data, flate.GZIP, self._header()))
            else:
                self._w.write(flate.nolz_member(data, self._level, flate.GZIP, self._header()))
            self._buf = bytearray()
            return
        if not self._wrote:
            self.Write(b"")
        self._w.write(b"\x03\x00" + struct.pack("<II", self._crc, self._size))

    close = Close


def NewWriterLevel(w, level):
    """gzip.NewWriterLevel; only StatelessCompression, HuffmanOnly, NoCompression and BestSpeed are built."""
    return Writer(w, level)


def header_bytes(Name="", Comment="", Extra=None, ModTime=ZERO_MODTIME, OS=255, level=StatelessCompression):
    """The member header gzip.Writer writes for these fields at this level (XFL 4 at BestSpeed, else 0), as flate.Encoder
    takes it for format GZIP."""
    w = Writer(io.BytesIO(), level)
    w.Name, w.Comment, w.Extra, w.ModTime, w.OS = Name, Comment, Extra, ModTime, OS
    return w._header()
