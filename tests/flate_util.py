"""Inflate test helpers: the oracle (oracle/liboracle_flate.so, built on demand), a seeded pool of zlib / gzip / raw streams
written by Python's zlib, and stream mutations."""
import ctypes
import os
import random
import struct
import subprocess
import zlib

import helpers as H

ORACLE_FLATE_SO = os.path.join(H.ORACLE_DIR, "liboracle_flate.so")
RAW, ZLIB, GZIP = 0, 1, 2
_L = None


def oracle():
    global _L
    if _L is None:
        if not os.path.exists(ORACLE_FLATE_SO):
            subprocess.run(["make", "-s", "-C", H.ORACLE_DIR, "-f", "flate.mk"], check=True)
        L = ctypes.CDLL(ORACLE_FLATE_SO)
        L.orc_flate_decode.restype = ctypes.c_int64
        L.orc_flate_decode.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_char_p, ctypes.c_size_t, ctypes.c_char_p, ctypes.c_size_t]
        _L = L
    return _L


def orc_decode(fmt, data, cap, multistream=True):
    """(code, content): code = content bytes or a negative B2C_ERR_* class."""
    out = ctypes.create_string_buffer(max(cap, 1))
    r = oracle().orc_flate_decode(fmt, 1 if multistream else 0, bytes(data), len(data), out, cap)
    return r, out.raw[:max(r, 0)]


def text(rng, n):
    words = [bytes(rng.choice(b"etaoinshrdlu ") for _ in range(rng.randint(1, 9))) for _ in range(200)]
    return b" ".join(rng.choice(words) for _ in range(n // 4 + 1))[:n]


def deflate(data, fmt, level=6, wbits=15, strategy=0, flush_every=0, flush_mode=zlib.Z_SYNC_FLUSH, memlevel=8):
    w = {RAW: -wbits, ZLIB: wbits, GZIP: 16 + wbits}[fmt]
    c = zlib.compressobj(level, zlib.DEFLATED, w, memlevel, strategy)
    if not flush_every:
        return c.compress(data) + c.flush()
    out = b""
    for i in range(0, len(data), flush_every):
        out += c.compress(data[i:i + flush_every]) + c.flush(flush_mode)
    return out + c.flush()


def gzip_member(data, level=6, name=None, comment=None, extra=None, fhcrc=False, mtime=0, os_byte=3):
    """A gzip member with the given header fields (FHCRC: CRC-32 of the header, low 16 bits)."""
    flg = (2 if fhcrc else 0) | (4 if extra is not None else 0) | (8 if name is not None else 0) | (16 if comment is not None else 0)
    h = b"\x1f\x8b\x08" + bytes([flg]) + struct.pack("<I", mtime) + b"\x00" + bytes([os_byte])
    if extra is not None:
        h += struct.pack("<H", len(extra)) + extra
    if name is not None:
        h += name + b"\x00"
    if comment is not None:
        h += comment + b"\x00"
    if fhcrc:
        h += struct.pack("<H", zlib.crc32(h) & 0xffff)
    return h + deflate(data, RAW, level) + struct.pack("<II", zlib.crc32(data), len(data) & 0xffffffff)


def pool(seed=7, n=160):
    """[(fmt, stream, content, multistream)]: levels 0-9, the five strategies, window bits 9-15, the three containers,
    gzip header fields (FHCRC included), multi-member gzip, empty contents, sync / full flush boundaries."""
    rng = random.Random(seed)
    out = []
    for i in range(n):
        size = rng.choice([0, 1, 7, 100, 1000, 5000, 40000, 100000])
        data = text(rng, size) if rng.random() < 0.7 else bytes(rng.getrandbits(8) for _ in range(size))
        if rng.random() < 0.15:
            data = bytes([rng.randrange(4)]) * size
        fmt = i % 3
        level, wbits, strat = rng.randint(0, 9), rng.randint(9, 15), rng.choice([0, 1, 2, 3, 4])
        flush = rng.choice([0, 0, 0, 997, 4096])
        mode = rng.choice([zlib.Z_SYNC_FLUSH, zlib.Z_FULL_FLUSH])
        if wbits == 8:
            wbits = 9
        s = deflate(data, fmt, level, wbits, strat, flush, mode)
        out.append((fmt, s, data, True))
    for k in range(12):                                  # header fields, several members, Multistream(false)
        parts = [text(rng, rng.choice([0, 50, 3000])) for _ in range(rng.randint(1, 4))]
        s = b"".join(gzip_member(p, rng.randint(0, 9), name=b"f%d.txt" % k if k & 1 else None,
                                 comment=b"c\xe9" if k & 2 else None, extra=b"ab\x00cd" if k & 4 else None, fhcrc=bool(k & 8),
                                 mtime=k * 1000) for p in parts)
        out.append((GZIP, s, b"".join(parts), True))
        out.append((GZIP, s + b"trailing garbage", parts[0], False))
    return out


def pack_bits(fields):
    """LSB-first bit packing of [(value, nbits)]; a Huffman code is given as ("h", code, nbits) and written MSB first."""
    acc, n = 0, 0
    for f in fields:
        if f[0] == "h":
            _, code, nb = f
            for k in range(nb - 1, -1, -1):
                acc |= ((code >> k) & 1) << n
                n += 1
        else:
            acc |= f[0] << n
            n += f[1]
    return acc.to_bytes((n + 7) // 8 + 1, "little")


def invalid_streams():
    """Hand-written invalid streams: [(fmt, bytes, expected code)]."""
    ok = zlib.compress(b"hello world" * 10)
    g = gzip_member(b"hello world" * 10)
    raw = deflate(b"abc" * 100, RAW)
    return [
        (RAW, b"\x07", -5),                                     # BTYPE 3
        (RAW, b"\x01\x05\x00\xfb\xff", -5),                     # stored: NLEN != ~LEN
        (RAW, b"\x01\x05\x00\xfa\xffab", -12),                  # stored: cut short
        (RAW, pack_bits([(1, 1), (2, 2), (30, 5), (0, 9), (0, 8)]), -5),   # HLIT = 30 (TestNlitOutOfRange class)
        (RAW, pack_bits([(1, 1), (2, 2), (0, 5), (31, 5), (0, 4), (0, 8)]), -5),   # HDIST = 31
        (RAW, pack_bits([(1, 1), (1, 2), ("h", 1, 7), (0, 5), (0, 8)]), -5),   # fixed: a match before any output
        (RAW, pack_bits([(1, 1), (1, 2), ("h", 0x61 + 0x30, 8), ("h", 0b11000110, 8), (0, 8)]), -5),   # length symbol 286
        (RAW, pack_bits([(1, 1), (1, 2), ("h", 0x61 + 0x30, 8), ("h", 1, 7), (30 << 0, 0), (0b01111, 5), (0, 8)]), -5),   # distance code 30
        (RAW, raw + b"junk", 300),                              # bytes after the final block are ignored
        (ZLIB, b"\x78\x9d" + ok[2:], -7),                       # FCHECK wrong
        (ZLIB, b"\x78\xbb\x00\x00\x00\x02" + ok[2:], -11),      # FDICT (not the empty dictionary)
        (ZLIB, ok[:-1] + bytes([ok[-1] ^ 1]), -9),              # Adler-32
        (ZLIB, ok + b"tail", 110),
        (GZIP, b"", -12),                                       # empty: NewReader's io.EOF
        (GZIP, g[:5], -12),
        (GZIP, b"\x1f\x8c" + g[2:], -7),                        # ID2
        (GZIP, g[:3] + b"\x20" + g[4:], -7),                    # reserved FLG bit
        (GZIP, g[:-5] + bytes([g[-5] ^ 1]) + g[-4:], -9),       # CRC-32
        (GZIP, g[:-1] + bytes([g[-1] ^ 1]), -9),                # ISIZE
        (GZIP, g + g[:5], -12),                                 # 5 bytes after a member
        (GZIP, g + b"x" * 12, -7),                              # not a header after a member
        (GZIP, g + b"x" * 12, 110, False),                      # ... ignored with Multistream(false)
    ]


STALE_BODY = [(1, 1), (2, 2), (0, 5), (0, 5), (0, 4), (0, 12), ("h", 0, 7), (127, 7), ("h", 0, 7), (109, 7), ("h", 0x72, 8),
              ("h", 0, 7)]   # a final dynamic block whose code-length code is empty


def stale_streams():
    """Streams whose outcome depends on which table an empty code leaves in place: [(fmt, bytes, expected code or None)]
    (None: an error, the class the oracle gives)."""
    fixed_then = pack_bits([(0, 1), (1, 2), ("h", 0x71, 8), ("h", 0, 7)] + STALE_BODY)   # fixed block "A", then the above
    c = zlib.compressobj(6, zlib.DEFLATED, -15)
    dyn = c.compress(text(random.Random(2), 3000)) + c.flush(zlib.Z_FULL_FLUSH)         # non-final dynamic block, aligned
    after_dyn = dyn + pack_bits(STALE_BODY)
    return [(RAW, fixed_then, -5),
            (GZIP, gzip_member(b"")[:10] + fixed_then + struct.pack("<II", zlib.crc32(b"AB"), 2), -5),
            (RAW, after_dyn, None), (RAW, dyn + pack_bits([(0, 1), (1, 2), ("h", 0x71, 8), ("h", 0, 7)] + STALE_BODY), None)]


def fixture_streams():
    """The reference's fixtures (tests/golden/make_flate_fixtures.py): [(table, fmt, stream, want)] -- want is the content
    (bytes), a B2C_ERR_* code, or None for "an error" (the reference's test checks only that it fails)."""
    import json
    import zipfile
    errs = {"io.ErrUnexpectedEOF": -12, "ErrChecksum": -9, "ErrHeader": -7, "io.EOF": -12}
    out = []
    for r in json.load(open(os.path.join(H.GOLDEN, "flate_tables.json"))):
        w = r["want"]
        want = None if w == "fail" else (errs[w] if w in errs else bytes.fromhex(w))
        out.append((r["table"] + ": " + r["desc"], r["format"], bytes.fromhex(r["stream"]), want))
    with zipfile.ZipFile(os.path.join(H.GOLDEN, "flate_testdata.zip")) as z:
        names = z.namelist()
        for n in names:
            if n.startswith("flate/") and not n.endswith(".in"):
                base = n[len("flate/"):].split(".")[0]
                src = "flate/" + base + ".in"
                if src in names:
                    # the huffman bit writer's blocks (huffman_bit_writer_test.go) carry no final block: a reader that
                    # reads one to the end stops with io.ErrUnexpectedEOF
                    out.append((n, RAW, z.read(n), -12))
        out.append(("gzip/issue6550.gz", GZIP, z.read("gzip/issue6550.gz"), None))
        j = z.read("gzip/test.json")
        out.append(("gzip/test.json", GZIP, gzip_member(j, 9), j))
        for n in names:
            if n.startswith("regress/"):
                d = z.read(n)
                for fmt, lv in ((RAW, 1), (ZLIB, 6), (GZIP, 9)):
                    out.append((n, fmt, deflate(d, fmt, lv), d))
    return out


def mutate(rng, s):
    b = bytearray(s)
    k = rng.randrange(4)
    if k == 0 and b:
        b[rng.randrange(len(b))] ^= 1 << rng.randrange(8)
    elif k == 1 and b:
        i = rng.randrange(len(b))
        b[i] = rng.randrange(256)
    elif k == 2 and len(b) > 1:
        del b[rng.randrange(len(b)):]
    else:
        i = rng.randrange(len(b) + 1)
        b[i:i] = bytes(rng.getrandbits(8) for _ in range(rng.randint(1, 4)))
    return bytes(b)
