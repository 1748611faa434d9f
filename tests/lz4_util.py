"""LZ4 / LZ4s helpers of the converter tests: the oracle's converter and lz4ref restatements (oracle/orc_lz4.c), a token
writer for hand-built blocks, the reference's fuzz seeds and a seeded pool of blocks.  Test infrastructure only."""
import ctypes
import io
import os
import subprocess
import zipfile

import numpy as np

import helpers as H

CORRUPT, DST_SMALL, TOO_BIG = -5, -4, -3


ORACLE_LZ4_SO = os.path.join(H.ORACLE_DIR, "liboracle_lz4.so")
EMU_LZ4_SO = os.path.join(H.EMU_DIR, "libb2c_emu_lz4.so")
_lib = None


def _L():
    """ctypes handle of oracle/liboracle_lz4.so (oracle/lz4.mk; built on demand)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(ORACLE_LZ4_SO):
        subprocess.run(["make", "-s", "-C", H.ORACLE_DIR, "-f", "lz4.mk"], check=True)
    L = ctypes.CDLL(ORACLE_LZ4_SO)
    c = ctypes
    L.orc_lz4_convert.restype = c.c_int64
    L.orc_lz4_convert.argtypes = [c.c_int, c.c_int, c.c_char_p, c.c_int64, c.c_int64, c.c_char_p, c.c_int64, c.POINTER(c.c_int64)]
    L.orc_lz4_compress_block.restype = c.c_int64
    L.orc_lz4_compress_block.argtypes = [c.c_int, c.c_char_p, c.c_int64, c.c_char_p, c.c_int64]
    L.orc_lz4_compress_bound.restype = c.c_int64
    L.orc_lz4_compress_bound.argtypes = [c.c_int64]
    L.orc_lz4_uncompress_block.restype = c.c_int64
    L.orc_lz4_uncompress_block.argtypes = [c.c_char_p, c.c_int64, c.c_char_p, c.c_int64]
    _lib = L
    return L


def emu():
    """ctypes handle of the emulated conversion kernels (tests/emu/lz4.mk; rebuilt when a kernel source changed)."""
    subprocess.run(["make", "-s", "-C", H.EMU_DIR, "-f", "lz4.mk"], check=True)
    E = ctypes.CDLL(EMU_LZ4_SO)
    c = ctypes
    E.emu_lz4_set_lane_order.argtypes = [c.c_int]
    E.emu_lz4_convert.argtypes = [c.c_void_p, c.c_void_p, c.c_void_p, c.c_uint32, c.c_void_p, c.c_void_p, c.c_void_p,
                                  c.c_void_p, c.c_void_p, c.c_int, c.c_int]
    return E


def convert(src, avail, lz4s=False, snappy=False, prefix=b""):
    """ConvertBlock(Snappy) of the oracle with dst = prefix and cap(dst) - len(dst) = avail.  -> (code, body, n): code = new
    length of dst or a negative error, body = the appended bytes."""
    L = _L()
    buf = ctypes.create_string_buffer(prefix, len(prefix) + max(avail, 0) + 1)
    n = ctypes.c_int64(0)
    r = L.orc_lz4_convert(int(lz4s), int(snappy), buf, len(prefix), len(prefix) + avail, bytes(src), len(src), ctypes.byref(n))
    return r, (buf.raw[len(prefix):r] if r >= 0 else None), n.value


def uvarint(v):
    out = bytearray()
    while v >= 0x80:
        out.append((v & 0x7F) | 0x80)
        v >>= 7
    out.append(v)
    return bytes(out)


def slot_result(src, cap, lz4s=False, snappy=False):
    """What slot capacity `cap` of the device calls must produce: (code, bytes, n) with bytes = uvarint(n) + body."""
    r, body, n = convert(src, max(cap - 5, 0), lz4s, snappy)
    if r < 0:
        return r, None, 0
    if n > 0xFFFFFFFF:
        return TOO_BIG, None, n
    blk = uvarint(n) + body
    if len(blk) > cap:
        return DST_SMALL, None, 0
    return len(blk), blk, n


def min_cap(src, lz4s=False, snappy=False, hi=None):
    """Smallest slot capacity the oracle converts src with (None: it never does)."""
    hi = hi or (2 * len(src) + 64)
    if slot_result(src, hi, lz4s, snappy)[0] < 0:
        return None
    lo = 0
    while lo < hi:
        mid = (lo + hi) // 2
        if slot_result(src, mid, lz4s, snappy)[0] >= 0:
            hi = mid
        else:
            lo = mid + 1
    return lo


def compress(data, lz4s=False):
    """lz4ref CompressBlock / CompressBlockLZ4s with a dst of CompressBlockBound bytes (never "incompressible")."""
    L = _L()
    cap = L.orc_lz4_compress_bound(len(data))
    out = ctypes.create_string_buffer(cap + 64)
    r = L.orc_lz4_compress_block(int(lz4s), bytes(data), len(data), out, cap)
    assert r > 0, r
    return out.raw[:r]


def uncompress(block, cap):
    """lz4ref UncompressBlock into a dst of cap bytes: (n or negative, bytes)."""
    L = _L()
    out = ctypes.create_string_buffer(max(cap, 1))
    r = L.orc_lz4_uncompress_block(out, cap, bytes(block), len(block))
    return r, out.raw[:max(r, 0)]


def _ext(v):
    out = bytearray()
    while v >= 255:
        out.append(255)
        v -= 255
    out.append(v)
    return bytes(out)


def block(seqs, last=b"", lz4s=False):
    """A hand-built block: seqs = [(literals, offset, match length)], then a final token with `last` (LZ4) -- for LZ4s a
    sequence with offset None is a token without a match."""
    mm = 3 if lz4s else 4
    out = bytearray()
    for lits, off, ml in list(seqs) + [(last, None, None)]:
        if off is None and not lz4s and ml is not None:
            raise ValueError("LZ4 has no match-less tokens but the last")
        ll = len(lits)
        mcode = 0 if off is None else ml - mm
        out.append(min(ll, 15) << 4 | min(mcode, 15))
        if ll >= 15:
            out += _ext(ll - 15)
        out += lits
        if off is not None:
            out += bytes([off & 0xFF, off >> 8])
            if mcode >= 15:
                out += _ext(mcode - 15)
    return bytes(out)


# ---- the reference's fuzz seeds (tests/golden/lz4_*.zip, from s2/testdata/fuzz) --------------------------------------------
def fuzz_seeds():
    out = []
    for name in ("lz4_convert_corpus_raw.zip", "lz4_fuzz_block.zip"):
        z = zipfile.ZipFile(io.BytesIO(H.golden(name)))
        for nm in sorted(z.namelist()):
            out.append((name + ":" + nm, z.read(nm)))
    return out


# ---- the seeded pool -------------------------------------------------------------------------------------------------------
def pool(seed=1, lz4s=False):
    """Blocks that reach every path of the converters: fixtures, golden texts compressed by lz4ref, edge sizes, mutated blocks
    and incompressible data.  Deterministic."""
    rng = np.random.default_rng(seed)
    tw = H.golden("twain.txt")
    html = H.golden("html.txt")
    out = [b""]
    for data in (tw[:65536], tw[10000:10000 + 4096], html[:65536], html[:1000], bytes(65536), b"ab" * 5000,
                 rng.integers(0, 256, 20000, dtype=np.uint8).tobytes(), tw[:17], tw[:13], tw[:1], tw[:200000]):
        out.append(compress(data, lz4s))
    for k in range(40):                              # small random-text blocks of every size class
        n = int(rng.integers(0, 3000))
        o = int(rng.integers(0, len(tw) - n))
        out.append(compress(tw[o:o + n], lz4s))
    base = [b for b in out if len(b) > 8]
    for k in range(80):                              # mutations: flipped bytes and cut blocks
        b = bytearray(base[int(rng.integers(0, len(base)))])
        if k % 2 == 0:
            for _ in range(int(rng.integers(1, 4))):
                b[int(rng.integers(0, len(b)))] = int(rng.integers(0, 256))
        else:
            del b[int(rng.integers(1, len(b))):]
        out.append(bytes(b))
    out += [s for _, s in fuzz_seeds() if len(s) <= (1 << 20)]
    return out


def record_count(src, lz4s=False):
    """Sequences that emit something (the device walk's records) of a block the converter accepts."""
    mm = 3 if lz4s else 4
    s, n = 0, 0
    while s < len(src):
        t = src[s]
        ll, ml = t >> 4, mm + (t & 15)
        if ll == 15:
            while True:
                s += 1
                ll += src[s]
                if src[s] != 255:
                    break
        s += 1 + ll
        if ml == mm and (lz4s or s == len(src)):
            n += ll > 0
            continue
        s += 2
        if ml == mm + 15:
            while True:
                v = src[s]
                s += 1
                if v != 255:
                    break
        n += 1
    return n
