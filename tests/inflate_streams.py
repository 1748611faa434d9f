"""Hand-built DEFLATE streams for the inflate tests (RFC 1951, with the zlib and gzip containers of RFC 1950 / 1952): a
bit writer that writes every field of a stream as given -- stored blocks with any LEN / NLEN, fixed blocks, dynamic blocks
from explicit code lengths with caller-controlled HLIT / HDIST / HCLEN and code-length sequence, symbols with explicit
extra bits -- and five families of streams built with it.

Every stream is a Stream(fmt, data, valid, name, cap, records): `valid` means well-formed DEFLATE that Python's zlib must
accept too; `cap` is the destination capacity to decode it into (None: any capacity that holds the content); `records` is
the number of match, stored-run and member records the walk writes for it (set where a test relies on it)."""
import random
import struct
import zlib
from collections import namedtuple

import flate_util as F

RAW, ZLIB, GZIP = F.RAW, F.ZLIB, F.GZIP
Stream = namedtuple("Stream", "fmt data valid name cap records", defaults=(None, None))

LEN_BASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
LEN_EXTRA = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
DIST_BASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097,
             6145, 8193, 12289, 16385, 24577]
DIST_EXTRA = [0, 0, 0, 0] + [k for k in range(1, 14) for _ in (0, 1)]
CL_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
CL_EXTRA = {16: 2, 17: 3, 18: 7}
FIXED_LIT = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
FIXED_DIST = [5] * 30
EOB = 256


def canon(lens):
    """Canonical codes (RFC 1951 3.2.2): [(code, length) or None] per symbol.  Over-subscribed lengths get codes too (cut
    to their length), so a stream can go on past a header the reader must refuse."""
    maxl = max(lens, default=0)
    count = [0] * (maxl + 2)
    for ln in lens:
        if ln:
            count[ln] += 1
    nxt, code = [0] * (maxl + 2), 0
    for b in range(1, maxl + 1):
        code = (code + count[b - 1]) << 1
        nxt[b] = code
    out = []
    for ln in lens:
        if ln:
            out.append((nxt[ln] & ((1 << ln) - 1), ln))
            nxt[ln] += 1
        else:
            out.append(None)
    return out


def complete_lengths(used, n):
    """Code lengths over n symbols that give the symbols in `used` a complete code (one symbol: a single 1-bit code)."""
    lens = [0] * n
    k = len(used)
    if k == 1:
        lens[used[0]] = 1
        return lens
    b = k.bit_length() - 1
    short = (1 << (b + 1)) - k if (1 << b) != k else k
    for i, s in enumerate(sorted(used)):
        lens[s] = b if i < short else b + 1
    return lens


def deep_lengths(syms, n):
    """A complete code in which the symbols take lengths 1, 2, ..., 14, 15, 15 in the given order (16 symbols)."""
    assert len(syms) == 16
    lens = [0] * n
    for i, s in enumerate(syms):
        lens[s] = min(i + 1, 15)
    return lens


def rle(lens):
    """The code-length sequence of lens as [(symbol, extra)]: 16 / 17 / 18 for runs, greedily."""
    out, i = [], 0
    while i < len(lens):
        ln, j = lens[i], i
        while j < len(lens) and lens[j] == ln:
            j += 1
        run = j - i
        if ln == 0:
            while run >= 11:
                k = min(run, 138)
                out.append((18, k - 11))
                run -= k
            if run >= 3:
                out.append((17, run - 3))
                run = 0
            out += [(0, 0)] * run
        else:
            out.append((ln, 0))
            run -= 1
            while run >= 3:
                k = min(run, 6)
                out.append((16, k - 3))
                run -= k
            out += [(ln, 0)] * run
        i = j
    return out


def len_code(length):
    """(symbol, extra value, extra bits) of a match length; 258 as symbol 285."""
    if length == 258:
        return 285, 0, 0
    c = max(i for i in range(28) if LEN_BASE[i] <= length)
    return 257 + c, length - LEN_BASE[c], LEN_EXTRA[c]


def dist_code(dist):
    c = max(i for i in range(30) if DIST_BASE[i] <= dist)
    return c, dist - DIST_BASE[c], DIST_EXTRA[c]


def match(length, dist):
    """A match as an explicit symbol: ("x", length symbol, its extra value, distance symbol, its extra value)."""
    lc, le, _ = len_code(length)
    dc, de, _ = dist_code(dist)
    return ("x", lc, le, dc, de)


def x_length(lc, le):
    return 258 if lc == 285 else LEN_BASE[lc - 257] + le


class Writer:
    """LSB-first bit writer.  Whole bytes move to `out` whenever the stream is byte-aligned, so long streams stay linear.
    `d` counts the content bytes the written symbols produce, `records` the walk's match and stored-run records."""

    def __init__(self):
        self.out = bytearray()
        self.pend, self.pn = [], 0
        self.d = 0
        self.records = 0

    @property
    def nbits(self):
        return 8 * len(self.out) + self.pn

    def _flush(self):
        if self.pn % 8 == 0 and self.pend:
            self.out += F.pack_bits(self.pend)[:self.pn // 8]
            self.pend, self.pn = [], 0

    def bits(self, v, n):
        if n:
            assert 0 <= v < (1 << n), (v, n)
            self.pend.append((v, n))
            self.pn += n
            if self.pn >= 256:
                self._flush()
        return self

    def huff(self, code):
        """A Huffman code (code, length), written MSB first."""
        self.pend.append(("h", code[0], code[1]))
        self.pn += code[1]
        if self.pn >= 256:
            self._flush()
        return self

    def align(self):
        self.bits(0, -self.pn % 8)
        self._flush()
        return self

    def raw(self, data):
        assert self.pn % 8 == 0
        self._flush()
        self.out += data
        return self

    def data(self):
        if self.pend:
            tail = F.pack_bits(self.pend)[:(self.pn + 7) // 8]
            return bytes(self.out) + tail
        return bytes(self.out)

    # ---- blocks
    def stored(self, content, final=False, length=None, nlen=None):
        """A stored block of `content`; LEN and NLEN may be given (wrong on purpose)."""
        n = len(content) if length is None else length
        self.bits(int(final), 1).bits(0, 2).align()
        self.raw(struct.pack("<HH", n, (n ^ 0xffff) if nlen is None else nlen) + content)
        self.d += len(content)
        self.records += 1 if content else 0
        return self

    def fixed(self, syms, final=False):
        self.bits(int(final), 1).bits(1, 2)
        self.symbols(syms, canon(FIXED_LIT), canon(FIXED_DIST + [5, 5]))
        return self

    def dynamic(self, lit_lens, dist_lens, syms, final=False, hlit=None, hdist=None, hclen=None, seq=None, cl_lens=None):
        """A dynamic block.  lit_lens / dist_lens: the code lengths (HLIT / HDIST default to their sizes); seq: the
        code-length sequence [(symbol, extra)] (default: rle of the lengths); cl_lens: the 19 lengths of the code-length
        code (default: a complete code over the symbols seq uses); hclen: how many of them are written (default: up to
        the last non-zero one in CL_ORDER)."""
        seq = rle(list(lit_lens) + list(dist_lens)) if seq is None else seq
        if cl_lens is None:
            used = sorted({c[0] for c in seq})
            if len(used) == 1:
                used.append(18 if used[0] != 18 else 0)
            cl_lens = complete_lengths(used, 19)
        if hclen is None:
            hclen = max([4] + [i + 1 for i, s in enumerate(CL_ORDER) if cl_lens[s]])
        hlit = len(lit_lens) - 257 if hlit is None else hlit
        hdist = len(dist_lens) - 1 if hdist is None else hdist
        self.bits(int(final), 1).bits(2, 2).bits(hlit, 5).bits(hdist, 5).bits(hclen - 4, 4)
        for i in range(hclen):
            self.bits(cl_lens[CL_ORDER[i]], 3)
        cc = canon(cl_lens)
        for c in seq:
            if c[0] == "h":                                     # a raw code: ("h", code, length)
                self.huff(c[1:])
                continue
            self.huff(cc[c[0]])
            if c[0] in CL_EXTRA:
                self.bits(c[1], CL_EXTRA[c[0]])
        self.symbols(syms, canon(list(lit_lens)), canon(list(dist_lens)))
        return self

    def symbols(self, syms, lc, dc):
        """Literals (0-255), EOB (256), matches ("x", lsym, lextra, dsym, dextra), raw bits ("bits", v, n) and raw codes
        ("h", code, length)."""
        for s in syms:
            if isinstance(s, int):
                self.huff(lc[s])
                self.d += s < 256
            elif s[0] == "bits":
                self.bits(s[1], s[2])
            elif s[0] == "h":
                self.huff(s[1:])
            else:
                _, ls, le, ds, de = s
                self.huff(lc[ls])
                self.bits(le, LEN_EXTRA[ls - 257] if ls < 286 else 0)
                self.huff(dc[ds])
                self.bits(de, DIST_EXTRA[ds] if ds < 30 else 0)
                self.d += x_length(ls, le) if ls < 286 else 0
                self.records += 1


# ---- containers
def zlib_wrap(raw, content, fdict=None, adler=None, cmf=0x78):
    """A zlib stream: CMF, FLG (FCHECK computed, FDICT with dictionary id fdict), raw, the Adler-32 (or `adler`)."""
    flg = 0x80 | (0x20 if fdict is not None else 0)
    flg |= 31 - ((cmf << 8) | flg) % 31 if ((cmf << 8) | flg) % 31 else 0
    h = bytes([cmf, flg]) + (struct.pack(">I", fdict) if fdict is not None else b"")
    return h + raw + struct.pack(">I", zlib.adler32(content) if adler is None else adler)


def gzip_header(name=None, comment=None, extra=None, fhcrc=False, mtime=0, os_byte=255):
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
    return h


def gzip_wrap(raw, content, header=None, crc=None, isize=None):
    """A gzip member: header (default: the plain 10 bytes), raw, the CRC-32 and ISIZE (or `crc` / `isize`)."""
    return ((gzip_header() if header is None else header) + raw +
            struct.pack("<II", zlib.crc32(content) if crc is None else crc, len(content) & 0xffffffff if isize is None else isize))


def stored_stream(content, block=65535):
    """content as raw DEFLATE of stored blocks of at most `block` bytes (the last one final)."""
    w = Writer()
    for i in range(0, max(len(content), 1), block):
        w.stored(content[i:i + block], final=i + block >= len(content))
    return w.data()


def zlib_decode(fmt, data):
    """Python's zlib on the whole input (every gzip member), or None if it refuses or the stream does not end."""
    wbits = {RAW: -15, ZLIB: 15, GZIP: 31}[fmt]
    out, rest = b"", data
    try:
        while True:
            d = zlib.decompressobj(wbits)
            out += d.decompress(rest)
            if not d.eof:
                return None
            rest = d.unused_data
            if fmt != GZIP or not rest:
                return out
    except zlib.error:
        return None


# ---- families
def _text(n, seed=1):
    return F.text(random.Random(seed), n)


def _lits(data):
    return list(data)


def code_shapes():
    """Decode-table and symbol edges: 15-bit codes, every symbol, single-code trees, under- and over-subscribed codes,
    HCLEN 4 and 19, every length and distance code at both ends of its extra bits, the distance limits, maxRead."""
    out = []

    def add(name, w, valid, fmt=RAW):
        out.append(Stream(fmt, w.data() if isinstance(w, Writer) else w, valid, name))

    lit_all, dist_all = complete_lengths(list(range(286)), 286), complete_lengths(list(range(30)), 30)
    # 15-bit codes: literals a.., a length code, EOB at 15 bits; distances 15 bits deep; the last EOB ends the input
    lsyms = [97 + i for i in range(13)] + [257, 285, EOB]           # lengths 1..13, 14, 15, EOB 15
    dsyms = list(range(16))                                         # distance codes 0..15 at lengths 1..15, 15
    ll, dl = deep_lengths(lsyms, 286), deep_lengths(dsyms, 30)
    for phase in range(8):
        w = Writer()
        syms = [97 + i % 13 for i in range(390)] + [("x", 257, 0, 14, 0)] + [("x", 285, 0, dc, 0) for dc in range(16)]
        w.dynamic(ll, dl, syms, final=True)
        while (w.nbits + 15) % 8 != phase:                          # 1-bit literals: the EOB ends `phase` bits into a byte
            w.symbols([97], canon(ll), canon(dl))
        w.symbols([EOB], canon(ll), canon(dl))
        add("15-bit codes, EOB phase %d" % phase, w, True)
    # the unused part of a 15-bit peek: a complete code with the 15-bit pair and nothing after the EOB's last bit
    w = Writer().fixed([0x61, EOB], final=False)
    w.dynamic(ll, dl, [97, 98, ("x", 285, 0, 0, 0), EOB], final=True)
    add("15-bit codes after a fixed block", w, True)

    # every literal / length and distance symbol, with a complete code of all 286 and all 30
    w = Writer()
    body = [i % 256 for i in range(33000)]
    for lc in range(257, 286):
        for le in {0, (1 << LEN_EXTRA[lc - 257]) - 1}:
            for dc in range(30):
                for de in {0, (1 << DIST_EXTRA[dc]) - 1}:
                    body.append(("x", lc, le, dc, de))
    w.dynamic(lit_all, dist_all, body + [EOB], final=True)
    add("every symbol, min and max extra bits", w, True)
    # 284 with extra 31 is 258, and every length code at its extremes, in a fixed block
    w = Writer().fixed([i % 256 for i in range(300)] + [("x", 284, 31, 0, 0), ("x", 284, 30, 1, 0), ("x", 284, 0, 4, 1)] +
                       [("x", lc, e, 0, 0) for lc in range(257, 286) for e in {0, (1 << LEN_EXTRA[lc - 257]) - 1}] + [EOB],
                       final=True)
    add("fixed: 284 + 31 and every length code", w, True)

    # single-code trees (code == 1 && maxL == 1), and the unused 1-bit pattern after them
    only_eob = [0] * 257
    only_eob[EOB] = 1
    add("single-code literal/length tree: EOB only", Writer().dynamic(only_eob, [1], [EOB], final=True), True)
    add("single-code literal/length tree, unused pattern", Writer().dynamic(only_eob, [1], [("bits", 1, 1)], final=True),
        False)
    two = complete_lengths([0x41, EOB, 257], 258)
    add("single-code distance tree", Writer().dynamic(two, [1], [0x41, ("x", 257, 0, 0, 0), ("x", 257, 0, 0, 0), EOB],
                                                         final=True), True)
    d3 = [0, 0, 1]
    add("single-code distance tree: distance 3",
        Writer().dynamic(two, d3, [0x41, 0x41, 0x41, ("x", 257, 0, 2, 0), EOB], final=True), True)
    add("single-code distance tree, unused pattern",
        Writer().dynamic(two, [1], [0x41, ("x", 257, 0, 0, 0), ("h", *canon(two)[257]), ("bits", 1, 1), EOB], final=True),
        False)
    add("single 2-bit literal/length code", Writer().dynamic([0] * 256 + [2], [1], [("bits", 0, 2)], final=True), False)
    add("single 2-bit distance code", Writer().dynamic(two, [0, 2], [0x41, ("x", 257, 0, 1, 0), EOB], final=True), False)
    text = _text(400, 3)
    lit = complete_lengths(sorted(set(text)) + [EOB, 257, 265], 286)
    dist = complete_lengths([0, 5, 9], 30)
    syms = _lits(text) + [("x", 257, 0, 5, 1), ("x", 265, 1, 9, 3), EOB]
    # a code-length code of one 1-bit code (the reference accepts it; zlib refuses an incomplete code-length code).  With
    # one symbol every length is the same: 0 here, so both trees are empty and keep the previous block's tables
    one_cl = [0] * 19
    one_cl[0] = 1
    for first in (True, False):
        for unused in (False, True):
            w = Writer()
            if not first:
                w.dynamic(lit, dist, syms, final=False)
            w.dynamic([0] * 257, [0], [], final=True, seq=[(0, 0)] * 257 + ([("h", 1, 1)] if unused else [(0, 0)]),
                      cl_lens=one_cl)
            w.symbols(_lits(b"tea") + [("x", 257, 0, 5, 0), EOB], canon(lit), canon(dist))
            add("single-code code-length code%s%s" % (", first block" if first else "", ", unused pattern" if unused else ""),
                w, False)

    # under- and over-subscribed codes in each of the three tables
    add("complete dynamic block", Writer().dynamic(lit, dist, syms, final=True), True)
    under_l, over_l = list(lit), list(lit)
    under_l[ord(" ") if ord(" ") in text else text[0]] += 1
    over_l[258] = max(lit)
    under_d, over_d = list(dist), list(dist)
    under_d[9] += 1
    over_d[3] = max(dist)
    add("under-subscribed literal/length code", Writer().dynamic(under_l, dist, syms, final=True), False)
    add("over-subscribed literal/length code", Writer().dynamic(over_l, dist, syms, final=True), False)
    add("under-subscribed distance code", Writer().dynamic(lit, under_d, syms, final=True), False)
    add("over-subscribed distance code", Writer().dynamic(lit, over_d, syms, final=True), False)
    used = sorted({s for s, _ in rle(lit + dist)})
    cl = complete_lengths(used, 19)
    under_c, over_c = list(cl), list(cl)
    under_c[used[-1]] += 1
    over_c[next(s for s in range(19) if s not in used)] = max(cl)
    add("under-subscribed code-length code", Writer().dynamic(lit, dist, syms, final=True, cl_lens=under_c), False)
    add("over-subscribed code-length code", Writer().dynamic(lit, dist, syms, final=True, cl_lens=over_c), False)
    add("code lengths past HLIT + HDIST (repeat too long)",
        Writer().dynamic(lit, dist, syms, final=True, seq=rle(lit + dist)[:-1] + [(18, 127)]), False)
    add("code-length 16 first", Writer().dynamic(lit, dist, syms, final=True, seq=[(16, 0)] + rle(lit + dist)), False)

    # HCLEN 19 (every code-length symbol written), and HCLEN 4 (only 16, 17, 18, 0: every length zero)
    add("HCLEN 19", Writer().dynamic(lit, dist, syms, final=True, hclen=19), True)
    add("HCLEN 19, complete 19-symbol code-length code",
        Writer().dynamic(lit, dist, syms, final=True, hclen=19, cl_lens=complete_lengths(list(range(19)), 19)), True)
    zero_seq = [(18, 127), (18, 127), (17, 1), (18, 25)]            # 138 + 138 + 4 + 36 = 316 zeros
    hc4_cl = [0] * 19
    hc4_cl[16], hc4_cl[17], hc4_cl[18], hc4_cl[0] = 2, 2, 2, 2
    add("HCLEN 4 as the first block (no table yet)",
        Writer().dynamic([0] * 286, [0] * 30, [("bits", 0, 16)], final=True, hclen=4, seq=zero_seq, cl_lens=hc4_cl), False)
    w = Writer().dynamic(lit, dist, syms[:-1] + [EOB], final=False)
    w.dynamic([0] * 286, [0] * 30, [], final=True, hclen=4, seq=zero_seq, cl_lens=hc4_cl)
    w.symbols([0x61, ("x", 257, 0, 5, 0), EOB], canon(lit), canon(dist))
    add("HCLEN 4 after a dynamic block (stale tables)", w, False)
    # 16, 17, 18 at their minimum and maximum repeats
    lens = complete_lengths(list(range(286)), 286)                  # 0..225 at 8 bits, 226..285 at 9
    seq = [(8, 0)] + [(16, 3)] * 37 + [(16, 0)] + [(9, 0)] + [(16, 3)] * 9 + [(16, 0)] + [(9, 0)] * 2
    dlens = [1, 1] + [0] * 28
    dseq = [(1, 0), (1, 0), (17, 7), (17, 0), (18, 0), (0, 0), (0, 0), (0, 0), (0, 0)]
    rep = {16: 3, 17: 3, 18: 11}
    assert sum(1 if s < 16 else rep[s] + e for s, e in seq + dseq) == 316
    add("code lengths with 16 and 17 at their minimum and maximum repeats",
        Writer().dynamic(lens, dlens, [0x61, 0x62, ("x", 257, 0, 1, 0), ("x", 258, 0, 0, 0), EOB], final=True,
                         seq=seq + dseq), True)
    two_lit = complete_lengths([0x41, EOB], 257)
    seq18 = [(18, 54), (1, 0), (18, 127), (18, 0), (18, 30), (1, 0), (1, 0)]   # 65, 1, 138 + 11 + 41, 1 | 1
    add("code lengths with 18 at its minimum and maximum repeats",
        Writer().dynamic(two_lit, [1], [0x41, 0x41, EOB], final=True, seq=seq18), True)

    # distances: exactly 32 768, exactly d - mstart, and one more
    big = random.Random(9).randbytes(32768 + 50)
    w = Writer()
    w.stored(big[:32768]).stored(big[32768:])
    w.fixed([match(258, 32768), match(3, 32768), ("x", 285, 0, 29, (1 << 13) - 1), EOB], final=True)
    add("distance 32768", w, True)
    for k in (1, 2, 7, 300):
        content = _text(k, k)
        for fmt in (RAW, ZLIB, GZIP):
            for extra in (0, 1):
                w = Writer().fixed(_lits(content) + [match(3, k + extra), EOB], final=True)
                raw = w.data()
                full = content + (content * 3)[:3] if not extra else content
                data = raw if fmt == RAW else (zlib_wrap(raw, full) if fmt == ZLIB else gzip_wrap(raw, full))
                add("distance d - mstart%s, %d bytes" % (" + 1" if extra else "", k), data, not extra, fmt)
    # across gzip members: the second member's history starts empty
    m1 = gzip_wrap(Writer().fixed(_lits(b"abcdef") + [EOB], final=True).data(), b"abcdef")
    for extra in (0, 1):
        w = Writer().fixed([0x78, 0x79, match(4, 2 + extra), EOB], final=True)
        c2 = b"xyxyxy" if not extra else b""
        add("second gzip member, distance d - mstart%s" % (" + 1" if extra else ""), m1 + gzip_wrap(w.data(), c2),
            not extra, GZIP)

    # maxRead: a non-final block's EOB, then the smallest final block (3 + 7 bits, exactly the + 10) at every bit phase;
    # then the same with the final block cut short, and with nothing after the EOB
    lit17 = complete_lengths(sorted(set(text)) + [EOB, 257, 265, 0x7e], 286)   # 257 and 265 at 5 bits
    odd = ("x", 265, 0, 0, 0)                                      # 5 + 1 + 1 bits
    for k in range(8):
        w = Writer().dynamic(lit17, dist, syms[:-1] + [odd] * k + [EOB], final=False)
        eob_end = w.nbits
        w.fixed([EOB], final=True)
        add("non-final dynamic block, EOB phase %d, then the smallest final block" % (eob_end % 8), w, True)
        data = w.data()
        add("non-final dynamic block, EOB phase %d, final block cut" % (eob_end % 8), data[:(eob_end + 9) // 8], False)
        add("non-final dynamic block, EOB phase %d, nothing after" % (eob_end % 8), data[:(eob_end + 7) // 8], False)
    return out


def exec_layouts():
    """Record layouts for the exec kernel: chains of matches that read the previous match's output (byte, word and
    whole-warp copy distances and lengths), chains across a 32-record step, and stored runs between literals and matches
    at every output offset mod 16 and input offset mod 4."""
    out = []
    seed = b"0123456789abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ" * 6
    for dists in ((1, 2, 3, 4, 5, 6, 7, 8), (8, 9, 12, 15, 16), (17, 31, 64, 100, 257, 300)):
        for length in (3, 63, 64, 258):
            for nmatch in (5, 31, 32, 33, 70):
                syms = _lits(seed[:301])
                for k in range(nmatch):
                    syms.append(match(length, dists[k % len(dists)]))
                    if k % 11 == 10:
                        syms.append(0x5f)                    # a literal inside the chain shifts the next step
                w = Writer().fixed(syms + [EOB], final=True)
                out.append(Stream(RAW, w.data(), True, "chain d%s len %d x%d" % (dists, length, nmatch), None, w.records))
    # stored runs of 1..40 bytes at every output offset mod 16 and input offset mod 4, with a literal and a match on each side
    rng = random.Random(4)
    for n in range(1, 41):
        for imod in range(4):
            w = Writer()
            w.fixed(_lits(seed[:20]) + [EOB], final=False)
            for omod in range(16):
                pre = [0x2e] * ((omod - (w.d + 1 + 5)) % 16)
                w.fixed(pre + [0x2d, match(5, 7), EOB], final=False)
                # empty stored blocks move the input by 5 bytes (1 mod 4) without output or records
                bits_after = w.nbits + 3
                pos = (bits_after + 7) // 8 + 4
                for _ in range((imod - pos) % 4):
                    w.stored(b"")
                assert w.d % 16 == omod
                run = bytes(rng.getrandbits(8) for _ in range(n))
                w.stored(run)
                assert (len(w.out) - n) % 4 == imod
                w.fixed([0x2b, match(n + 3, n + 1), match(3, n + 6), EOB], final=False)
            w.fixed([EOB], final=True)
            out.append(Stream(RAW, w.data(), True, "stored runs of %d bytes, input offset %d mod 4" % (n, imod), None,
                              w.records))
    return out


def checksum_sizes(big=True):
    """zlib and gzip streams of stored content, each with its right trailer and with one checksum bit flipped: sizes
    0-300, 128k + 0..3, 177 664 - 1 .. + 1 (the Adler-32 fold's per-lane NMAX edge), and with big: 1 MiB and 16 MiB of
    0xff (the Adler-32 worst case).  Plus multi-member gzip with members of 1-7 bytes and one bad CRC, before and after a
    later walk error."""
    rng = random.Random(12)
    sizes = list(range(301)) + [128 * k + j for k in (3, 17, 100, 511, 1000) for j in range(4)] + [177663, 177664, 177665]
    if big:
        sizes += [1 << 20, 16 << 20]
    out = []
    for n in sizes:
        content = b"\xff" * n if n == 16 << 20 else rng.randbytes(n)
        raw = stored_stream(content)
        bit = n % 32
        for fmt in (ZLIB, GZIP):
            for bad in (False, True):
                if fmt == ZLIB:
                    s = zlib_wrap(raw, content, adler=zlib.adler32(content) ^ (1 << bit) if bad else None)
                else:
                    s = gzip_wrap(raw, content, crc=zlib.crc32(content) ^ (1 << bit) if bad else None)
                out.append(Stream(fmt, s, not bad, "%s %d bytes%s" % ("zlib" if fmt == ZLIB else "gzip", n,
                                                                      ", bad checksum" if bad else ""), n + 16))
    members = [bytes(rng.getrandbits(8) for _ in range(k)) for k in (1, 2, 3, 4, 5, 6, 7, 3, 1, 6)]
    good = [gzip_wrap(Writer().fixed(_lits(m) + [EOB], final=True).data(), m) for m in members]
    out.append(Stream(GZIP, b"".join(good), True, "members of 1-7 bytes"))
    for j in range(len(members)):
        m = members[j]
        bad = gzip_wrap(Writer().fixed(_lits(m) + [EOB], final=True).data(), m, crc=zlib.crc32(m) ^ 0x80000000)
        walk_err = gzip_wrap(Writer().fixed([0x41, match(3, 5), EOB], final=True).data(), b"Axxx")
        parts = good[:j] + [bad] + good[j + 1:]
        out.append(Stream(GZIP, b"".join(parts), False, "members of 1-7 bytes, bad CRC in member %d" % j))
        out.append(Stream(GZIP, b"".join(parts[:j + 1] + [walk_err] + parts[j + 1:]), False,
                          "bad CRC in member %d, then a walk error" % j))
        out.append(Stream(GZIP, b"".join(good[:j] + [walk_err] + parts[j:]), False,
                          "walk error, then a bad CRC in member %d" % j))
    return out


def _two_bit_matches(length, nbody, cap_exact):
    """One raw stream: a 1-byte stored block, then a final dynamic block whose literal/length code is {EOB, the code of
    `length`} at 1 bit each and whose distance code is one 1-bit code (distance 1): every match takes 2 bits."""
    lc = len_code(length)[0]
    lit = [0] * (lc + 1)
    lit[EOB], lit[lc] = 1, 1
    w = Writer().stored(b"\x07")
    w.dynamic(lit, [1], [("x", lc, 0, 0, 0)] * nbody + [EOB], final=True)
    data = w.data()
    return Stream(RAW, data, True, "%d 2-bit matches of %d bytes" % (nbody, length), w.d if cap_exact else w.d + 64, w.records)


def record_bound(big=True):
    """Streams whose record count comes as close to inf_rec_cap(slen, cap) as the format allows, one per term: 2-bit
    258-byte matches (4 * slen binds), 2-bit 3-byte matches into exactly their content (cap / 3 binds), runs of 1-byte
    non-final stored blocks (slen / 5), gzip of 20-byte empty members (slen / 18).  With big: long enough that the
    records reach 99% of the match term (or slen / 6 and slen / 20)."""
    k = 12000 if big else 300
    out = [_two_bit_matches(258, k, False), _two_bit_matches(3, 4 * k, True)]
    rng = random.Random(5)
    w = Writer()
    for i in range(k):
        w.stored(bytes([rng.getrandbits(8)]), final=i == k - 1)
    out.append(Stream(RAW, w.data(), True, "%d 1-byte stored blocks" % k, w.d + 16, w.records))
    empty = gzip_wrap(Writer().fixed([EOB], final=True).data(), b"")
    assert len(empty) == 20
    out.append(Stream(GZIP, empty * k, True, "%d empty gzip members" % k, 16, k))
    return out


def record_term(s):
    """(records, the lower bound the stream is built to reach) for a record_bound() stream."""
    slen = len(s.data)
    if "matches" in s.name:
        return s.records, 0.99 * min(s.cap // 3, 4 * slen)
    if "stored" in s.name:
        return s.records, slen / 6
    return s.records, slen / 20


def header_edges():
    """gzip and zlib header edges: FNAME / FCOMMENT at the 512-byte readString limit, a second member cut inside FNAME
    (io.EOF: the members end), FEXTRA or FHCRC (io.ErrUnexpectedEOF), FHCRC right and wrong, zlib FDICT with dictionary
    id 1 (the empty dictionary: read without one) and any other id."""
    content = b"header edges " * 5
    raw = Writer().fixed(_lits(content) + [EOB], final=True).data()
    out = []
    for field in ("name", "comment"):
        for n in (0, 1, 510, 511, 512, 600):
            h = gzip_header(**{field: b"n" * n})
            # readString reads at most 512 bytes, the NUL included: a 512-byte string is ErrHeader (Python's zlib reads it)
            out.append(Stream(GZIP, gzip_wrap(raw, content, h), n < 512, "%s of %d bytes" % (field, n)))
    first = gzip_wrap(raw, content)
    for fields, valid_cut in ((dict(name=b"second.txt"), True), (dict(comment=b"a comment"), True),
                              (dict(extra=b"EXTRA!"), False), (dict(fhcrc=True), False),
                              (dict(name=b"nm", extra=b"xx", fhcrc=True), False)):
        h = gzip_header(**fields)
        for cut in range(10, len(h)):
            # a cut inside FNAME / FCOMMENT is io.EOF, the clean end of the members; inside FEXTRA / FHCRC it is
            # io.ErrUnexpectedEOF (-12).  Python's zlib refuses every cut member, so none of these is `valid`.
            out.append(Stream(GZIP, first + h[:cut], False, "second member cut at %d of %r" % (cut, sorted(fields))))
        out.append(Stream(GZIP, first + gzip_wrap(raw, content, h), True, "second member with %r" % sorted(fields)))
    h = gzip_header(name=b"x", fhcrc=True)
    out.append(Stream(GZIP, gzip_wrap(raw, content, h[:-1] + bytes([h[-1] ^ 4])), False, "FHCRC wrong"))
    for dict_id in (1, 0, 2, 0xffffffff, zlib.adler32(b"dict")):
        # Python's zlib needs the dictionary for any FDICT stream; the reference reads id 1 without one
        out.append(Stream(ZLIB, zlib_wrap(raw, content, fdict=dict_id), False, "FDICT id %#x" % dict_id))
    for cut in range(2, 6):
        out.append(Stream(ZLIB, zlib_wrap(raw, content, fdict=1)[:cut], False, "FDICT cut at %d" % cut))
    out.append(Stream(ZLIB, zlib_wrap(raw, content), True, "zlib"))
    out.append(Stream(ZLIB, zlib_wrap(raw, content, cmf=0x08), True, "zlib CINFO 0"))
    out.append(Stream(ZLIB, zlib_wrap(raw, content, cmf=0x88), False, "zlib CINFO 8"))
    return out


def truncation_set():
    """Streams to cut at every length: a few code_shapes() and exec_layouts() streams, the level 0 / 1 / 9 streams of
    3000 bytes of text in each format, and a raw stream of non-final dynamic blocks with length and distance extra bits
    (a cut there meets maxRead's + 10)."""
    shapes = code_shapes()
    pick = [s for s in shapes if s.name in ("15-bit codes, EOB phase 0", "complete dynamic block", "HCLEN 19",
                                            "code lengths with 16, 17, 18 at their minimum and maximum repeats")]
    pick += [s for s in exec_layouts() if s.name in ("chain d(8, 9, 12, 15, 16) len 64 x33",
                                                     "stored runs of 13 bytes, input offset 3 mod 4")]
    out = [(s.fmt, s.data) for s in pick]
    data = F.text(random.Random(3), 3000)
    for fmt in (RAW, ZLIB, GZIP):
        for level in (0, 1, 9):
            out.append((fmt, F.deflate(data, fmt, level)))
    text = _text(600, 8)
    lit = complete_lengths(sorted(set(text)) + [EOB] + list(range(265, 286)), 286)
    dist = complete_lengths(list(range(4, 30)), 30)
    w = Writer()
    for blk in range(3):
        syms = _lits(text[blk * 200:blk * 200 + 200])
        syms += [("x", lc, (1 << LEN_EXTRA[lc - 257]) - 1 if lc % 2 else 0, dc, (1 << DIST_EXTRA[dc]) - 1 if dc % 2 else 0)
                 for lc, dc in zip(range(265, 285), range(4, 18)) if DIST_BASE[dc] + (1 << DIST_EXTRA[dc]) <= 200 * blk + 200]
        w.dynamic(lit, dist, syms + [EOB], final=blk == 2)
    out.append((RAW, w.data()))
    return out
