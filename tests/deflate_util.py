"""Deflate-encoder test helpers: the oracle (oracle/liboracle_deflate.so, built on demand), a seeded input pool, the
reference's encoder fuzz corpus and inputs that reach particular decision paths."""
import ctypes
import io
import os
import random
import subprocess
import zipfile

import helpers as H

ORACLE_DEFLATE_SO = os.path.join(H.ORACLE_DIR, "liboracle_deflate.so")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
STEP = 24575                        # maxStatelessBlock - maxStatelessDict: every block after the first
PATHS = ["stored_empty_tokens", "huff_stored_test", "huff_stored_est", "huff_new", "huff_reuse", "dyn_new", "dyn_reuse",
         "dyn_fixed", "dyn_stored", "eob_before_stored", "long_match"]
_L = None


def oracle():
    global _L
    if _L is None:
        if not os.path.exists(ORACLE_DEFLATE_SO):
            subprocess.run(["make", "-s", "-C", H.ORACLE_DIR, "-f", "deflate.mk"], check=True)
        L = ctypes.CDLL(ORACLE_DEFLATE_SO)
        c = ctypes
        L.orc_deflate_stateless.restype = c.c_int64
        L.orc_deflate_stateless.argtypes = [c.c_char_p, c.c_size_t, c.c_int, c.c_char_p, c.c_size_t, c.c_char_p, c.c_size_t]
        L.orc_deflate_gzip.restype = c.c_int64
        L.orc_deflate_gzip.argtypes = [c.c_char_p, c.c_size_t, c.c_char_p, c.c_size_t, c.c_char_p, c.c_size_t]
        L.orc_deflate_block_huff.restype = c.c_int64
        L.orc_deflate_block_huff.argtypes = [c.c_char_p, c.c_size_t, c.c_uint, c.c_char_p, c.c_size_t]
        L.orc_deflate_block_dynamic.restype = c.c_int64
        L.orc_deflate_block_dynamic.argtypes = [c.c_void_p, c.c_size_t, c.c_char_p, c.c_size_t, c.c_int, c.c_char_p,
                                                c.c_size_t]
        L.orc_deflate_paths.argtypes = [c.c_void_p]
        _L = L
    return _L


def blocks(n, dict_len=0):
    """StatelessDeflate's blocks for an n-byte input: the first 32 767 - dict bytes, then 24 575 each."""
    b0 = 32767 - min(dict_len, 8192)
    return 0 if n == 0 else 1 + max(0, -(-(n - b0) // STEP))


def bound(n):
    return n + 5 * (n // 16384 + 2) + 64


def stateless(data, eof=True, dict=None):
    """StatelessDeflate(out, data, eof, dict) by the oracle."""
    cap = bound(len(data))
    out = ctypes.create_string_buffer(cap)
    d = bytes(dict) if dict else None
    r = oracle().orc_deflate_stateless(bytes(data), len(data), int(eof), d, len(d) if d else 0, out, cap)
    assert r >= 0, r
    return out.raw[:r]


def gzip_member(data, header=b"\x1f\x8b\x08\x00\x00\x00\x00\x00\x00\xff"):
    cap = bound(len(data)) + len(header) + 16
    out = ctypes.create_string_buffer(cap)
    r = oracle().orc_deflate_gzip(header, len(header), bytes(data), len(data), out, cap)
    assert r >= 0, r
    return out.raw[:r]


def paths():
    a = (ctypes.c_int64 * len(PATHS))()
    oracle().orc_deflate_paths(a)
    return dict(zip(PATHS, list(a)))


def text(rng, n):
    words = [bytes(rng.choice(b"etaoinshrdlu ETAOIN.,\n") for _ in range(rng.randint(1, 9))) for _ in range(300)]
    return b" ".join(rng.choice(words) for _ in range(n // 4 + 1))[:n]


def sparse(rng, n):
    """Random bytes with a repeated snippet now and then: a few matches, an almost flat histogram."""
    snip = rng.randbytes(12)
    return b"".join(rng.randbytes(600) + snip for _ in range(n // 612 + 1))[:n]


def skewed(rng, n):
    """Bytes from a mildly skewed distribution over 15 symbols: few matches found, under 4 bits of entropy per byte, so the
    blocks take the Huffman-only paths."""
    return bytes(rng.choices(range(40, 55), weights=[1.03 ** -i for i in range(15)], k=n))


def debruijn(k, n):
    """The de Bruijn sequence B(k, n): every n-symbol word over k symbols exactly once (cyclically)."""
    a, seq = [0] * k * n, []

    def db(t, p):
        if t > n:
            if n % p == 0:
                seq.extend(a[1:p + 1])
        else:
            a[t] = a[t - p]
            db(t + 1, p)
            for j in range(a[t - p] + 1, k):
                a[t] = j
                db(t + 1, t)
    db(1, 1)
    return seq


def huff_runs(n):
    """Consecutive Huffman-only blocks that reuse their table: B(14, 4) (no 4-byte word repeats within 38 416 bytes, so
    within no block's window; 3.86 bits per byte) with one fixed 48-byte snippet per 1 000 bytes, so each block finds a few
    matches (dst.n > 0) but removes less than 1/16 of its bytes."""
    s = bytes(97 + x for x in debruijn(14, 4))
    snip, out, i = s[5000:5048], b"", 0
    while len(out) < n:
        out += s[i % len(s):i % len(s) + 1000] + snip
        i += 1000
    return out[:n]


def sizes():
    s = [0, 1, 12, 13, 14, 100, 1025, 4000, STEP, 32766, 32767, 32768]
    for k in (1, 2, 3, 5):
        s += [32767 + k * STEP - 1, 32767 + k * STEP, 32767 + k * STEP + 1]
    return s


def pool(seed=5):
    """(label, data): every size of sizes() as text, random, zeros and periodic content."""
    rng = random.Random(seed)
    out = []
    for n in sizes():
        out.append(("text", text(rng, n)))
        out.append(("random", rng.randbytes(n)))
        out.append(("zeros", bytes(n)))
        per = rng.randbytes(rng.randint(1, 300))
        out.append(("periodic", (per * (n // max(len(per), 1) + 1))[:n]))
    # mixed content: blocks whose decisions differ from their neighbours' (table reuse, owed EOBs, fixed blocks)
    mix = b""
    while len(mix) < 6 * STEP:
        k = rng.randrange(7)
        m = rng.randint(200, 20000)
        mix += [text(rng, m), rng.randbytes(m), bytes(m), b"ab" * (m // 2), bytes(rng.choice(b"acgt") for _ in range(m)),
                sparse(rng, m), skewed(rng, m)][k]
    out.append(("mixed", mix))
    for n in (3000, STEP, 4 * STEP + 7):
        out.append(("sparse", sparse(rng, n)))
        out.append(("skewed", skewed(rng, n)))
    return out


def dict_cases(seed=7):
    """(data, dict): dicts of 1 byte to 8 KiB and longer ones (only their last 8 KiB count)."""
    rng = random.Random(seed)
    base = text(rng, 200000)
    out = []
    for dl in (1, 4, 13, 100, 4096, 8191, 8192, 8193, 20000):
        for n in (0, 5, 13, 3000, 32767 - min(dl, 8192), 32767 - min(dl, 8192) + 1, 70000):
            st = rng.randrange(0, 100000)
            out.append((base[st + dl:st + dl + n], base[st:st + dl]))
    out.append((rng.randbytes(40000), rng.randbytes(9000)))
    return out


def fuzz_inputs():
    with zipfile.ZipFile(os.path.join(GOLDEN, "deflate_fuzz_corpus.zip")) as z:
        return [z.read(n) for n in sorted(z.namelist())]


def fuzz_split(data):
    """FuzzEncoding's stateless leg (flate/fuzz_test.go:100-124): the first half, then the rest with the first half as
    dict.  Returns [(data, eof, dict)]."""
    h = len(data) // 2
    return [(data[:h], False, None), (data[h:], True, data[:h])]


def testdata(name):
    with zipfile.ZipFile(os.path.join(GOLDEN, "flate_testdata.zip")) as z:
        return z.read(name)


def testdata_names():
    with zipfile.ZipFile(os.path.join(GOLDEN, "flate_testdata.zip")) as z:
        return z.namelist()
