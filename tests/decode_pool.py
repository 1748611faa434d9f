"""A seeded pool of zstd and S2 inputs with their expected decode results, shared by test_emu_decode_shapes.py (the
emulated kernels, CPU) and test_decode_shapes_gpu.py (the device).  Expected results come from the oracle decoders;
valid zstd frames are also read back with libzstd when the pool is built.

The encoders that make the library's own frames are passed in: the emulated kernels on the CPU, the device on the GPU.
Both must produce the same bytes, and every entry carries a digest so the GPU module can tell (the per-form staged flags
recorded by the CPU module in tests/golden/decode_pool_flags.json belong to exactly these bytes).

Entries are dicts: name, data, cap (capacity the pool's own runs use), code (oracle result at cap), out (bytes),
blocks (block count of a single frame, or None), valid (an undamaged input), sha."""
import hashlib
import json
import os

import numpy as np

import helpers as H

POOL_CAP = 200000            # capacity of every small entry (>= the largest small entry's content, except "cap_over")
FORMS = (4, 16, 127, 128)    # the staged decoder's blocks per input: per-input form (4), per-block form (> 4)
FLAGS_PATH = os.path.join(H.GOLDEN, "decode_pool_flags.json")
FB = 49152                   # frame mode's block size at level 1
SENT = 0xA5


def maxb_for(n):
    """Blocks per input of the staged decoder for a batch of n inputs (b2c_api.cu launch_decode)."""
    return 4 if n > 4096 else min(128, 65536 // n)


def sha(b):
    return hashlib.sha1(bytes(b)).hexdigest()[:16]


def _data(kind, n, seed):
    rng = np.random.default_rng(seed)
    tw = H.golden("twain.txt")
    if n == 0:
        return b""
    if kind == "text":
        return H.synth_text(n, seed=seed)
    if kind == "twain":
        return (tw * (n // len(tw) + 1))[:n]
    if kind == "random":
        return rng.integers(0, 256, n, dtype=np.uint8).tobytes()
    if kind == "zeros":
        return bytes(n)
    if kind == "low":
        return rng.integers(0, 4, n, dtype=np.uint8).tobytes()
    raise ValueError(kind)


_KINDS = ("text", "twain", "random", "zeros", "low")


# ---------------------------------------------------------------------------------------------- hand-assembled frames
def raw_rle_frame(content_blocks):
    """One frame of raw / RLE blocks: content_blocks = list of (kind, bytes); header with a 64 KiB window, 4-byte content
    size and a content checksum (XXH64's low 32 bits)."""
    content = b"".join(b for _, b in content_blocks)
    out = bytearray(b"\x28\xb5\x2f\xfd")
    out += bytes([0x84, 0x30])                      # FCS field 4 bytes, checksum, window 1 << 16
    out += len(content).to_bytes(4, "little")
    for i, (kind, b) in enumerate(content_blocks):
        last = 1 if i + 1 == len(content_blocks) else 0
        t = 0 if kind == "raw" else 1
        out += (last | t << 1 | len(b) << 3).to_bytes(3, "little")
        out += b if kind == "raw" else b[:1]
    out += (H.oracle().orc_xxh64(content, len(content), 0) & 0xFFFFFFFF).to_bytes(4, "little")
    return bytes(out), content


def raw_rle_blocks(k, seed):
    rng = np.random.default_rng(seed)
    blocks = []
    for i in range(k):
        if i % 2 == 0:
            blocks.append(("raw", rng.integers(0, 256, int(rng.integers(1, 40)), dtype=np.uint8).tobytes()))
        else:
            blocks.append(("rle", bytes([int(rng.integers(0, 256))]) * int(rng.integers(1, 300))))
    return blocks


def reach_back_frame():
    """Two blocks: a raw one, then a compressed one whose only sequence (no literals, offset code 1) is a repeat offset --
    it resolves to the frame's initial repeat offset 4, which the per-block form cannot know."""
    first = b"abcd" * 40
    second = b"abcd" * 25
    r, blk = H.oracle_encode_block(second, b"", [[0, len(second) - 3, 1]], last=1)
    assert r > 0 and (blk[0] >> 1) & 3 == 2, "expected a compressed block"
    content = first + second
    out = bytearray(b"\x28\xb5\x2f\xfd") + bytes([0x84, 0x30]) + len(content).to_bytes(4, "little")
    out += (len(first) << 3).to_bytes(3, "little") + first
    out += blk
    out += (H.oracle().orc_xxh64(content, len(content), 0) & 0xFFFFFFFF).to_bytes(4, "little")
    return bytes(out), content


def libzstd_frame(data, level):
    Z = H.libzstd()
    import ctypes
    cap = Z.ZSTD_compressBound(len(data))
    out = ctypes.create_string_buffer(cap)
    r = Z.ZSTD_compress(out, cap, bytes(data), len(data), level)
    assert not Z.ZSTD_isError(r)
    return out.raw[:r]


def frame_blocks(f):
    """Block count of the first frame of f (None if it cannot be walked)."""
    if len(f) < 6 or f[:4] != b"\x28\xb5\x2f\xfd":
        return None
    fhd = f[4]
    q = 5 + (0 if fhd & 0x20 else 1) + [0, 1, 2, 4][fhd & 3]
    q += [1 if fhd & 0x20 else 0, 2, 4, 8][fhd >> 6]
    nb = 0
    while q + 3 <= len(f):
        bh = int.from_bytes(f[q:q + 3], "little")
        q += 3 + (1 if (bh >> 1) & 3 == 1 else bh >> 3)
        nb += 1
        if bh & 1:
            return nb
    return None


def skippable(payload):
    return b"\x5a\x2a\x4d\x18" + len(payload).to_bytes(4, "little") + payload


# ---------------------------------------------------------------------------------------------- zstd pool
def build_zstd(enc_chunks, enc_frames):
    """enc_chunks(level, chunks) -> one-block frames (the library's chunk encoder); enc_frames(inputs) -> level-1 frame-mode
    frames.  Returns the list of entries."""
    ents = []

    def add(name, data, want=None, cap=POOL_CAP, valid=True):
        r, out = H.oracle_decode(data, cap)
        if want is not None:
            assert r == len(want) and out == want, (name, r)
        if valid and r > 0 and data[:4] == b"\x28\xb5\x2f\xfd":
            assert H.libzstd_decode(data, r) == out, name
        ents.append(dict(name=name, data=bytes(data), cap=cap, code=int(r), out=out, blocks=frame_blocks(data), valid=valid,
                         sha=sha(data)))

    sizes = {1: [0, 1, 2, 9, 100, 1023, 1025, 4097, 33333, 65535, 65536],
             2: [0, 1, 2, 777, 65537, 131071, 131072],
             3: [0, 2, 5001, 131072]}
    for level, ss in sizes.items():
        chunks = [_data(_KINDS[i % len(_KINDS)], s, 100 * level + i) for i, s in enumerate(ss)]
        for s, c, f in zip(ss, chunks, enc_chunks(level, chunks)):
            add("L%d_%d" % (level, s), f, c)
    fm = [1000, FB + 1, 2 * FB + 7, 3 * FB + 100, 4 * FB, 4 * FB + 1]       # 1 .. 5 blocks; 4 * FB (+1): the 4 / 5 boundary
    fm_data = [_data(_KINDS[i % len(_KINDS)], s, 300 + i) for i, s in enumerate(fm)]
    for s, c, f in zip(fm, fm_data, enc_frames(fm_data)):
        add("FM_%d" % s, f, c)
    cap_data = [_data("text", POOL_CAP, 400), _data("text", POOL_CAP + 1, 401)]
    cf = enc_frames(cap_data)
    add("cap_exact", cf[0], cap_data[0])                                   # content == capacity: decodes
    add("cap_over", cf[1])                                                 # one byte more: the oracle's error
    assert ents[-1]["code"] < 0
    lz = _data("twain", 150000, 0)[:75000] + _data("low", 75000, 500)       # two 128 KiB-window blocks
    for level in (-5, 1, 3, 19):
        add("libzstd_%d" % level, libzstd_frame(lz, level), lz)
        add("libzstd_%d_small" % level, libzstd_frame(lz[:3000], level), lz[:3000])
    for i, (s, level) in enumerate([(70000, 1), (150000, 2), (3000, 3)]):
        d = _data(_KINDS[i], s, 600 + i)
        add("oracle_L%d_%d" % (level, s), H.oracle_encode(d, level=level)[1], d)
    add("empty", b"")
    add("skippable_only", skippable(b"xyz" * 5))
    a, b = _data("text", 5000, 700), _data("twain", 7001, 701)
    fa, fb = enc_chunks(1, [a, b])
    add("two_frames_skippable", fa + skippable(b"pad") + fb, a + b)
    for kk in (4, 5, 16, 17, 127, 128, 129):                              # k and k + 1 blocks for k = 4, 16, 127, 128
        f, content = raw_rle_frame(raw_rle_blocks(kk, 800 + kk))
        add("rawrle_%d" % kk, f, content)
    f, content = reach_back_frame()
    add("reach_back", f, content)
    # damaged variants of small frames
    rng = np.random.default_rng(900)
    bases = [e for e in ents if e["name"] in ("L1_1025", "L1_4097", "L1_33333", "L2_777", "L2_65537", "L3_5001", "FM_1000",
                                              "FM_49153", "libzstd_1_small", "libzstd_19_small", "oracle_L3_3000",
                                              "oracle_L1_70000")]
    assert len(bases) == 12
    for e in bases:
        d = e["data"]
        fh = 6 + (0 if d[4] & 0x20 else 1) + [1 if d[4] & 0x20 else 0, 2, 4, 8][d[4] >> 6] - 1
        tail = 4 if d[4] & 4 else 0
        spots = {"hdr": int(rng.integers(4, fh)), "lit": fh + 3 + int(rng.integers(0, 4)),
                 "seq": len(d) - tail - 1 - int(rng.integers(0, 3)), "crc": len(d) - 1 - int(rng.integers(0, 4))}
        for where, pos in spots.items():
            if where == "crc" and not tail:
                continue
            b = bytearray(d)
            b[pos] ^= 1 << int(rng.integers(0, 8))
            add("%s_flip_%s" % (e["name"], where), bytes(b), valid=False)
        add(e["name"] + "_trunc1", d[:-1], valid=False)
        add(e["name"] + "_trunc_half", d[:len(d) // 2], valid=False)
        add(e["name"] + "_cap_size", d, e["out"], cap=len(e["out"]))
        add(e["name"] + "_cap_short", d, cap=len(e["out"]) - 1, valid=False)
    names = [e["name"] for e in ents]
    assert len(set(names)) == len(names)
    return ents


def small(ents):
    """The entries the batch sweep tiles: everything but the per-entry-capacity variants."""
    return [e for e in ents if e["cap"] == POOL_CAP]


def frame_mode_boundary(enc_frames, ks):
    """Level-1 frame-mode frames of k * 48 KiB (k blocks) and k * 48 KiB + 1 bytes (k + 1 blocks).  Returns
    {blocks: (frame, content)}; the frames are checked with the oracle decoder."""
    datas = []
    for k in ks:
        base = _data("text", k * FB + 1, 1000 + k)
        datas += [base[:-1], base]
    out = {}
    for d, f in zip(datas, enc_frames(datas)):
        nb = frame_blocks(f)
        assert nb == (len(d) + FB - 1) // FB, (len(d), nb)
        r, back = H.oracle_decode(f, len(d))
        assert r == len(d) and back == d, nb
        out[nb] = (f, d)
    return out


# ---------------------------------------------------------------------------------------------- S2 pool
def s2_varint(n):
    out = bytearray()
    while n >= 0x80:
        out.append(n & 0x7F | 0x80)
        n >>= 7
    out.append(n)
    return bytes(out)


def s2_copy1_block(k):
    """One literal byte, then k two-byte copy1 tags (offset 1): slen = 3 + 2k, k elements; the staged walk holds
    slen / 3 + 1 of them, so k = 6 is the largest count it takes and k = 7 one more."""
    lens = [4 + (i * 5) % 8 for i in range(k)]
    body = bytes([0]) + b"Q" + b"".join(bytes([1 | (ln - 4) << 2, 1]) for ln in lens)
    return s2_varint(1 + sum(lens)) + body


def build_s2(enc_blocks):
    """enc_blocks(blocks, better) -> S2 blocks (the library's encoders)."""
    from test_oracle_s2 import s2_decode, s2_encode
    ents = []

    def add(name, data, cap=POOL_CAP, want=None, valid=True):
        r, out = s2_decode(data, cap)
        if want is not None:
            assert r == len(want) and out == want, (name, r)
        ents.append(dict(name=name, data=bytes(data), cap=cap, code=int(r), out=out, blocks=None, valid=valid, sha=sha(data)))

    srcs = [b"", b"a", _data("twain", 65536, 0), _data("text", 30001, 1), _data("random", 5000, 2), bytes(65536),
            b"ab" * 1000, _data("low", 40000, 3)]
    for better in (False, True):
        for i, (s, c) in enumerate(zip(srcs, enc_blocks(srcs, better))):
            add("s2_%s_%d" % ("better" if better else "fast", i), c, want=s)
    rnd = _data("random", 3000, 4)
    add("s2_stored", s2_varint(3000) + bytes([61 << 2]) + (2999).to_bytes(2, "little") + rnd, want=rnd)
    big = _data("twain", 100000, 0)
    add("s2_over_64k", s2_encode(big, 0), want=big)
    for k in (6, 7):
        add("s2_copy1_%d" % k, s2_copy1_block(k))
        assert ents[-1]["code"] > 0
    base = ents[2]["data"]
    add("s2_trunc", base[:-3], valid=False)
    b = bytearray(base)
    b[len(b) // 2] ^= 0x40
    add("s2_flip", bytes(b), valid=False)
    add("s2_bad_varint", b"\xff\xff\xff\xff\xff\xff", valid=False)
    names = [e["name"] for e in ents]
    assert len(set(names)) == len(names)
    return ents


# ---------------------------------------------------------------------------------------------- layout and checks
def layout(lens, caps, seed):
    """Offsets for n inputs / outputs that take every residue mod 16, with 64-byte gaps between slots.
    Returns (src_off, src_total, dst_off, dst_total) as numpy uint64 arrays / ints."""
    n = len(lens)
    rng = np.random.default_rng(seed)
    r_src = (np.arange(n) * 7 + int(rng.integers(0, 16))) % 16
    r_dst = (np.arange(n) * 11 + int(rng.integers(0, 16))) % 16
    so = np.zeros(n, dtype=np.uint64)
    do = np.zeros(n, dtype=np.uint64)
    s = d = 64
    for i in range(n):
        so[i] = s + int(r_src[i])
        s = (int(so[i]) + lens[i] + 15) // 16 * 16 + 64
        do[i] = d + int(r_dst[i])
        d = (int(do[i]) + caps[i] + 15) // 16 * 16 + 64
    return so, s + 64, do, d + 64


def load_flags():
    with open(FLAGS_PATH) as f:
        return json.load(f)
