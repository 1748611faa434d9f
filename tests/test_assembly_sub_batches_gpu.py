"""GPU tests of the two calls that assemble one output from blocks encoded in sub-batches, at sizes that take several:
zstd frame mode (b2c_zstd_encode_frames_device: 8 192 blocks of 48 KiB per sub-batch at level 1, 4 096 of 96 KiB at levels
2 and 3) and S2 / Snappy streams (b2c_s2_encode_stream_device: 4 096 blocks per sub-batch).  Every sub-batch is encoded into
slots shared by all of them and placed at the running base of the earlier ones; a frame or a run of chunks can begin in one
sub-batch and end in the next.

Calls of fewer blocks than one sub-batch are tied to the emulated kernels, and through them to the oracle, by
test_frames_gpu.py and test_s2_stream_gpu.py.  Two exact invariants tie the large calls to such small calls:

- frame mode: a block depends only on its bytes, its history and its last flag, so block i >= 1 of the frame of
  D[b*B : e*B] equals block b + i of the frame of D (the slice's last block excepted, unless e is the end of D);
- streams: a stream is the identifier followed by one chunk per block, so for X a multiple of the block size
  stream(D) == identifier + stream(D[:X])[10:] + stream(D[X:])[10:].

The launch count of every large call shows how many sub-batches it ran: a call adds a fixed number of launches plus the
same number again for each sub-batch, both measured on calls of one and of two sub-batches."""
import gc

import numpy as np
import pytest
import torch

import helpers as H
import s2_stream_ref as R
from test_emu_frames import split_blocks
from test_oracle_s2 import s2_decode as orc_s2_decode

pytestmark = pytest.mark.gpu

FRAME_BLOCK = {1: 49152, 2: 98304, 3: 98304}       # frame-mode block size per level (b2c_frame.cuh)
FRAME_SUB = {1: 8192, 2: 4096, 3: 4096}            # blocks per frame-mode sub-batch (384 MiB of input)
WINDOW = {1: 4 << 20, 2: 8 << 20, 3: 8 << 20}      # frames longer than this carry a window byte, no single-segment flag
STREAM_SUB = 4096                                  # blocks per stream sub-batch
ERR_DST_SMALL = -4
SENTINEL = 0xA5


def _free():
    torch.cuda.synchronize()
    gc.collect()
    torch.cuda.empty_cache()


def _cdiv(a, b):
    return -(-a // b)


def _nblocks(size, block):
    return max(1, _cdiv(size, block))


def _boundary_text(n, block, bounds, seed):
    """n bytes of synthetic text on the device with zero runs and noise: every 53rd block carries a zero run, every 71st a
    stretch of noise, and around the j-th boundary `bd` of `bounds` blocks (bd - 1, bd) are (noise, zeros) for even j and
    (zeros, noise) for odd j.  In a zstd frame that puts raw, RLE and compressed blocks side by side at the boundary; in a
    stream, an uncompressed chunk next to compressed ones."""
    src = H.synth_text_torch(n, "cuda", seed=seed)
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    nblk = _cdiv(n, block)
    z0, zn, r0, rn = block // 8, block // 16, block // 2, block // 12
    for b in range(5, nblk - 1, 53):
        src[b * block + z0:b * block + z0 + zn] = 0
    for b in range(11, nblk - 1, 71):
        src[b * block + r0:b * block + r0 + rn] = torch.randint(0, 256, (rn,), generator=g, device="cuda", dtype=torch.uint8)
    for j, bd in enumerate(bounds):
        noise, zeros = (bd - 1, bd) if j % 2 == 0 else (bd, bd - 1)
        src[noise * block:(noise + 1) * block] = torch.randint(0, 256, (block,), generator=g, device="cuda", dtype=torch.uint8)
        src[zeros * block:(zeros + 1) * block] = 0
    return src


# ------------------------------------------------------------------------------------------------------------ zstd frames
def _hdr_len(buf, at=0):
    """Bytes of the frame header at buf[at:] (RFC 8878 3.1.1.1: descriptor, window byte, dictionary id, content size)."""
    d = int(buf[at + 4])
    single = (d >> 5) & 1
    return 5 + (0 if single else 1) + (0, 1, 2, 4)[d & 3] + ((1 if single else 0), 2, 4, 8)[d >> 6]


_oracle_headers = {}


def _oracle_header(size, level, crc=True):
    """The oracle's frame header for an input of `size` bytes (it depends only on the length, the level and the checksum)."""
    key = (size, level, crc)
    if key not in _oracle_headers:
        r, fr = H.oracle_encode(bytes(size), level, crc)
        assert r > 0
        _oracle_headers[key] = fr[:_hdr_len(fr)]
    return _oracle_headers[key]


def _libzstd_into(frame, out):
    """libzstd's ZSTD_decompress of the numpy frame into the numpy buffer `out`: bytes written, or -1."""
    Z = H.libzstd()
    frame = np.ascontiguousarray(frame)
    r = Z.ZSTD_decompress(out.ctypes.data, out.size, frame.ctypes.data, frame.size)
    return -1 if Z.ZSTD_isError(r) else int(r)


def _fetch(dst, foff, fsz):
    """(output bytes up to the end of the last frame, frame offsets, frame sizes) on the host."""
    torch.cuda.synchronize()
    fo, fz = foff.cpu().numpy().astype(np.int64), fsz.cpu().numpy()
    end = int((fo + np.maximum(fz, 0)).max()) if len(fz) else 0
    return dst[:end].cpu().numpy(), fo, fz


def _frame_launch_model(enc, src):
    """(launches of a frame-mode call of one sub-batch, launches each further sub-batch adds) on this encoder, from calls
    of 16 and of one sub-batch + 1 one-byte frames."""
    counts = []
    for nframes in (16, FRAME_SUB[enc.level] + 1):
        before = enc.launches
        enc.encode_frames_device(src, [0] * nframes, [1] * nframes)
        counts.append(enc.launches - before)
    torch.cuda.synchronize()
    one, two = counts
    assert two > one > 0
    return one, two - one


def _encode_frames_counted(enc, src, offsets, sizes, dst=None):
    """encode_frames_device, checking by the launch count that it ran as many sub-batches as its blocks need."""
    one, per = _frame_launch_model(enc, src)
    nblk = sum(_nblocks(int(s), FRAME_BLOCK[enc.level]) for s in sizes)
    nsub = _cdiv(nblk, FRAME_SUB[enc.level])
    before = enc.launches
    res = enc.encode_frames_device(src, offsets, sizes, dst=dst)
    assert enc.launches - before == one + (nsub - 1) * per, f"{nblk} blocks: expected {nsub} sub-batches"
    return res, nsub


def _encoder(level, crc=True):
    from compress_b200 import zstd
    return zstd.Encoder(level=level, crc=crc)


@pytest.mark.parametrize("level", [1, 2, 3])
def test_one_gib_frame_across_sub_batches(level):
    """One 1 GiB frame: three sub-batches (8 192 + 8 192 + 5 462 blocks at level 1, 4 096 + 4 096 + 2 731 above).  libzstd
    decodes it (XXH64 included), its header is the oracle's, only its final block is last, and every block equals the
    same block of slice frames encoded in calls of at most 2 000 blocks."""
    n, B, sub = 1 << 30, FRAME_BLOCK[level], FRAME_SUB[level]
    nblk = _cdiv(n, B)
    bounds = [sub, 2 * sub]
    src = _boundary_text(n, B, bounds, seed=100 + level)
    enc = _encoder(level)
    (dst, foff, fsz), nsub = _encode_frames_counted(enc, src, [0], [n])
    assert nsub == 3
    out, fo, fz = _fetch(dst, foff, fsz)
    del dst
    assert fo[0] == 0 and fz[0] == len(out)
    host = src.cpu().numpy()
    back = np.empty(n, dtype=np.uint8)
    assert _libzstd_into(out, back) == n and np.array_equal(back, host), f"level {level}: libzstd does not give the input back"
    del back, host
    hdr = _oracle_header(n, level)
    assert bytes(out[:len(hdr)]) == hdr
    full = split_blocks(memoryview(out), len(hdr), True)
    assert len(full) == nblk
    assert [blk[0] for blk in full[:-1]].count(1) == 0 and full[-1][0] == 1, "only the final block is last"
    # raw (0), RLE (1) and compressed (2) blocks meet at both boundaries
    got = [[full[bd + d][1] for d in (-2, -1, 0, 1)] for bd in bounds]
    assert got == [[2, 0, 1, 2], [2, 1, 0, 2]], got
    # slice frames of at most 2 000 blocks, each starting two blocks before the previous one ends: every block of the
    # frame is an interior block of a slice (block 0 and the final block: of the first and the last slice)
    b = 0
    while True:
        e = min(b + 2000, nblk)
        size = min(e * B, n) - b * B
        sd, sfo, sfz = enc.encode_frames_device(src, [b * B], [size])
        sout, _, _ = _fetch(sd, sfo, sfz)
        del sd
        sblk = split_blocks(memoryview(sout), _hdr_len(sout), True)
        assert len(sblk) == e - b
        lo, hi = (1 if b else 0), (e - b if e == nblk else e - b - 1)
        for i in range(lo, hi):
            assert sblk[i][3] == full[b + i][3], (
                f"level {level}: block {b + i} of the 1 GiB frame differs from block {i} of the frame of blocks [{b}, {e})")
        if e == nblk:
            break
        b = e - 2
    enc.close()
    del src, out, full, sblk, sout
    _free()


def _mixed_sizes(level, seed):
    """Frame sizes of a mixed batch of more than two sub-batches of blocks, and the (frame, boundary) pairs of the frames
    placed to start just before a sub-batch boundary and end three blocks after it."""
    B, sub, W = FRAME_BLOCK[level], FRAME_SUB[level], WINDOW[level]
    rng = np.random.default_rng(seed)
    specials = [0, 1, 255, 256, 1024, 1025, 65791, 65792, B - 1, B, B + 1, 2 * B, 7 * B, W - 1, W, W + 1]
    sizes, straddlers, nblk, k = [], [], 0, 1
    while nblk < 2 * sub + sub // 8 or specials:
        while k * sub <= nblk:
            k += 1
        bd = k * sub
        if bd - 40 <= nblk:
            s = (bd - nblk + 3) * B - int(rng.integers(0, B))
            straddlers.append((len(sizes), bd))
            k += 1
        elif specials and rng.random() < 0.01:
            s = specials.pop(int(rng.integers(0, len(specials))))
        else:
            u = rng.random()
            s = (int(rng.integers(0, 2000)) if u < 0.75 else
                 int(rng.integers(1, 2 * B)) if u < 0.95 else int(rng.integers(2 * B, 16 * B)))
        sizes.append(s)
        nblk += _nblocks(s, B)
    return np.array(sizes, dtype=np.int64), straddlers


class _Mixed:
    """A batch of frames of mixed sizes at one level, more than two sub-batches of blocks, and its frame-mode encoding in
    one call.  The sizes include 0, 1, 255, 256, 1 024, 1 025, 65 791, 65 792, B - 1, B, B + 1, multiples of B, the window
    and the window + 1; before every sub-batch boundary a multi-block frame starts that ends after it.  Frames sit at
    16-byte aligned offsets of one device buffer."""

    def __init__(self, level, seed):
        B = FRAME_BLOCK[level]
        self.level = level
        self.sizes, self.straddlers = _mixed_sizes(level, seed)
        nb = np.array([_nblocks(int(s), B) for s in self.sizes], dtype=np.int64)
        self.nblk = int(nb.sum())
        self.first_block = np.cumsum(nb) - nb
        self.offsets = np.concatenate([[0], np.cumsum((self.sizes + 15) & ~15)[:-1]]).astype(np.int64)
        self.total = int(self.offsets[-1] + self.sizes[-1])
        self.src = _boundary_text(self.total, B, [], seed=seed)
        enc = _encoder(level)
        (dst, foff, fsz), self.nsub = _encode_frames_counted(enc, self.src, self.offsets, self.sizes)
        self.out, self.fo, self.fz = _fetch(dst, foff, fsz)
        enc.close()


@pytest.fixture(scope="module")
def mixed():
    """_Mixed batches by level; one kept at a time."""
    cache = {}

    def get(level):
        if level not in cache:
            cache.clear()
            _free()
            cache[level] = _Mixed(level, seed=200 + level)
        return cache[level]
    yield get
    cache.clear()
    _free()


@pytest.mark.parametrize("level", [2, 1])
def test_mixed_batch_across_sub_batches(mixed, level):
    """Thousands of frames of mixed sizes in one call of three or more sub-batches: every frame equals the same frame
    encoded in small calls, decodes with libzstd and with the library's decoder, has the oracle's header (single segment
    up to the window, a window byte above), and the frames are back to back."""
    from compress_b200 import zstd
    M = mixed(level)
    sub = FRAME_SUB[level]
    assert M.nsub >= 3
    assert len(M.straddlers) >= 2 and all(
        M.first_block[f] < bd < M.first_block[f] + _nblocks(int(M.sizes[f]), FRAME_BLOCK[level])
        for f, bd in M.straddlers), "multi-block frames cross the sub-batch boundaries"
    fo, fz, out, sizes = M.fo, M.fz, M.out, M.sizes
    assert (fz > 0).all()
    assert fo[0] == 0 and np.array_equal(fo[1:], np.cumsum(fz)[:-1]), "frames are written back to back"
    # the same frames in small calls (at most 300 frames, fewer blocks than one sub-batch): identical bytes
    enc = _encoder(level)
    i0 = 0
    while i0 < len(sizes):
        i1, blocks = i0, 0
        while i1 < len(sizes) and i1 - i0 < 300 and blocks + _nblocks(int(sizes[i1]), FRAME_BLOCK[level]) < sub:
            blocks += _nblocks(int(sizes[i1]), FRAME_BLOCK[level])
            i1 += 1
        gd, gfo, gfz = enc.encode_frames_device(M.src, M.offsets[i0:i1], sizes[i0:i1])
        gout, gfo, gfz = _fetch(gd, gfo, gfz)
        del gd
        assert (np.array_equal(gfz, fz[i0:i1]) and np.array_equal(gfo, fo[i0:i1] - fo[i0])
                and np.array_equal(gout, out[fo[i0]:fo[i1 - 1] + fz[i1 - 1]])), (
            f"level {level}: frames [{i0}, {i1}) differ from the same frames encoded in a call of their own")
        i0 = i1
    enc.close()
    # libzstd and the oracle's headers
    host = M.src.cpu().numpy()
    buf = np.empty(int(sizes.max()) + 1, dtype=np.uint8)
    for f in range(len(sizes)):
        s, o, fr = int(sizes[f]), int(M.offsets[f]), out[fo[f]:fo[f] + fz[f]]
        assert _libzstd_into(fr, buf) == s and np.array_equal(buf[:s], host[o:o + s]), f"level {level} frame {f} ({s} B)"
        hdr = _oracle_header(s, level)
        assert bytes(fr[:len(hdr)]) == hdr, f"level {level} frame {f} ({s} B): header differs from the oracle's"
    # the library's own decoder
    d = zstd.Decoder()
    back, codes = d.decode_chunks([out[fo[f]:fo[f] + fz[f]] for f in range(len(sizes))], [int(s) + 16 for s in sizes])
    d.close()
    for f in range(len(sizes)):
        o, s = int(M.offsets[f]), int(sizes[f])
        assert codes[f] == s and np.array_equal(np.frombuffer(back[f], dtype=np.uint8), host[o:o + s]), (
            f"level {level} frame {f}: Decoder.decode_chunks gives {codes[f]}")
    _free()


@pytest.mark.parametrize("shift", [1, 8, 13])
def test_mixed_batch_at_unaligned_offsets(mixed, shift):
    """The level-1 batch (frames that cross sub-batch boundaries, frames longer than the window) moved by 1, 8 and 13 bytes
    in device memory: the output is byte-identical to the aligned call's."""
    M = mixed(1)
    src = torch.empty(M.total + 16, dtype=torch.uint8, device="cuda")
    src[shift:shift + M.total] = M.src[:M.total]
    enc = _encoder(1)
    (dst, foff, fsz), _ = _encode_frames_counted(enc, src, M.offsets + shift, M.sizes)
    out, fo, fz = _fetch(dst, foff, fsz)
    enc.close()
    assert np.array_equal(fz, M.fz) and np.array_equal(fo, M.fo) and np.array_equal(out, M.out), f"source offset +{shift}"
    del src, dst
    _free()


def test_mixed_batch_without_checksum(mixed):
    """Encoder(crc=False) on the level-1 batch: the checksum flag is clear, no frame has a trailer, and the rest is the
    checksummed frames' bytes."""
    M = mixed(1)
    enc = _encoder(1, crc=False)
    (dst, foff, fsz), _ = _encode_frames_counted(enc, M.src, M.offsets, M.sizes)
    out, fo, fz = _fetch(dst, foff, fsz)
    enc.close()
    has_crc = M.sizes > 0                   # (an empty frame has no checksum either way)
    assert (M.out[M.fo[has_crc] + 4] & 4 == 4).all() and (out[fo + 4] & 4 == 0).all()
    assert np.array_equal(fz, M.fz - 4 * has_crc)
    # the checksummed output with the flag cleared and the trailers cut out
    want = M.out.copy()
    want[M.fo + 4] &= 0xFB
    keep = np.ones(len(want), dtype=bool)
    keep[((M.fo + M.fz - 4)[has_crc][:, None] + np.arange(4)).ravel()] = False
    assert np.array_equal(out, want[keep])
    host = M.src.cpu().numpy()
    for f in [int(np.argmax(M.sizes))] + [f for f, _ in M.straddlers]:
        s, o = int(M.sizes[f]), int(M.offsets[f])
        buf = np.empty(s, dtype=np.uint8)
        assert _libzstd_into(out[fo[f]:fo[f] + fz[f]], buf) == s and np.array_equal(buf, host[o:o + s])
        assert bytes(out[fo[f]:fo[f] + _hdr_len(out, fo[f])]) == _oracle_header(s, 1, crc=False)
    _free()


def test_mixed_batch_destination_too_small(mixed):
    """A destination that ends inside a frame of the second sub-batch: the frames before it are those of the full-capacity
    call, every later frame reports B2C_ERR_DST_SMALL, and no byte past the capacity changes."""
    M = mixed(1)
    sub, B = FRAME_SUB[1], FRAME_BLOCK[1]
    nb = np.array([_nblocks(int(s), B) for s in M.sizes])
    cand = np.nonzero((nb >= 4) & (M.first_block >= sub + 64) & (M.first_block + nb <= 2 * sub))[0]
    assert len(cand)
    f = int(cand[0])
    cap = int(M.fo[f] + M.fz[f] // 2)
    big = torch.full((len(M.out) + 4096,), SENTINEL, dtype=torch.uint8, device="cuda")
    enc = _encoder(1)
    (_, foff, fsz), _ = _encode_frames_counted(enc, M.src, M.offsets, M.sizes, dst=big[:cap])
    torch.cuda.synchronize()
    enc.close()
    fo, fz, got = foff.cpu().numpy().astype(np.int64), fsz.cpu().numpy(), big.cpu().numpy()
    assert np.array_equal(fz[:f], M.fz[:f]) and np.array_equal(fo[:f], M.fo[:f])
    assert (fz[f:] == ERR_DST_SMALL).all(), np.unique(fz[f:])
    assert np.array_equal(got[:M.fo[f]], M.out[:M.fo[f]])
    assert (got[cap:] == SENTINEL).all(), "bytes past the capacity were written"
    del big
    _free()


# ------------------------------------------------------------------------------------------------------------ S2 streams
S2_MODES = {"fast": {}, "better": {"better": True}, "best": {"best": True}, "snappy": {"snappy": True}}


def _stream(codec, src, block, mode, dst=None):
    d, total, err = codec.encode_stream_device(src, block_size=block, dst=dst, **S2_MODES[mode])
    torch.cuda.synchronize()
    return d, int(total.cpu().numpy()[0]), int(err.cpu().numpy()[0])


def _stream_counted(codec, src, block, mode, dst=None):
    """encode_stream_device, checking by the launch count that it ran as many sub-batches as its blocks need."""
    counts = []
    for nb in (16, STREAM_SUB + 1):
        before = codec.launches
        _stream(codec, src[:nb * block], block, mode)
        counts.append(codec.launches - before)
    one, per = counts[0], counts[1] - counts[0]
    assert per > 0 and one > 0
    nsub = _cdiv(_cdiv(src.numel(), block), STREAM_SUB)
    before = codec.launches
    res = _stream(codec, src, block, mode, dst=dst)
    assert codec.launches - before == one + (nsub - 1) * per, f"expected {nsub} sub-batches"
    return res, nsub


def _chunk_offsets(st):
    """Start of every chunk after the identifier, and the stream's end."""
    offs, o, n = [], 10, len(st)
    while o < n:
        offs.append(o)
        b = bytes(st[o:o + 4])
        o += 4 + (b[1] | b[2] << 8 | b[3] << 16)
    assert o == n
    return offs + [n]


def _orc_decode_block(body, n):
    r, out = orc_s2_decode(body, n)
    return out if r == n else None


@pytest.mark.parametrize("mode,block,mib", [("fast", 4096, 40), ("better", 4096, 40), ("best", 4096, 40),
                                            ("snappy", 4096, 40), ("fast", 65536, 600)])
def test_stream_across_sub_batches(mode, block, mib):
    """A stream of three sub-batches (4 KiB blocks over 40 MiB, 64 KiB blocks over 600 MiB, each with a ragged tail) equals
    the identifier and the chunks of streams of at most 3 000 blocks; it decodes, the reference-format reader reads the
    chunks around every boundary, and at 40 MiB the host-buffer call gives the same bytes."""
    from compress_b200 import s2
    n = (mib << 20) + 1234
    nblk = _cdiv(n, block)
    bounds = list(range(STREAM_SUB, nblk, STREAM_SUB))
    src = _boundary_text(n, block, bounds, seed=300 + block // 4096)
    codec = s2.Codec()
    (dst, total, err), nsub = _stream_counted(codec, src, block, mode)
    assert nsub == 3 and err == 0
    magic = R.MAGIC_SNAPPY if mode == "snappy" else R.MAGIC_S2
    assert bytes(dst[:10].cpu().numpy()) == magic
    # the concatenation of the streams of pieces of 3 000 blocks, compared on the device
    pos = 10
    for a in range(0, nblk, 3000):
        b = min(a + 3000, nblk)
        pd, pt, pe = _stream(codec, src[a * block:min(b * block, n)], block, mode)
        assert pe == 0
        assert torch.equal(dst[pos:pos + pt - 10], pd[10:pt]), f"{mode}: chunks of blocks [{a}, {b}) differ"
        pos += pt - 10
        del pd
    assert total == pos
    st, host = dst[:total].cpu().numpy(), src.cpu().numpy()
    del dst
    back = codec.DecodeStream(st, max_size=n)
    assert len(back) == n and np.array_equal(np.frombuffer(back, dtype=np.uint8), host)
    del back
    # the reference-format reader on the chunks around each boundary, the first and the last
    offs = _chunk_offsets(st)
    assert len(offs) == nblk + 1
    for bd in [2] + bounds + [nblk]:
        a, b = bd - 2, min(bd + 2, nblk)
        piece = magic + st[offs[a]:offs[b]].tobytes()
        assert R.read_stream(piece, _orc_decode_block) == host[a * block:min(b * block, n)].tobytes(), f"{mode}: chunks [{a}, {b})"
    for bd in bounds:       # an uncompressed and a compressed chunk meet at the boundary
        assert sorted([int(st[offs[bd - 1]]), int(st[offs[bd]])]) == [0, 1]
    if mib <= 40:
        kw = S2_MODES[mode]
        assert np.array_equal(np.frombuffer(codec.EncodeStream(host.tobytes(), block_size=block, **kw), dtype=np.uint8), st)
    codec.close()
    del src
    _free()


def test_stream_destination_too_small():
    """A destination that ends inside a chunk of the second sub-batch: the error is B2C_ERR_DST_SMALL, the chunks before
    the cut are those of the full stream, and no byte past the capacity changes."""
    from compress_b200 import s2
    block, n = 4096, (40 << 20) + 1234
    nblk = _cdiv(n, block)
    src = _boundary_text(n, block, list(range(STREAM_SUB, nblk, STREAM_SUB)), seed=400)
    codec = s2.Codec()
    full, total, err = _stream(codec, src, block, "fast")
    assert err == 0
    st = full[:total].cpu().numpy()
    del full
    offs = _chunk_offsets(st)
    cut = STREAM_SUB + 1000
    cap = offs[cut] + 7
    big = torch.full((total + 4096,), SENTINEL, dtype=torch.uint8, device="cuda")
    (_, _, err), nsub = _stream_counted(codec, src, block, "fast", dst=big[:cap])
    assert nsub == 3 and err == ERR_DST_SMALL
    got = big.cpu().numpy()
    assert np.array_equal(got[:offs[cut]], st[:offs[cut]])
    assert (got[cap:] == SENTINEL).all(), "bytes past the capacity were written"
    codec.close()
    del src, big
    _free()
