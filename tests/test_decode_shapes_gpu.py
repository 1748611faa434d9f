"""The device decoders at the batch shapes that choose their code paths: batch sizes on both sides of every switch of
the staged zstd decoder's form (blocks per input = min(128, 65536 / n) up to 4096 inputs, 4 above), frames with exactly
maxb and maxb + 1 blocks, input and output offsets at every residue mod 16, sentinel bytes around every output slot,
per-input staged flags equal to the emulator's (tests/golden/decode_pool_flags.json, checked by
test_emu_decode_shapes.py), frames cut out of host streams at unaligned offsets, and two streams sharing one context.
Expected results are the oracle decoders' (tests/decode_pool.py)."""
import ctypes

import numpy as np
import pytest
import torch

import decode_pool as DP
import helpers as H

pytestmark = pytest.mark.gpu

SWEEP = (1, 2, 31, 33, 511, 512, 513, 4095, 4096, 4097, 4099, 16397)
PAIRS = {512: (128, 129), 513: (127, 128), 4096: (16, 17), 4097: (4, 5), 4099: (4, 5), 16397: (4, 5)}


@pytest.fixture(scope="module")
def dev(oracle_lib):
    from compress_b200 import s2, zstd
    encs = {lv: zstd.Encoder(level=lv, max_chunks=256) for lv in (1, 2, 3)}
    d = zstd.Decoder()
    c = s2.Codec()
    yield encs, d, c
    for e in encs.values():
        e.close()
    d.close()
    c.close()
    torch.cuda.empty_cache()


@pytest.fixture(scope="module")
def pool(dev):
    encs, _, codec = dev
    enc_frames = lambda inputs: encs[1].encode_frames(inputs)
    zs = DP.build_zstd(lambda level, chunks: encs[level].encode_chunks(chunks), enc_frames)
    s2 = DP.build_s2(lambda blocks, better: codec.encode_blocks(blocks, better=better))
    rec = DP.load_flags()
    sm = DP.small(zs)
    # the device's encoders wrote the same bytes as the emulated ones the recorded flags belong to
    assert {e["name"]: e["sha"] for e in sm} == {k: v["sha"] for k, v in rec["zstd"].items()}
    assert {e["name"]: e["sha"] for e in s2} == {k: v["sha"] for k, v in rec["s2"].items()}
    bnd = DP.frame_mode_boundary(enc_frames, (4, 16, 127, 128))
    return sm, s2, rec, bnd


def _place(datas, caps, seed):
    so, stot, do, dtot = DP.layout([len(d) for d in datas], caps, seed)
    src = np.full(stot, DP.SENT, dtype=np.uint8)
    for i, d in enumerate(datas):
        src[int(so[i]):int(so[i]) + len(d)] = np.frombuffer(d, dtype=np.uint8)
    return (torch.from_numpy(src).cuda(), torch.from_numpy(so.astype(np.int64)).cuda(),
            torch.tensor([len(d) for d in datas], dtype=torch.int32).cuda(), do, dtot)


def _launch(kind, ctx_obj, src, so_t, sizes, do, dtot, cap):
    """One device decode call with per-input offsets on the current stream; returns (dst, out_sizes)."""
    n = sizes.numel()
    dst = torch.full((dtot,), DP.SENT, dtype=torch.uint8, device="cuda")
    do_t = torch.from_numpy(do.astype(np.int64)).cuda()
    if kind == "zstd":
        _, outs = ctx_obj.decode_device(src, sizes, src_offsets=so_t, dst=dst, dst_cap=cap, dst_offsets=do_t)
    else:
        from compress_b200._lib import lib, check
        outs = torch.empty(n, dtype=torch.int64, device="cuda")
        check(lib.b2c_s2_decode_device(ctx_obj._ctx, src.data_ptr(), 0, so_t.data_ptr(), sizes.data_ptr(), dst.data_ptr(), 0,
                                       do_t.data_ptr(), cap, outs.data_ptr(), n,
                                       ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), ctx_obj._ctx)
    # keep the offset tensor alive until the call has run
    dst._keep = do_t
    return dst, outs


def _check(names, wants, cap, do, dst, outs):
    """codes and bytes equal the expected ones; outside [off, off + cap) of every slot -- and, for an input that decodes,
    beyond its output's end -- every byte is still the sentinel."""
    codes = outs.cpu().numpy()
    for i, (nm, (wc, _)) in enumerate(zip(names, wants)):
        assert codes[i] == wc, (i, nm, int(codes[i]), wc)
    uniq, cat, pos = {}, [], 0
    for nm, (wc, wout) in zip(names, wants):
        if wc > 0 and nm not in uniq:
            uniq[nm] = pos
            cat.append(np.frombuffer(wout, dtype=np.uint8))
            pos += len(wout)
    cat_t = torch.from_numpy(np.concatenate(cat) if cat else np.zeros(1, dtype=np.uint8)).cuda()
    exp = torch.full_like(dst, DP.SENT)
    for i, (nm, (wc, _)) in enumerate(zip(names, wants)):
        o = int(do[i])
        if wc > 0:
            exp[o:o + wc].copy_(cat_t[uniq[nm]:uniq[nm] + wc])
        elif wc < 0:
            exp[o:o + cap].copy_(dst[o:o + cap])          # a failed input may leave anything inside its slot
    if not torch.equal(dst, exp):
        bad = int(torch.nonzero(dst != exp)[0])
        i = int(np.searchsorted(do, bad, side="right")) - 1
        raise AssertionError("byte %d differs: slot %d (%s) at offset %d, code %d" % (bad, i, names[max(i, 0)], bad - int(do[max(i, 0)]),
                                                                                   int(codes[max(i, 0)])))


def _tile(members, n, rng):
    reps = -(-n // len(members))
    return [members[i] for i in np.concatenate([rng.permutation(len(members)) for _ in range(reps)])[:n]]


def _zstd_batch(pool, n, seed):
    """n inputs for a sweep batch: the pool's small entries tiled with a seeded permutation, and the frame-mode pair of
    maxb / maxb + 1 blocks for the batch's form.  Returns (names, datas, wants, flags wanted, cap)."""
    sm, _, rec, bnd = pool
    form = DP.maxb_for(n)
    pair = PAIRS.get(n)
    cap, members = DP.POOL_CAP, sm
    if pair and len(bnd[pair[1]][1]) > cap:
        # a larger capacity for the long pair: only inputs whose result and path cannot depend on the capacity go with it
        cap = len(bnd[pair[1]][1])
        members = [e for e in sm if e["valid"] and e["code"] >= 0]
    rng = np.random.default_rng(seed)
    items = [(e["name"], e["data"], (e["code"], e["out"]), rec["zstd"][e["name"]][str(form)]) for e in _tile(members, n, rng)]
    if pair:
        for nb, p in zip(pair, rng.choice(n, 2, replace=False)):
            f, content = bnd[nb]
            items[int(p)] = ("fm_%d_blocks" % nb, f, (len(content), content), int(nb <= form))
    names, datas, wants, flags = zip(*items)
    return list(names), list(datas), list(wants), list(flags), cap


@pytest.mark.parametrize("n", SWEEP)
def test_zstd_batch_sweep(dev, pool, n):
    _, dec, _ = dev
    names, datas, wants, flags, cap = _zstd_batch(pool, n, seed=n)
    src, so_t, sizes, do, dtot = _place(datas, [cap] * n, seed=n)
    dst, outs = _launch("zstd", dec, src, so_t, sizes, do, dtot, cap)
    torch.cuda.synchronize()
    _check(names, wants, cap, do, dst, outs)
    got = dec.staged_flags(n)
    bad = [(i, names[i], int(got[i]), flags[i]) for i in range(n) if int(got[i]) != flags[i]]
    assert not bad, ("maxb", DP.maxb_for(n), bad[:10])
    print("n=%d maxb=%d staged=%d/%d" % (n, DP.maxb_for(n), int(got.sum()), n))


def _s2_stride(codec, datas, cap):
    """S2 block decode of datas laid out at an odd fixed stride (the form of call the staged kernels take); outputs at a
    stride of cap bytes, pre-filled with the sentinel.  Returns (dst, out_sizes, output offsets)."""
    stride = max(len(d) for d in datas) + 13
    src = np.full(len(datas) * stride + 64, DP.SENT, dtype=np.uint8)
    for i, d in enumerate(datas):
        src[i * stride:i * stride + len(d)] = np.frombuffer(d, dtype=np.uint8)
    sizes = torch.tensor([len(d) for d in datas], dtype=torch.int32).cuda()
    dst = torch.full((len(datas), cap), DP.SENT, dtype=torch.uint8, device="cuda")
    _, outs = codec.decode_device(torch.from_numpy(src).cuda(), sizes, stride, dst=dst, dst_cap=cap)
    return dst.view(-1), outs, np.arange(len(datas), dtype=np.uint64) * cap


@pytest.mark.parametrize("n", (1, 33, 4097))
def test_s2_batch_sweep(dev, pool, n):
    _, _, codec = dev
    _, s2, rec, _ = pool
    rng = np.random.default_rng(50 + n)
    ents = _tile(s2, n, rng)
    if n == 1:
        ents = [e for e in s2 if e["name"] == "s2_copy1_6"]
    names = [e["name"] for e in ents]
    wants = [(e["code"], e["out"]) for e in ents]
    # per-block offsets at every residue mod 16: the one-warp kernel alone (the staged walk places its records by the
    # source offsets, whose extent the host does not know)
    src, so_t, sizes, do, dtot = _place([e["data"] for e in ents], [DP.POOL_CAP] * n, seed=n)
    dst, outs = _launch("s2", codec, src, so_t, sizes, do, dtot, DP.POOL_CAP)
    torch.cuda.synchronize()
    _check(names, wants, DP.POOL_CAP, do, dst, outs)
    assert not codec.staged_flags(n).any()
    # the same blocks at a fixed stride: the staged kernels take exactly the blocks the emulated ones take
    dst, outs, do = _s2_stride(codec, [e["data"] for e in ents], DP.POOL_CAP)
    torch.cuda.synchronize()
    _check(names, wants, DP.POOL_CAP, do, dst, outs)
    got = codec.staged_flags(n)
    assert [int(x) for x in got] == [rec["s2"][nm]["flag"] for nm in names]
    print("s2 n=%d staged=%d/%d" % (n, int(got.sum()), n))
    if n > 1:        # recCap is exact: the block at the bound is staged, one element more is not
        assert {(nm, int(f)) for nm, f in zip(names, got) if nm.startswith("s2_copy1_")} == {("s2_copy1_6", 1), ("s2_copy1_7", 0)}


def _odd_stream(enc, rng, nframes, seed):
    """A stream of nframes level-2 frames of odd content sizes (1 .. 70 000 bytes) with skippable frames mixed in.
    Returns (stream, content, frames, where each frame starts in the stream)."""
    sizes = rng.integers(0, 1000, nframes) * 2 + 1
    big = rng.integers(0, 8, nframes) == 0
    sizes[big] = rng.integers(0, 35000, int(big.sum())) * 2 + 1
    data = H.synth_text(int(sizes.sum()), seed=seed)
    cuts = np.concatenate([[0], np.cumsum(sizes)])
    frames = enc.encode_chunks([data[cuts[i]:cuts[i + 1]] for i in range(nframes)])
    parts, starts, pos = [], [], 0
    for i, f in enumerate(frames):
        starts.append(pos)
        parts.append(f)
        pos += len(f)
        if i % 997 == 500:
            parts.append(DP.skippable(b"s" * (i % 13)))
            pos += len(parts[-1])
    return b"".join(parts), data, frames, starts


def test_host_split_frames(dev, oracle_lib):
    encs, dec, _ = dev
    rng = np.random.default_rng(77)
    stream, data, frames, _ = _odd_stream(encs[2], rng, 4200, seed=78)
    assert dec.DecodeAll(stream, size_hint=len(data)) == data
    assert dec.staged_count(len(frames)) > len(frames) // 4     # one input per frame, in the per-input form
    r, back = H.oracle_decode(stream, len(data))
    assert r == len(data) and back == data
    # several streams in one call; the largest frame of one of them gets a flipped byte in the middle of its payload
    streams, datas = [], []
    for k in range(4):
        s, d, fr, starts = _odd_stream(encs[2], rng, 1100, seed=80 + k)
        if k == 2:
            j = int(np.argmax([len(f) for f in fr]))
            bad = bytearray(s)
            bad[starts[j] + len(fr[j]) // 2] ^= 0x21
            s = bytes(bad)
        streams.append(s)
        datas.append(d)
    caps = [len(d) for d in datas]
    outs, codes = dec.decode_chunks(streams, caps)
    for i in (0, 1, 3):
        assert codes[i] == len(datas[i]) and outs[i] == datas[i], i
    ro, _ = H.oracle_decode(streams[2], caps[2])
    assert ro < 0 and codes[2] == ro, (ro, codes[2])


def _long_batch(enc, n, seed):
    rng = np.random.default_rng(seed)
    base = H.synth_text(8 << 20, seed=seed)
    datas = []
    for _ in range(n):
        ln = int(rng.integers(5 * DP.FB, 9 * DP.FB))
        o = int(rng.integers(0, len(base) - ln))
        datas.append(base[o:o + ln])
    return enc.encode_frames(datas), datas


def test_two_streams_one_context(dev, pool):
    encs, dec, codec = dev
    a = _zstd_batch(pool, 4099, seed=1)
    c = _zstd_batch(pool, 4099, seed=2)
    capL = 9 * DP.FB
    bf, bd = _long_batch(encs[1], 300, 3)
    df, dd = _long_batch(encs[1], 300, 4)
    batches = []
    for names, datas, wants, _, cap in (a, c):
        batches.append((datas, cap, [w[0] for w in wants]))
    batches = [batches[0], (bf, capL, [len(x) for x in bd]), batches[1], (df, capL, [len(x) for x in dd])]
    placed = [_place(d, [cap] * len(d), seed=10 + i) for i, (d, cap, _) in enumerate(batches)]
    # each batch alone (this also grows the context's scratch to its largest size, so no allocation happens below)
    alone = []
    for (d, cap, want), (src, so_t, sizes, do, dtot) in zip(batches, placed):
        dst, outs = _launch("zstd", dec, src, so_t, sizes, do, dtot, cap)
        torch.cuda.synchronize()
        assert outs.cpu().tolist() == want
        alone.append((dst, outs))
    assert dec.staged_count(300) == 300
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    res = []
    for i, ((d, cap, _), (src, so_t, sizes, do, dtot)) in enumerate(zip(batches, placed)):
        with torch.cuda.stream(s1 if i % 2 == 0 else s2):
            res.append(_launch("zstd", dec, src, so_t, sizes, do, dtot, cap))
    torch.cuda.synchronize()
    for i, ((dst, outs), (dst0, outs0)) in enumerate(zip(res, alone)):
        assert torch.equal(outs, outs0) and torch.equal(dst, dst0), "batch %d" % i
    # the same with S2 block decode on one codec context (fixed strides: the staged kernels' form of call)
    _, s2p, _, _ = pool
    sb = [_tile(s2p, n, np.random.default_rng(90 + n)) for n in (4099, 300, 4097, 301)]
    alone = []
    for ents in sb:
        dst, outs, do = _s2_stride(codec, [e["data"] for e in ents], DP.POOL_CAP)
        torch.cuda.synchronize()
        _check([e["name"] for e in ents], [(e["code"], e["out"]) for e in ents], DP.POOL_CAP, do, dst, outs)
        assert codec.staged_flags(len(ents)).sum() > len(ents) // 2
        alone.append((dst, outs))
    torch.cuda.synchronize()
    res = []
    for i, ents in enumerate(sb):
        with torch.cuda.stream(s1 if i % 2 == 0 else s2):
            res.append(_s2_stride(codec, [e["data"] for e in ents], DP.POOL_CAP)[:2])
    torch.cuda.synchronize()
    for i, ((dst, outs), (dst0, outs0)) in enumerate(zip(res, alone)):
        assert torch.equal(outs, outs0) and torch.equal(dst, dst0), "s2 batch %d" % i
