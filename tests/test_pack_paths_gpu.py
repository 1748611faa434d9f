"""GPU tests for the code paths of the zstd pack kernel (K4): literals staged in shared memory by a bulk copy or read
from global memory when there are more than fit, sequence groups of eight with ragged ends, empty and tiny sequence
sections, raw / RLE blocks and raw literals beside sequences, u16 (64 KiB) and u32 (128 KiB) length arrays.  Every frame
is checked against the oracle's blockEnc.encode for the device's parse, decoded with libzstd, and compared byte for
byte with the SIMT-emulated build of the same kernels (which stages literals with plain loads) in both lane orders."""
import numpy as np
import pytest
import torch

import helpers as H
from check_util import check_frames
from emu_util import emu_encode

pytestmark = pytest.mark.gpu

LIT_SMEM = 40 * 1024   # literal bytes K4 stages in shared memory for 64 KiB blocks


def _chunks(B, seed):
    rng = np.random.Generator(np.random.PCG64(seed))
    tw = H.golden("twain.txt")

    def alpha(n, k):   # n random bytes over k symbols: few matches, literals Huffman-compressible when k < 256
        return rng.integers(0, k, n, dtype=np.uint8).tobytes()

    out = []
    # more literals than shared memory holds (compressed literals, a handful of sequences)
    big = alpha(B - 4096, 128)
    out.append(big + big[1000:1000 + 4096])
    out.append(alpha(B, 112))
    # 0 (the parse stores such a chunk raw), 1 and 2 sequences beside compressible literals
    r = alpha(1500, 96)
    out.append(r)
    out.append(r + r[100:160])
    out.append(r + r[100:160] + alpha(500, 96) + r[1000:1050])
    # sequence counts of every residue mod 8: text prefixes of growing length
    for k in range(24):
        out.append(tw[5000:5000 + 700 + 97 * k])
    # raw literals beside sequences, a raw block, RLE blocks, a chunk of one repeated short unit
    noise = alpha(20000, 256)
    out.append(noise + noise[:3000] + alpha(10000, 256) + noise[5000:9000])
    out.append(alpha(B, 256))
    out.append(bytes(B))
    out.append(b"\x07" * 777)
    out.append((b"a" * 30 + alpha(1, 256)) * 500)
    # full-size text: many sequences, literals in shared memory
    out.append(tw[:B])
    out.append(H.synth_text(B, seed))
    return out


@pytest.mark.parametrize("level", [1, 2])
def test_pack_paths(level, emu_lib):
    from compress_b200 import zstd
    enc = zstd.Encoder(level=level, max_chunks=64)
    try:
        B = enc.block
        chunks = _chunks(B, 17 + level)
        n = len(chunks)
        src = torch.zeros(n * B, dtype=torch.uint8)
        sizes = torch.zeros(n, dtype=torch.int32)
        for i, c in enumerate(chunks):
            if c:
                src[i * B:i * B + len(c)] = torch.frombuffer(bytearray(c), dtype=torch.uint8)
            sizes[i] = len(c)
        dst, outs, hdr, seqs, lits = enc.encode_device_debug(src.cuda(), sizes.cuda())
        torch.cuda.synchronize()
        outs = outs.cpu().numpy()
        assert (outs > 0).all(), outs
        frames = [bytes(dst[i, :int(outs[i])].cpu().numpy()) for i in range(n)]
        hdr = hdr.cpu().numpy()
        check_frames(chunks, frames, hdr, seqs.cpu().numpy(), lits.cpu().numpy(), label="pack-L%d" % level, level=level)
        for desc in (0, 1):
            assert emu_encode(emu_lib, chunks, level=level, desc=desc)[0] == frames, "lane order %d" % desc
    finally:
        enc.close()
    # the chunks reach the paths they are meant for (hdr: nseq, nlit, kind 0 compressed / 1 raw / 2 RLE, literal mode)
    comp = hdr[hdr[:, 2] == 0]
    if level == 1:
        assert (comp[:, 1] > LIT_SMEM).any(), "no compressed block with literals beyond shared memory"
    assert {1, 2} <= set(comp[:, 0].tolist()), sorted(set(comp[:, 0].tolist()))[:8]
    assert set((comp[:, 0] % 8).tolist()) == set(range(8))
    assert ((comp[:, 3] == 0) & (comp[:, 0] > 0)).any(), "no raw literals beside sequences"
    assert (comp[:, 3] == 2).any()
    assert (hdr[:, 2] == 1).any() and (hdr[:, 2] == 2).any(), "raw and RLE blocks"
