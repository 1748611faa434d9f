"""One device-resident call covers a 1 GiB batch in a single pass of the encode pipeline: 16384 x 64 KiB chunks at
level 1, 8192 x 128 KiB blocks at levels 2 and 3.  A call of one full pass + 3 chunks (the remainder starts at the
second pass's first chunk) must produce exactly the frames that calls of at most half a pass produce for the same
chunks.  Run on an H100: python -m pytest tests -m gpu."""
import pytest
import torch

import helpers as H

pytestmark = pytest.mark.gpu

LAUNCHES_PER_PASS = 5      # parse, hist, tables, chains (XXH64 fused), pack


@pytest.mark.parametrize("level", [1, 2])
def test_full_pass_plus_remainder_matches_smaller_calls(level):
    from compress_b200 import zstd
    chunk = 65536 if level == 1 else 131072
    npass = (1 << 30) // chunk
    n = npass + 3
    half = npass // 2
    dev = torch.device("cuda", 0)
    src = H.synth_text_torch(n * chunk, dev, seed=2024 + level)
    # chunk sizes vary (full, short, tiny, empty) so that frames differ from chunk to chunk, the remainder included
    idx = torch.arange(n, device=dev, dtype=torch.int64)
    sizes = torch.where(idx % 7 == 0, torch.full_like(idx, chunk), chunk - (idx * 977) % 60000)
    sizes[5] = 0
    sizes[n - 2] = 1
    sizes[n - 1] = 4097
    sizes = sizes.to(torch.int32)
    enc = zstd.Encoder(level=level, max_chunks=64)
    try:
        l0 = enc.launches
        dst1, out1 = enc.encode_device(src, sizes=sizes)
        torch.cuda.synchronize()
        assert enc.launches - l0 == 2 * LAUNCHES_PER_PASS       # one full pass, then the remainder
        dst2 = torch.empty_like(dst1)
        out2 = torch.empty_like(out1)
        for c0 in range(0, n, half):
            c1 = min(c0 + half, n)
            enc.encode_device(src[c0 * chunk:c1 * chunk], sizes=sizes[c0:c1], dst=dst2[c0:c1], out_sizes=out2[c0:c1])
        torch.cuda.synchronize()
    finally:
        enc.close()
    assert bool((out1 > 0).all())
    assert torch.equal(out1, out2)
    live = torch.arange(dst1.shape[1], device=dev)[None, :] < out1[:, None]
    assert bool(((dst1 == dst2) | ~live).all()), "frames of the one-call encode differ from the split encode"
    # a few frames, the remainder's among them, also decode to their chunks
    for i in (0, 5, half - 1, half, npass - 1, npass, n - 2, n - 1):
        frame = bytes(dst1[i, :int(out1[i])].cpu().numpy())
        m = int(sizes[i])
        assert H.libzstd_decode(frame, m) == bytes(src[i * chunk:i * chunk + m].cpu().numpy()), i
