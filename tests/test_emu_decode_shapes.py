"""The decode pool (tests/decode_pool.py) through the emulated decode kernels, in each of the staged zstd decoder's forms:
results equal the oracle's, a frame of maxb blocks is staged and one of maxb + 1 is not, outputs land at unaligned
offsets without touching the bytes around them, and the per-input staged flags equal the ones recorded in
tests/golden/decode_pool_flags.json, which test_decode_shapes_gpu.py compares with the device.  CPU only.

Rewrite the recorded flags (after a deliberate change to the pool or to the staged decoder's rules) with
    python tests/test_emu_decode_shapes.py --write-flags"""
import json
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import decode_pool as DP  # noqa: E402
import helpers as H  # noqa: E402
from emu_util import emu_encode, emu_encode_frames, emu_s2_encode  # noqa: E402


def emu_pools(E):
    enc_chunks = lambda level, chunks: emu_encode(E, chunks, level=level)[0]
    enc_frames = lambda inputs: emu_encode_frames(E, inputs, level=1, dump=False)[0]
    zs = DP.build_zstd(enc_chunks, enc_frames)
    s2 = DP.build_s2(lambda blocks, better: emu_s2_encode(E, blocks, better=better)[0])
    return zs, s2


def emu_run(E, datas, caps, maxb=0, seed=0, s2=False):
    """One emulated decode launch with decode_pool.layout's offsets and sentinel-filled gaps.  maxb: the staged form
    (0: the device's choice for this batch size).  Returns (codes, staged flags, dst, dst_off)."""
    n = len(datas)
    so, stot, do, dtot = DP.layout([len(d) for d in datas], caps, seed)
    src = np.full(stot, DP.SENT, dtype=np.uint8)
    for i, d in enumerate(datas):
        src[int(so[i]):int(so[i]) + len(d)] = np.frombuffer(d, dtype=np.uint8)
    dst = np.full(dtot, DP.SENT, dtype=np.uint8)
    sizes = np.array([len(d) for d in datas], dtype=np.uint32)
    capv = np.array(caps, dtype=np.uint32)
    outs = np.zeros(n, dtype=np.int64)
    flags = np.zeros(max(n, 1), dtype=np.uint8)
    if s2:
        E.emu_s2_decode(src.ctypes.data, so.ctypes.data, sizes.ctypes.data, n, dst.ctypes.data, do.ctypes.data,
                        capv.ctypes.data, outs.ctypes.data)
        # the emulator counts the blocks of its last launch the staged kernels finished: one launch per block gives each
        # block's flag (the staged walk decides from the block alone)
        for i, d in enumerate(datas):
            one = np.zeros(len(d) + 16, dtype=np.uint8)
            one[:len(d)] = np.frombuffer(d, dtype=np.uint8)
            off0 = np.zeros(1, dtype=np.uint64)
            dst1 = np.zeros(caps[i] + 64, dtype=np.uint8)
            out1 = np.zeros(1, dtype=np.int64)
            E.emu_s2_decode(one.ctypes.data, off0.ctypes.data, sizes[i:i + 1].ctypes.data, 1, dst1.ctypes.data, off0.ctypes.data,
                            capv[i:i + 1].ctypes.data, out1.ctypes.data)
            assert int(out1[0]) == int(outs[i])
            flags[i] = E.emu_get_s2_staged_count()
    else:
        E.emu_set_dec_maxb(maxb)
        try:
            E.emu_zstd_decode_mode(src.ctypes.data, so.ctypes.data, sizes.ctypes.data, n, dst.ctypes.data, do.ctypes.data,
                                   capv.ctypes.data, outs.ctypes.data, 0, flags.ctypes.data)
        finally:
            E.emu_set_dec_maxb(0)
    return [int(x) for x in outs], [int(x) for x in flags[:n]], dst, do


def check_results(names, wants, caps, codes, dst, do):
    """Code and bytes equal the expected ones; the bytes outside every slot are still the sentinel, and so are the bytes
    between a decoded output's end and its slot's capacity."""
    keep = np.ones(dst.size, dtype=bool)
    for i, (nm, (wc, wout)) in enumerate(zip(names, wants)):
        assert codes[i] == wc, (i, nm, codes[i], wc)
        o = int(do[i])
        if wc >= 0:
            assert dst[o:o + wc].tobytes() == wout, (i, nm)
            keep[o:o + wc] = False
        else:
            keep[o:o + caps[i]] = False
    bad = np.nonzero(keep & (dst != DP.SENT))[0]
    assert bad.size == 0, "bytes written outside the outputs at %s" % bad[:8]


@pytest.fixture(scope="module")
def pools(emu_lib, oracle_lib):
    return emu_pools(emu_lib)


def run_forms(E, zs):
    """{form: [flag per small entry]} after checking every result of each form."""
    sm = DP.small(zs)
    caps = [DP.POOL_CAP] * len(sm)
    got = {}
    for form in DP.FORMS:
        codes, flags, dst, do = emu_run(E, [e["data"] for e in sm], caps, maxb=form, seed=form)
        check_results([e["name"] for e in sm], [(e["code"], e["out"]) for e in sm], caps, codes, dst, do)
        got[form] = flags
    return sm, got


@pytest.fixture(scope="module")
def form_flags(emu_lib, pools):
    return run_forms(emu_lib, pools[0])


def test_pool_matches_oracle_in_every_form(form_flags):
    sm, got = form_flags
    assert len(sm) > 100
    for form, flags in got.items():
        assert sum(flags) > len(sm) // 4, (form, sum(flags))          # the staged kernels take every valid simple frame


def test_block_count_switch_points(form_flags):
    sm, got = form_flags
    by = {e["name"]: i for i, e in enumerate(sm)}
    for form, flags in got.items():
        for k in (4, 16, 127, 128):
            if k == form:
                assert flags[by["rawrle_%d" % k]] == 1, (form, k)
                assert flags[by["rawrle_%d" % (k + 1)]] == 0, (form, k + 1)
        for e in sm:                  # valid single frames the staged kernels take: exactly those with <= maxb blocks
            if e["name"].startswith(("rawrle_", "FM_", "L1_", "L2_", "L3_")) and e["code"] >= 0:
                assert flags[by[e["name"]]] == (e["blocks"] <= form), (form, e["name"], e["blocks"])


@pytest.mark.parametrize("n", (512, 513, 4096, 4097))
def test_form_switch_by_batch_size(emu_lib, pools, n):
    # the form the launch picks from the batch size alone (no override): frames of maxb blocks staged, maxb + 1 not
    by = {e["name"]: e for e in pools[0]}
    maxb = DP.maxb_for(n)
    pick = {512: (128, 129), 513: (127, 128), 4096: (16, 17), 4097: (4, 5)}[n]
    ents = [by["rawrle_%d" % k] for k in pick] + [by["rawrle_4"], by["L1_1"], by["L1_0"]] * ((n - 2) // 3 + 1)
    ents = ents[:n]
    caps = [max(len(e["out"]) for e in ents) + 7] * n
    codes, flags, dst, do = emu_run(emu_lib, [e["data"] for e in ents], caps, seed=n)
    check_results([e["name"] for e in ents], [(e["code"], e["out"]) for e in ents], caps, codes, dst, do)
    assert flags[:2] == [1, 0] and all(flags[2:]), (n, maxb, flags[:8])


def test_reach_back_repeat_offsets(form_flags):
    # a block that starts from the repeat offsets an earlier block left: the per-block form cannot resolve it, the per-input
    # form does
    sm, got = form_flags
    by = {e["name"]: i for i, e in enumerate(sm)}
    i = by["reach_back"]
    assert got[4][i] == 1 and got[16][i] == 0 and got[127][i] == 0 and got[128][i] == 0
    # libzstd's two-block frames take the same path in every per-block form
    lz = [e for e in sm if e["name"].startswith("libzstd_") and (e["blocks"] or 0) > 1]
    assert len(lz) == 4
    for e in lz:
        j = by[e["name"]]
        assert got[16][j] == got[127][j] == got[128][j], e["name"]


def test_flags_match_recorded(pools, form_flags):
    zs, s2 = pools
    sm, got = form_flags
    rec = DP.load_flags()
    for k, e in enumerate(sm):
        r = rec["zstd"][e["name"]]
        assert r["sha"] == e["sha"], e["name"]
        assert [r[str(f)] for f in DP.FORMS] == [got[f][k] for f in DP.FORMS], e["name"]
    assert set(rec["zstd"]) == {e["name"] for e in sm}


def test_per_entry_capacity(emu_lib, pools):
    # capacity == content size decodes; one byte less is the oracle's error (both forms)
    zs, _ = pools
    ents = [e for e in zs if e["cap"] != DP.POOL_CAP]
    assert len(ents) == 24
    for form in (4, 128):
        codes, _, dst, do = emu_run(emu_lib, [e["data"] for e in ents], [e["cap"] for e in ents], maxb=form, seed=3)
        check_results([e["name"] for e in ents], [(e["code"], e["out"]) for e in ents], [e["cap"] for e in ents], codes, dst, do)
        assert all(c >= 0 for c, e in zip(codes, ents) if e["name"].endswith("_cap_size"))
        assert all(c < 0 for c, e in zip(codes, ents) if e["name"].endswith("_cap_short"))


def test_frame_mode_boundary_4_and_16(emu_lib):
    # frame-mode frames of k and k + 1 blocks (48 KiB each) at the per-input and the 16-block per-block forms
    fr = DP.frame_mode_boundary(lambda inputs: emu_encode_frames(emu_lib, inputs, level=1, dump=False)[0], (4, 16))
    for form, ks in ((4, (4, 5)), (16, (16, 17))):
        caps = [len(fr[k][1]) for k in ks]
        codes, flags, dst, do = emu_run(emu_lib, [fr[k][0] for k in ks], caps, maxb=form, seed=form)
        check_results(["fm%d" % k for k in ks], [(len(fr[k][1]), fr[k][1]) for k in ks], caps, codes, dst, do)
        assert flags == [1, 0], (form, flags)


def test_s2_pool(emu_lib, pools):
    _, s2 = pools
    caps = [DP.POOL_CAP] * len(s2)
    codes, flags, dst, do = emu_run(emu_lib, [e["data"] for e in s2], caps, seed=5, s2=True)
    check_results([e["name"] for e in s2], [(e["code"], e["out"]) for e in s2], caps, codes, dst, do)
    by = {e["name"]: i for i, e in enumerate(s2)}
    assert flags[by["s2_copy1_6"]] == 1 and flags[by["s2_copy1_7"]] == 0      # recCap = slen / 3 + 1, exactly
    assert flags[by["s2_over_64k"]] == 0 and flags[by["s2_stored"]] == 1
    rec = DP.load_flags()["s2"]
    assert set(rec) == set(by)
    for e, f in zip(s2, flags):
        assert rec[e["name"]]["sha"] == e["sha"] and rec[e["name"]]["flag"] == f, e["name"]


if __name__ == "__main__" and "--write-flags" in sys.argv:
    E = H.emu()
    zs, s2 = emu_pools(E)
    sm, got = run_forms(E, zs)
    rec = {"zstd": {e["name"]: dict({"sha": e["sha"]}, **{str(f): got[f][k] for f in DP.FORMS}) for k, e in enumerate(sm)}}
    _, s2flags, _, _ = emu_run(E, [e["data"] for e in s2], [DP.POOL_CAP] * len(s2), s2=True)
    rec["s2"] = {e["name"]: {"sha": e["sha"], "flag": f} for e, f in zip(s2, s2flags)}
    with open(DP.FLAGS_PATH, "w") as f:
        json.dump(rec, f, indent=0, sort_keys=True)
        f.write("\n")
    print("wrote", DP.FLAGS_PATH)
