"""Helpers of the S2 best tests: the oracle's EncodeBest / EncodeSnappyBest (oracle/orc_s2best.c, modes 3 and 4 of
orc_s2x_encode), the emulated best kernels (tests/emu/s2best.mk) and the shared inputs.  Test infrastructure only."""
import ctypes
import io
import os
import subprocess
import zipfile

import numpy as np

import helpers as H

ORACLE_SO = os.path.join(H.ORACLE_DIR, "liboracle_s2best.so")
EMU_SO = os.path.join(H.EMU_DIR, "libb2c_emu_s2best.so")
FAST, BETTER, SNAPPY, BEST, SNAPPY_BEST = 0, 1, 2, 3, 4
_lib = None


def oracle():
    """ctypes handle of oracle/liboracle_s2best.so (oracle/s2best.mk; built on demand)."""
    global _lib
    if _lib is not None:
        return _lib
    subprocess.run(["make", "-s", "-C", H.ORACLE_DIR, "-f", "s2best.mk"], check=True)
    L = ctypes.CDLL(ORACLE_SO)
    c = ctypes
    for nm in ("orc_s2x_encode", "orc_s2_decode", "orc_s2_max_encoded_len", "orc_s2_size_helper_mismatch",
               "orc_s2_emit_copy_size", "orc_s2_emit_repeat_size", "orc_s2_emit_copy_norepeat_size", "orc_s2_emit_copy_norepeat"):
        getattr(L, nm).restype = c.c_int64
    L.orc_s2x_encode.argtypes = [c.c_char_p, c.c_size_t, c.c_char_p, c.c_int64, c.c_int]
    L.orc_s2_decode.argtypes = [c.c_char_p, c.c_size_t, c.c_char_p, c.c_size_t]
    L.orc_s2_max_encoded_len.argtypes = [c.c_int64]
    L.orc_s2_size_helper_mismatch.argtypes = [c.c_int, c.c_int64, c.c_int64, c.c_int64]
    for nm in ("orc_s2_emit_copy_size", "orc_s2_emit_repeat_size", "orc_s2_emit_copy_norepeat_size"):
        getattr(L, nm).argtypes = [c.c_int64, c.c_int64]
    L.orc_s2_emit_copy_norepeat.argtypes = [c.c_char_p, c.c_int64, c.c_int64]
    _lib = L
    return L


def encode(data, mode):
    """Encode (0), EncodeBetter (1), EncodeSnappy (2), EncodeBest (3), EncodeSnappyBest (4) of the oracle."""
    L = oracle()
    cap = L.orc_s2_max_encoded_len(len(data))
    out = ctypes.create_string_buffer(cap + 16)
    r = L.orc_s2x_encode(out, cap, bytes(data), len(data), mode)
    assert r > 0, r
    return out.raw[:r]


def decode(comp, n):
    L = oracle()
    out = ctypes.create_string_buffer(max(n, 1))
    r = L.orc_s2_decode(out, n, bytes(comp), len(comp))
    return r, out.raw[:max(r, 0)]


def emu():
    subprocess.run(["make", "-s", "-C", H.EMU_DIR, "-f", "s2best.mk"], check=True)
    E = ctypes.CDLL(EMU_SO)
    c = ctypes
    E.emu_s2best_set_lane_order.argtypes = [c.c_int]
    E.emu_s2best_encode.argtypes = [c.c_void_p, c.c_uint64, c.c_void_p, c.c_uint32, c.c_void_p, c.c_uint64, c.c_void_p, c.c_int]
    return E


def emu_encode(E, blocks, snappy=False, desc=0):
    """The emulated best kernel over blocks (each <= 64 KiB) -> (outputs, out_sizes)."""
    E.emu_s2best_set_lane_order(desc)
    n, stride, dstride = len(blocks), 65536, 65536 + 512
    src = np.zeros(n * stride + 64, dtype=np.uint8)
    sizes = np.zeros(max(n, 1), dtype=np.uint32)
    for i, b in enumerate(blocks):
        src[i * stride:i * stride + len(b)] = np.frombuffer(b, dtype=np.uint8)
        sizes[i] = len(b)
    dst = np.zeros(n * dstride + 16, dtype=np.uint8)
    outs = np.zeros(max(n, 1), dtype=np.int64)
    E.emu_s2best_encode(src.ctypes.data, stride, sizes.ctypes.data, n, dst.ctypes.data, dstride, outs.ctypes.data, int(snappy))
    return [bytes(dst[i * dstride:i * dstride + max(int(outs[i]), 0)]) for i in range(n)], [int(x) for x in outs[:n]]


def fuzz_seeds(limit=None):
    """The reference's S2 encoder fuzz seeds committed under tests/golden (inputs only)."""
    z = zipfile.ZipFile(io.BytesIO(H.golden("s2_enc_regressions.zip")))
    out = [z.read(nm) for nm in sorted(z.namelist()) if not nm.endswith("/")]
    return out[:limit] if limit else out


def random_with_repeat(seed=7):
    """64 KiB of seeded random bytes with one 1 KiB run repeated: EncodeBest emits tags (dstLimit n - 5), EncodeBetter
    (dstLimit n - n/32 - 6) stores the block as one literal."""
    rng = np.random.default_rng(seed)
    b = bytearray(rng.integers(0, 256, 65536, dtype=np.uint8).tobytes())
    b[2000:3024] = b[16:1040]
    return bytes(b)


def corpora():
    tw = H.golden("twain.txt")
    return {"twain": [tw[i:i + 65536] for i in range(0, 3 * 65536, 65536)], "html": [H.golden("html.txt")[:65536]],
            "e": [H.golden("e.txt")[:65536]], "synth": [H.synth_text(65536, 3)]}
