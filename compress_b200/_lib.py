"""ctypes binding of libb200comp.so (the C ABI in include/b2c.h).

There is deliberately NO fallback: if the CUDA library has not been built, or no CUDA device is
present, importing / using the package raises.  The CPU oracle under oracle/ is test
infrastructure and is never imported from here.
"""
import ctypes
import os

import numpy as np
import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("B2C_LIB") or os.path.join(_HERE, "_lib", "libb200comp.so")   # B2C_LIB: tuning builds


class B2CError(RuntimeError):
    pass


def _load():
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a).  compress_b200 has no CPU fallback."
        )
    lib = ctypes.CDLL(LIB_PATH)
    c = ctypes
    lib.b2c_device_count.restype = c.c_int
    lib.b2c_ctx_create.restype = c.c_void_p
    lib.b2c_ctx_create.argtypes = [c.c_int, c.c_size_t]
    lib.b2c_ctx_destroy.argtypes = [c.c_void_p]
    lib.b2c_strerror.restype = c.c_char_p
    lib.b2c_strerror.argtypes = [c.c_int]
    lib.b2c_last_cuda_error.restype = c.c_char_p
    lib.b2c_last_cuda_error.argtypes = [c.c_void_p]
    lib.b2c_sm_count.restype = c.c_int
    lib.b2c_sm_count.argtypes = [c.c_void_p]
    lib.b2c_launch_count.restype = c.c_uint64
    lib.b2c_launch_count.argtypes = [c.c_void_p]
    lib.b2c_zstd_bound.restype = c.c_size_t
    lib.b2c_zstd_bound.argtypes = [c.c_size_t, c.c_int]
    lib.b2c_zstd_encode_device.restype = c.c_int
    lib.b2c_zstd_encode_device.argtypes = [
        c.c_void_p, c.c_int, c.c_int, c.c_void_p, c.c_size_t, c.c_void_p, c.c_uint32, c.c_void_p, c.c_size_t,
        c.c_void_p, c.c_uint32, c.c_void_p]
    lib.b2c_zstd_encode_device_debug.restype = c.c_int
    lib.b2c_zstd_encode_device_debug.argtypes = [
        c.c_void_p, c.c_int, c.c_int, c.c_void_p, c.c_size_t, c.c_void_p, c.c_uint32, c.c_void_p, c.c_size_t, c.c_void_p,
        c.c_uint32, c.c_void_p, c.c_void_p, c.c_void_p, c.c_uint32, c.c_void_p]
    lib.b2c_zstd_encode_chunks.restype = c.c_int
    lib.b2c_zstd_encode_chunks.argtypes = [
        c.c_void_p, c.c_int, c.c_int, c.c_void_p, c.c_void_p, c.c_void_p, c.c_void_p, c.c_void_p, c.c_size_t]
    lib.b2c_s2_decode_staged_count.restype = c.c_int
    lib.b2c_s2_decode_staged_count.argtypes = [c.c_void_p, c.c_uint32, c.c_void_p]
    lib.b2c_s2_stream_bound.restype = c.c_size_t
    lib.b2c_s2_stream_bound.argtypes = [c.c_size_t, c.c_size_t]
    lib.b2c_s2_encode_stream_device.restype = c.c_int
    lib.b2c_s2_encode_stream_device.argtypes = [c.c_void_p, c.c_int, c.c_int, c.c_void_p, c.c_uint64, c.c_uint32, c.c_void_p,
                                                c.c_uint64, c.c_void_p, c.c_void_p, c.c_void_p]
    lib.b2c_s2_encode_stream.restype = c.c_int
    lib.b2c_s2_encode_stream.argtypes = [c.c_void_p, c.c_int, c.c_int, c.c_void_p, c.c_size_t, c.c_uint32, c.c_void_p, c.c_size_t,
                                         c.c_void_p]
    lib.b2c_s2_decode_stream.restype = c.c_int
    lib.b2c_s2_decode_stream.argtypes = [c.c_void_p, c.c_void_p, c.c_size_t, c.c_void_p, c.c_size_t, c.c_void_p]
    lib.b2c_zstd_frame_bound.restype = c.c_size_t
    lib.b2c_zstd_frame_bound.argtypes = [c.c_size_t, c.c_int]
    lib.b2c_zstd_encode_frames_device.restype = c.c_int
    lib.b2c_zstd_encode_frames_device.argtypes = [
        c.c_void_p, c.c_int, c.c_int, c.c_void_p, c.c_void_p, c.c_void_p, c.c_uint32, c.c_void_p, c.c_uint64, c.c_void_p,
        c.c_void_p, c.c_void_p]
    lib.b2c_zstd_encode_frames.restype = c.c_int
    lib.b2c_zstd_encode_frames.argtypes = [
        c.c_void_p, c.c_int, c.c_int, c.c_void_p, c.c_void_p, c.c_void_p, c.c_void_p, c.c_void_p, c.c_size_t]
    lib.b2c_zstd_encode_packed.restype = c.c_int
    lib.b2c_zstd_encode_packed.argtypes = [
        c.c_void_p, c.c_int, c.c_int, c.c_void_p, c.c_size_t, c.c_uint32, c.c_void_p, c.c_size_t, c.c_void_p,
        c.c_void_p, c.c_void_p]
    lib.b2c_zstd_encode_device_timed.restype = c.c_int
    lib.b2c_zstd_encode_device_timed.argtypes = [
        c.c_void_p, c.c_int, c.c_void_p, c.c_size_t, c.c_uint32, c.c_void_p, c.c_size_t, c.c_void_p, c.c_uint32,
        c.c_void_p, c.c_void_p]
    lib.b2c_profile_enable.restype = c.c_int
    lib.b2c_profile_enable.argtypes = [c.c_void_p, c.c_int]
    lib.b2c_profile_read.restype = c.c_int
    lib.b2c_profile_read.argtypes = [c.c_void_p, c.c_void_p, c.c_void_p]
    lib.b2c_decode_profile_enable.restype = c.c_int
    lib.b2c_decode_profile_enable.argtypes = [c.c_void_p, c.c_int]
    lib.b2c_decode_profile_read.restype = c.c_int
    lib.b2c_decode_profile_read.argtypes = [c.c_void_p, c.c_void_p]
    lib.b2c_decode_staged_count.restype = c.c_int
    lib.b2c_decode_staged_count.argtypes = [c.c_void_p, c.c_uint32, c.c_void_p]
    for nm in ("b2c_decode_staged_flags", "b2c_s2_decode_staged_flags"):
        getattr(lib, nm).restype = c.c_int
        getattr(lib, nm).argtypes = [c.c_void_p, c.c_uint32, c.c_void_p]
    lib.b2c_zstd_decode_device.restype = c.c_int
    lib.b2c_zstd_decode_device.argtypes = [
        c.c_void_p, c.c_void_p, c.c_size_t, c.c_void_p, c.c_void_p, c.c_void_p, c.c_size_t, c.c_void_p, c.c_uint32,
        c.c_void_p, c.c_uint32, c.c_void_p]
    lib.b2c_zstd_decode_chunks.restype = c.c_int
    lib.b2c_zstd_decode_chunks.argtypes = [
        c.c_void_p, c.c_void_p, c.c_void_p, c.c_void_p, c.c_void_p, c.c_void_p, c.c_size_t]
    lib.b2c_s2_bound.restype = c.c_size_t
    lib.b2c_s2_bound.argtypes = [c.c_size_t]
    lib.b2c_s2_encode_device.restype = c.c_int
    lib.b2c_s2_encode_device.argtypes = [
        c.c_void_p, c.c_int, c.c_int, c.c_void_p, c.c_size_t, c.c_void_p, c.c_uint32, c.c_void_p, c.c_size_t,
        c.c_void_p, c.c_uint32, c.c_void_p]
    lib.b2c_s2_decode_device.restype = c.c_int
    lib.b2c_s2_decode_device.argtypes = [
        c.c_void_p, c.c_void_p, c.c_size_t, c.c_void_p, c.c_void_p, c.c_void_p, c.c_size_t, c.c_void_p, c.c_uint32,
        c.c_void_p, c.c_uint32, c.c_void_p]
    lib.b2c_s2_encode_chunks.restype = c.c_int
    lib.b2c_s2_encode_chunks.argtypes = [
        c.c_void_p, c.c_int, c.c_int, c.c_void_p, c.c_void_p, c.c_void_p, c.c_void_p, c.c_void_p, c.c_size_t]
    lib.b2c_s2_decode_chunks.restype = c.c_int
    lib.b2c_s2_decode_chunks.argtypes = [
        c.c_void_p, c.c_void_p, c.c_void_p, c.c_void_p, c.c_void_p, c.c_void_p, c.c_size_t]
    lib.b2c_s2_convert_lz4_device.restype = c.c_int
    lib.b2c_s2_convert_lz4_device.argtypes = [
        c.c_void_p, c.c_int, c.c_int, c.c_void_p, c.c_size_t, c.c_void_p, c.c_void_p, c.c_void_p, c.c_size_t, c.c_void_p,
        c.c_uint32, c.c_void_p, c.c_void_p, c.c_uint32, c.c_void_p]
    lib.b2c_s2_convert_lz4_chunks.restype = c.c_int
    lib.b2c_s2_convert_lz4_chunks.argtypes = [
        c.c_void_p, c.c_int, c.c_int, c.c_void_p, c.c_void_p, c.c_void_p, c.c_void_p, c.c_void_p, c.c_void_p, c.c_size_t]
    lib.b2c_flate_decode_device.restype = c.c_int
    lib.b2c_flate_decode_device.argtypes = [
        c.c_void_p, c.c_int, c.c_int, c.c_void_p, c.c_size_t, c.c_void_p, c.c_void_p, c.c_void_p, c.c_size_t, c.c_void_p,
        c.c_uint32, c.c_void_p, c.c_uint32, c.c_void_p]
    lib.b2c_flate_decode_chunks.restype = c.c_int
    lib.b2c_flate_decode_chunks.argtypes = [
        c.c_void_p, c.c_int, c.c_int, c.c_void_p, c.c_void_p, c.c_void_p, c.c_void_p, c.c_void_p, c.c_size_t]
    lib.b2c_flate_stateless_bound.restype = c.c_size_t
    lib.b2c_flate_stateless_bound.argtypes = [c.c_size_t, c.c_size_t]
    lib.b2c_flate_stateless_device.restype = c.c_int
    lib.b2c_flate_stateless_device.argtypes = [
        c.c_void_p, c.c_int, c.c_int, c.c_void_p, c.c_size_t, c.c_void_p, c.c_void_p, c.c_void_p, c.c_void_p, c.c_void_p,
        c.c_void_p, c.c_char_p, c.c_size_t, c.c_void_p, c.c_size_t, c.c_void_p, c.c_uint32, c.c_void_p, c.c_void_p,
        c.c_void_p, c.c_uint32, c.c_void_p]
    lib.b2c_flate_stateless_chunks.restype = c.c_int
    lib.b2c_flate_stateless_chunks.argtypes = [
        c.c_void_p, c.c_int, c.c_int, c.c_void_p, c.c_void_p, c.c_void_p, c.c_void_p, c.c_void_p, c.c_char_p, c.c_size_t,
        c.c_void_p, c.c_void_p, c.c_void_p, c.c_void_p, c.c_void_p, c.c_size_t]
    lib.b2c_flate_best_speed_bound.restype = c.c_size_t
    lib.b2c_flate_best_speed_bound.argtypes = [c.c_size_t]
    lib.b2c_flate_best_speed_device.restype = c.c_int
    lib.b2c_flate_best_speed_device.argtypes = [
        c.c_void_p, c.c_int, c.c_int, c.c_void_p, c.c_size_t, c.c_void_p, c.c_void_p, c.c_char_p, c.c_size_t, c.c_void_p,
        c.c_size_t, c.c_void_p, c.c_uint32, c.c_void_p, c.c_void_p, c.c_uint32, c.c_void_p]
    lib.b2c_flate_best_speed_chunks.restype = c.c_int
    lib.b2c_flate_best_speed_chunks.argtypes = [
        c.c_void_p, c.c_int, c.c_int, c.c_void_p, c.c_void_p, c.c_char_p, c.c_size_t, c.c_void_p, c.c_void_p, c.c_void_p,
        c.c_void_p, c.c_size_t]
    lib.b2c_flate_nolz_bound.restype = c.c_size_t
    lib.b2c_flate_nolz_bound.argtypes = [c.c_int, c.c_size_t]
    lib.b2c_flate_nolz_device.restype = c.c_int
    lib.b2c_flate_nolz_device.argtypes = [
        c.c_void_p, c.c_int, c.c_int, c.c_int, c.c_void_p, c.c_size_t, c.c_void_p, c.c_void_p, c.c_char_p, c.c_size_t,
        c.c_void_p, c.c_size_t, c.c_void_p, c.c_uint32, c.c_void_p, c.c_void_p, c.c_uint32, c.c_void_p]
    lib.b2c_flate_nolz_chunks.restype = c.c_int
    lib.b2c_flate_nolz_chunks.argtypes = [
        c.c_void_p, c.c_int, c.c_int, c.c_int, c.c_void_p, c.c_void_p, c.c_char_p, c.c_size_t, c.c_void_p, c.c_void_p,
        c.c_void_p, c.c_void_p, c.c_size_t]
    lib.b2c_huf_compress_device.restype = c.c_int
    lib.b2c_huf_compress_device.argtypes = [
        c.c_void_p, c.c_int, c.c_void_p, c.c_size_t, c.c_void_p, c.c_uint32, c.c_void_p, c.c_size_t, c.c_void_p,
        c.c_uint32, c.c_void_p]
    lib.b2c_huf_decompress_device.restype = c.c_int
    lib.b2c_huf_decompress_device.argtypes = [
        c.c_void_p, c.c_int, c.c_void_p, c.c_size_t, c.c_void_p, c.c_void_p, c.c_size_t, c.c_void_p, c.c_void_p,
        c.c_uint32, c.c_void_p]
    for nm in ("b2c_huf_compress_chunks", "b2c_huf_decompress_chunks"):
        getattr(lib, nm).restype = c.c_int
        getattr(lib, nm).argtypes = [c.c_void_p, c.c_int, c.c_void_p, c.c_void_p, c.c_void_p, c.c_void_p, c.c_void_p, c.c_size_t]
    lib.b2c_huf_read_table.restype = c.c_int
    lib.b2c_huf_read_table.argtypes = [c.c_void_p, c.c_void_p, c.c_void_p, c.c_void_p, c.c_void_p, c.c_size_t]
    lib.b2c_queue_create.restype = c.c_void_p
    lib.b2c_queue_create.argtypes = [c.c_int, c.c_size_t, c.c_uint]
    lib.b2c_queue_destroy.argtypes = [c.c_void_p]
    for nm in ("b2c_queue_zstd_encode", "b2c_queue_s2_encode"):
        getattr(lib, nm).restype = c.c_int64
        getattr(lib, nm).argtypes = [c.c_void_p, c.c_int, c.c_int, c.c_void_p, c.c_size_t, c.c_void_p, c.c_size_t]
    for nm in ("b2c_queue_zstd_decode", "b2c_queue_s2_decode"):
        getattr(lib, nm).restype = c.c_int64
        getattr(lib, nm).argtypes = [c.c_void_p, c.c_void_p, c.c_size_t, c.c_void_p, c.c_size_t]
    lib.b2c_queue_stats.restype = c.c_int
    lib.b2c_queue_stats.argtypes = [c.c_void_p, c.c_void_p, c.c_void_p]
    return lib


lib = _load()

# every symbol include/b2c.h declares; tests assert the built library exports all of them
EXPORTED_SYMBOLS = [
    "b2c_device_count", "b2c_ctx_create", "b2c_ctx_destroy", "b2c_strerror", "b2c_last_cuda_error",
    "b2c_sm_count", "b2c_launch_count", "b2c_zstd_bound", "b2c_zstd_encode_device",
    "b2c_zstd_encode_chunks", "b2c_zstd_encode_device_debug", "b2c_zstd_encode_packed", "b2c_zstd_encode_device_timed",
    "b2c_zstd_decode_device", "b2c_zstd_decode_chunks", "b2c_profile_enable", "b2c_profile_read", "b2c_decode_profile_enable", "b2c_decode_profile_read", "b2c_decode_staged_count", "b2c_s2_decode_staged_count",
    "b2c_decode_staged_flags", "b2c_s2_decode_staged_flags",
    "b2c_huf_compress_device", "b2c_huf_decompress_device",
    "b2c_s2_bound", "b2c_s2_encode_device", "b2c_s2_decode_device", "b2c_s2_encode_chunks", "b2c_s2_decode_chunks",
    "b2c_huf_compress_chunks", "b2c_huf_decompress_chunks", "b2c_huf_read_table",
    "b2c_queue_create", "b2c_queue_destroy", "b2c_queue_zstd_encode", "b2c_queue_zstd_decode", "b2c_queue_s2_encode",
    "b2c_queue_s2_decode", "b2c_queue_stats",
    "b2c_zstd_frame_bound", "b2c_zstd_encode_frames_device", "b2c_zstd_encode_frames",
    "b2c_s2_stream_bound", "b2c_s2_encode_stream_device", "b2c_s2_encode_stream", "b2c_s2_decode_stream",
    "b2c_s2_convert_lz4_device", "b2c_s2_convert_lz4_chunks",
    "b2c_flate_decode_device", "b2c_flate_decode_chunks",
    "b2c_flate_stateless_bound", "b2c_flate_stateless_device", "b2c_flate_stateless_chunks",
    "b2c_flate_best_speed_bound", "b2c_flate_best_speed_device", "b2c_flate_best_speed_chunks",
    "b2c_flate_nolz_bound", "b2c_flate_nolz_device", "b2c_flate_nolz_chunks",
]


def check(rc, ctx=None):
    if rc != 0:
        msg = lib.b2c_strerror(rc).decode()
        if ctx:
            msg += ": " + lib.b2c_last_cuda_error(ctx).decode()
        raise B2CError(f"libb200comp error {rc}: {msg}")


class Context:
    """Owner of one library context (b2c_ctx) on a CUDA device, freed by close(), at the end of a with block or with the
    object.  Raises B2CError without a device: there is no CPU fallback."""

    _ctx = None

    def __init__(self, device=0, max_chunks=0):
        if not torch.cuda.is_available() or lib.b2c_device_count() == 0:
            raise B2CError("no CUDA device: compress_b200 has no CPU fallback")
        self._ctx = lib.b2c_ctx_create(device, max_chunks)
        if not self._ctx:
            raise B2CError("b2c_ctx_create failed")

    def close(self):
        if self._ctx:
            lib.b2c_ctx_destroy(self._ctx)
            self._ctx = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()


class PointerTable:
    """The arguments of a pointer-table call for n blobs: srcs / ssz (their addresses and sizes), dsts / dcap (one output
    buffer of caps[i] bytes each) and res (the per-blob results), kept alive with the table.  An empty blob is passed as a
    one-byte placeholder."""

    def __init__(self, blobs, caps):
        self.n = len(blobs)
        self._keep = []
        self.srcs = self.pointers(blobs)
        self.ssz = (ctypes.c_size_t * self.n)(*[len(b) for b in blobs])
        self.outs = [np.empty(max(int(c), 1), dtype=np.uint8) for c in caps]
        self.dsts = (ctypes.c_void_p * self.n)(*[o.ctypes.data for o in self.outs])
        self.dcap = (ctypes.c_size_t * self.n)(*[int(c) for c in caps])
        self.res = (ctypes.c_int64 * self.n)()

    def pointers(self, blobs):
        """A c_void_p array of the blobs' addresses; the blobs' buffers live as long as the table."""
        a = [np.frombuffer(bytes(b), dtype=np.uint8) if len(b) else np.zeros(1, dtype=np.uint8) for b in blobs]
        self._keep.append(a)
        return (ctypes.c_void_p * len(a))(*[x.ctypes.data for x in a])

    def results(self):
        """-> (outputs, codes): outputs[i] the result's bytes, None where codes[i] is a negative error."""
        codes = [int(r) for r in self.res]
        return [o[:c].tobytes() if c >= 0 else None for o, c in zip(self.outs, codes)], codes
