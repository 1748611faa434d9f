"""Host-side mirror of the reference's huff0 block interface for the accelerated path.

``Compress4X`` / ``Compress1X`` (huff0/compress.go:27,14; fresh Scratch, ReusePolicyNone) and
``Decompress4X`` / ``Decompress1X`` after ``ReadTable`` (huff0/decompress.go:29,234,622), with the package's
sentinel errors (huff0/huff0.go:30-42).  Batches of blocks go through libb200comp.so (include/b2c.h).
"""
import ctypes

import numpy as np
import torch

from ._lib import lib, check, B2CError, Context, PointerTable

BlockSizeMax = (1 << 18) - 1


class ErrIncompressible(B2CError):
    pass


class ErrUseRLE(B2CError):
    pass


class ErrTooBig(B2CError):
    pass


class ErrCorrupt(B2CError):
    pass


_ERR = {-1: ErrIncompressible, -2: ErrUseRLE, -3: ErrTooBig, -5: ErrCorrupt}


class Codec(Context):
    def __init__(self, device=0):
        super().__init__(device)
        self.dev = torch.device("cuda", device)

    # ---- device-resident batches ----------------------------------------------------------------
    def compress_device(self, src, stride, sizes=None, four=True, dst=None, out_sizes=None):
        """src: uint8 CUDA tensor, block i at i*stride (sizes: optional uint32/int32 CUDA tensor, else all `stride`
        bytes).  Returns (dst [n, slot], out_sizes int64: bytes or negative huff0 error).  Async."""
        n = src.numel() // stride if sizes is None else sizes.numel()
        slot = (stride + 15) // 16 * 16
        if dst is None:
            dst = torch.empty((n, slot), dtype=torch.uint8, device=src.device)
        if out_sizes is None:
            out_sizes = torch.empty((n,), dtype=torch.int64, device=src.device)
        stream = torch.cuda.current_stream(src.device).cuda_stream
        check(lib.b2c_huf_compress_device(self._ctx, 1 if four else 0, src.data_ptr(), stride,
                                          None if sizes is None else sizes.data_ptr(), stride, dst.data_ptr(), dst.stride(0),
                                          out_sizes.data_ptr(), n, ctypes.c_void_p(stream)), self._ctx)
        return dst, out_sizes

    def decompress_device(self, src, src_stride, src_sizes, dst_sizes, dst_stride, four=True, dst=None, out_sizes=None):
        n = src_sizes.numel()
        if dst is None:
            dst = torch.empty((n, dst_stride), dtype=torch.uint8, device=src.device)
        if out_sizes is None:
            out_sizes = torch.empty((n,), dtype=torch.int64, device=src.device)
        stream = torch.cuda.current_stream(src.device).cuda_stream
        check(lib.b2c_huf_decompress_device(self._ctx, 1 if four else 0, src.data_ptr(), src_stride, src_sizes.data_ptr(),
                                            dst.data_ptr(), dst_stride, dst_sizes.data_ptr(), out_sizes.data_ptr(), n,
                                            ctypes.c_void_p(stream)), self._ctx)
        return dst, out_sizes

    # ---- host lists ---------------------------------------------------------------------------------
    def compress_blocks(self, blocks, four=True):
        """-> list of (bytes or None, code)."""
        n = len(blocks)
        if n == 0:
            return []
        stride = max(16, (max(len(b) for b in blocks) + 15) // 16 * 16)
        host = np.zeros((n, stride), dtype=np.uint8)
        for i, b in enumerate(blocks):
            host[i, :len(b)] = np.frombuffer(bytes(b), dtype=np.uint8)
        src = torch.from_numpy(host).to(self.dev)
        sizes = torch.tensor([len(b) for b in blocks], dtype=torch.int32, device=self.dev)
        dst, outs = self.compress_device(src.view(-1), stride, sizes, four)
        torch.cuda.synchronize()
        outs = outs.cpu().numpy()
        dsth = dst.cpu().numpy()
        return [(dsth[i, :outs[i]].tobytes() if outs[i] >= 0 else None, int(outs[i])) for i in range(n)]

    def decompress_blocks(self, blocks, dst_sizes, four=True):
        n = len(blocks)
        if n == 0:
            return []
        stride = max(16, (max(len(b) for b in blocks) + 15) // 16 * 16)
        host = np.zeros((n, stride), dtype=np.uint8)
        for i, b in enumerate(blocks):
            host[i, :len(b)] = np.frombuffer(bytes(b), dtype=np.uint8)
        src = torch.from_numpy(host).to(self.dev)
        ss = torch.tensor([len(b) for b in blocks], dtype=torch.int32, device=self.dev)
        ds = torch.tensor([int(d) for d in dst_sizes], dtype=torch.int32, device=self.dev)
        dstride = max(16, (max(int(d) for d in dst_sizes) + 15) // 16 * 16)
        dst, outs = self.decompress_device(src.view(-1), stride, ss, ds, dstride, four)
        torch.cuda.synchronize()
        outs = outs.cpu().numpy()
        dsth = dst.cpu().numpy()
        return [(dsth[i, :outs[i]].tobytes() if outs[i] >= 0 else None, int(outs[i])) for i in range(n)]

    # ---- host-buffer C-ABI calls (what a cgo shim binds) ------------------------------------------------------
    def _host(self, fn, blobs, caps, four):
        """-> list of (bytes or None, code)."""
        if not blobs:
            return []
        t = PointerTable(blobs, caps)
        check(fn(self._ctx, 1 if four else 0, t.srcs, t.ssz, t.dsts, t.dcap, t.res, t.n), self._ctx)
        return list(zip(*t.results()))

    def compress_chunks(self, blocks, four=True):
        """b2c_huf_compress_chunks: -> list of (bytes or None, code)."""
        return self._host(lib.b2c_huf_compress_chunks, blocks, [len(b) + 16 for b in blocks], four)

    def decompress_chunks(self, blocks, dst_sizes, four=True):
        return self._host(lib.b2c_huf_decompress_chunks, blocks, dst_sizes, four)

    def ReadTable(self, data):
        """huff0.ReadTable(in, nil) (huff0/decompress.go:29): -> (code length per symbol [256], tableLog, remaining input)."""
        t = PointerTable([data], [260])
        check(lib.b2c_huf_read_table(self._ctx, t.srcs, t.ssz, t.dsts, t.res, t.n), self._ctx)
        code = int(t.res[0])
        if code < 0:
            raise _ERR.get(code, B2CError)(lib.b2c_strerror(code).decode())
        row = t.outs[0]
        used = int(row[2]) | (int(row[3]) << 8)
        return [int(x) for x in row[4:260]], int(row[0]), bytes(data)[used:]

    def _one(self, res):
        out, code = res
        if code < 0:
            raise _ERR.get(code, B2CError)(lib.b2c_strerror(code).decode())
        return out

    def Compress4X(self, data):
        return self._one(self.compress_blocks([data], True)[0])

    def Compress1X(self, data):
        return self._one(self.compress_blocks([data], False)[0])

    def Decompress4X(self, data, dst_size):
        return self._one(self.decompress_blocks([data], [dst_size], True)[0])

    def Decompress1X(self, data, dst_size):
        return self._one(self.decompress_blocks([data], [dst_size], False)[0])
