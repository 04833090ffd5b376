"""libbsc_b200 -- GPU (H100, sm_90a) block-sorting compression hot path (libbsc 3.3.5 compatible).

The product is the C-ABI shared library ``libbsc_b200/libbsc_b200.so`` (sources in ``csrc/``,
interface in ``include/libbsc_b200.h``).  This package is only a thin ctypes binding of that ABI
for tests and bench.py; it contains no algorithmic code and has NO fallback: if the CUDA library is
missing or no CUDA device is usable, loading / ``bsc_init`` fails loudly.
"""
import ctypes
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libbsc_b200.so")

vp, ci = ctypes.c_void_p, ctypes.c_int
_lib = None

NO_ERROR, BAD_PARAMETER, NOT_ENOUGH_MEMORY, NOT_COMPRESSIBLE, NOT_SUPPORTED = 0, -1, -2, -3, -4
UNEXPECTED_EOB, DATA_CORRUPT, GPU_ERROR, GPU_NOT_SUPPORTED, GPU_NOT_ENOUGH_MEMORY = -5, -6, -7, -8, -9
HEADER_SIZE = 28

_SIGNATURES = {
    # group 1 (libbsc-compatible)
    "bsc_init": ([ci], ci),
    "bsc_init_full": ([ci, vp, vp, vp], ci),
    "bsc_compress": ([vp, vp, ci, ci, ci, ci, ci, ci], ci),
    "bsc_store": ([vp, vp, ci, ci], ci),
    "bsc_block_info": ([vp, ci, vp, vp, ci], ci),
    "bsc_decompress": ([vp, ci, vp, ci, ci], ci),
    "bsc_bwt_init": ([ci], ci),
    "bsc_bwt_encode": ([vp, ci, vp, vp, ci], ci),
    "bsc_bwt_decode": ([vp, ci, ci, ctypes.c_ubyte, vp, ci], ci),
    "bsc_st_init": ([ci], ci),
    "bsc_st_encode": ([vp, ci, ci, ci], ci),
    "bsc_st_decode": ([vp, ci, ci, ci, ci], ci),
    "bsc_coder_init": ([ci], ci),
    "bsc_coder_compress": ([vp, vp, ci, ci, ci], ci),
    "bsc_coder_decompress": ([vp, vp, ci, ci], ci),
    "bsc_qlfc_init": ([ci], ci),
    "bsc_qlfc_static_encode_block": ([vp, vp, ci, ci], ci),
    "bsc_qlfc_adaptive_encode_block": ([vp, vp, ci, ci], ci),
    "bsc_qlfc_fast_encode_block": ([vp, vp, ci, ci], ci),
    "bsc_qlfc_static_decode_block": ([vp, vp], ci),
    "bsc_qlfc_adaptive_decode_block": ([vp, vp], ci),
    "bsc_qlfc_fast_decode_block": ([vp, vp], ci),
    "bsc_adler32": ([vp, ci, ci], ctypes.c_uint32),
    "bsc_platform_init": ([ci, vp, vp, vp], ci),
    "bsc_malloc": ([ctypes.c_size_t], vp),
    "bsc_zero_malloc": ([ctypes.c_size_t], vp),
    "bsc_free": ([vp], None),
    # group 2 (extensions)
    "bscb200_coder_decompress": ([vp, ci, vp, ci, ci, ci], ci),
    "bscb200_ctx_create": ([ci, vp], vp),
    "bscb200_ctx_destroy": ([vp], None),
    "bscb200_ctx_reserve": ([vp, ctypes.c_longlong], ci),
    "bscb200_ctx_set_sort_budget": ([vp, ctypes.c_longlong], ci),
    "bscb200_lzp_decompress_host": ([vp, ci, vp, ci, ci, ci], ci),
    "bscb200_lzp_compress_host": ([vp, vp, ci, ci, ci, ci], ci),
    "bscb200_device_count": ([], ci),
    "bscb200_set_device": ([ci], ci),
    "bscb200_device_free_bytes": ([], ctypes.c_longlong),
    "bscb200_release_pools": ([], None),
    "bscb200_workspace_bytes": ([ci, ci], ctypes.c_longlong),
    "bscb200_workspace_bytes_decode": ([ci], ctypes.c_longlong),
    "bscb200_scratch_bytes": ([ci, ci], ctypes.c_longlong),
    "bscb200_inplace_bytes": ([ci, ci, ci], ctypes.c_longlong),
    "bscb200_decompress_bytes": ([ci, ci], ctypes.c_longlong),
    "bscb200_st_encode_bytes": ([ci], ctypes.c_longlong),
    "bscb200_ctx_kernel_launches": ([vp], ctypes.c_ulonglong),
    "bscb200_total_kernel_launches": ([], ctypes.c_ulonglong),
    "bscb200_ctx_set_profile": ([vp, ci], None),
    "bscb200_ctx_profile_report": ([vp, ctypes.c_char_p, ci], ci),
    "bscb200_version": ([], ctypes.c_char_p),
    "bscb200_compress_device": ([vp, vp, vp, ci, ci, ci, ci], ci),
    "bscb200_decompress_device": ([vp, vp, ci, vp, ci, ci], ci),
    "bscb200_bwt_encode_device": ([vp, vp, ci, vp, vp], ci),
    "bscb200_bwt_decode_device": ([vp, vp, ci, ci], ci),
    "bscb200_st_encode_device": ([vp, vp, ci, ci], ci),
    "bscb200_st_decode_device": ([vp, vp, ci, ci, ci], ci),
    "bscb200_coder_compress_device": ([vp, vp, vp, ci, ci, ci], ci),
    "bscb200_coder_decompress_device": ([vp, vp, ci, vp, ci, ci, ci], ci),
    "bscb200_adler32_device": ([vp, vp, ci], ctypes.c_uint32),
}
EXPORTED_SYMBOLS = tuple(_SIGNATURES)


def lib():
    """Load the CUDA library (built by __graft_entry__.build() / libbsc_b200/build.py)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError("libbsc_b200.so is not built (%s); run `python libbsc_b200/build.py` -- there is no CPU fallback" % LIB_PATH)
        L = ctypes.CDLL(LIB_PATH)
        for name, (args, res) in _SIGNATURES.items():
            f = getattr(L, name)
            f.argtypes = args
            f.restype = res
        _lib = L
    return _lib


class BscError(RuntimeError):
    pass


class Bsc:
    """numpy-level view of the host-pointer C ABI (same method names as oracle/pyoracle.py)."""
    kind = "b200"

    def __init__(self, features=3):
        self.lib = lib()
        r = self.lib.bsc_init(features)
        if r != 0:
            raise BscError("bsc_init failed with %d (no usable CUDA device? this library has no CPU path)" % r)
        self.features = features

    def adler32(self, a):
        a = np.ascontiguousarray(a, dtype=np.uint8)
        return int(self.lib.bsc_adler32(a.ctypes.data, a.size, 0))

    def bwt_encode(self, data, aux=True):
        T = np.array(data, dtype=np.uint8, copy=True)
        idx = (ci * 256)()
        ni = ctypes.c_ubyte(0)
        if aux:
            r = self.lib.bsc_bwt_encode(T.ctypes.data, T.size, ctypes.cast(ctypes.byref(ni), vp), ctypes.cast(idx, vp), self.features)
        else:
            r = self.lib.bsc_bwt_encode(T.ctypes.data, T.size, None, None, self.features)
        return r, T, [idx[t] for t in range(ni.value)]

    def bwt_decode(self, L, index, indexes=()):
        T = np.array(L, dtype=np.uint8, copy=True)
        arr = (ci * 256)(*indexes)
        r = self.lib.bsc_bwt_decode(T.ctypes.data, T.size, index, len(indexes), ctypes.cast(arr, vp), self.features)
        return r, T

    def st_encode(self, data, k):
        n = len(data)
        T = np.empty(n + 64, dtype=np.uint8)
        T[:n] = data
        r = self.lib.bsc_st_encode(T.ctypes.data, n, k, self.features)
        return r, T[:n].copy()

    def st_decode(self, L, k, index):
        T = np.array(L, dtype=np.uint8, copy=True)
        r = self.lib.bsc_st_decode(T.ctypes.data, T.size, k, index, self.features)
        return r, T

    _QLFC = {1: "static", 2: "adaptive", 3: "fast"}

    def encode_block(self, data, out_size=None, coder=1):
        """bsc_qlfc_<coder>_encode_block: one QLFC stream (same method as oracle/pyoracle.py)"""
        data = np.ascontiguousarray(data, dtype=np.uint8)
        cap = data.size if out_size is None else out_size
        out = np.empty(max(cap, data.size) + 64, dtype=np.uint8)
        r = getattr(self.lib, "bsc_qlfc_%s_encode_block" % self._QLFC[coder])(data.ctypes.data, out.ctypes.data, data.size, cap)
        return r, out[:max(r, 0)].copy()

    def decode_block(self, stream, n, coder=1):
        stream = np.concatenate([np.ascontiguousarray(stream, dtype=np.uint8), np.zeros(n + 64, dtype=np.uint8)])   # size-less ABI: n + 16 readable bytes
        out = np.empty(n + 64, dtype=np.uint8)
        r = getattr(self.lib, "bsc_qlfc_%s_decode_block" % self._QLFC[coder])(stream.ctypes.data, out.ctypes.data)
        return r, out[:max(r, 0)].copy()

    def coder_compress(self, L, coder=1, features=3):
        L = np.ascontiguousarray(L, dtype=np.uint8)
        out = np.empty(L.size + 4096, dtype=np.uint8)
        r = self.lib.bsc_coder_compress(L.ctypes.data, out.ctypes.data, L.size, coder, features)
        return r, (out[:r].copy() if r > 0 else None)

    def coder_decompress(self, stream, n, coder=1, features=3):
        s = np.zeros(len(stream) + 64, dtype=np.uint8)
        s[:len(stream)] = stream
        out = np.empty(n + 64, dtype=np.uint8)
        r = self.lib.bsc_coder_decompress(s.ctypes.data, out.ctypes.data, coder, features)
        return r, out[:max(r, 0)].copy()

    def store(self, data):
        data = np.ascontiguousarray(data, dtype=np.uint8)
        out = np.empty(data.size + 28, dtype=np.uint8)
        r = self.lib.bsc_store(data.ctypes.data, out.ctypes.data, data.size, 0)
        return r, out

    def compress(self, data, sorter=1, coder=1, features=3, lzp_hash=0, lzp_min=0):
        data = np.ascontiguousarray(data, dtype=np.uint8)
        out = np.empty(data.size + 28 + 64, dtype=np.uint8)
        r = self.lib.bsc_compress(data.ctypes.data, out.ctypes.data, data.size, lzp_hash, lzp_min, sorter, coder, features)
        return r, (out[:r].copy() if r > 0 else None)

    def block_info(self, block):
        block = np.ascontiguousarray(block, dtype=np.uint8)
        bs, ds = ci(0), ci(0)
        r = self.lib.bsc_block_info(block.ctypes.data, block.size, ctypes.cast(ctypes.byref(bs), vp), ctypes.cast(ctypes.byref(ds), vp), 0)
        return r, bs.value, ds.value

    def decompress(self, block, features=3):
        block = np.ascontiguousarray(block, dtype=np.uint8)
        r, bs, ds = self.block_info(block)
        if r != 0:
            return r, None
        out = np.empty(ds + 64, dtype=np.uint8)
        r = self.lib.bsc_decompress(block.ctypes.data, block.size, out.ctypes.data, ds, features)
        return r, out[:ds].copy()


class DeviceCtx:
    """One stream + workspace on one GPU (bscb200_ctx_*); operates on raw device pointers."""

    def __init__(self, device=0, cuda_stream=0):
        self.lib = lib()
        self.handle = self.lib.bscb200_ctx_create(device, cuda_stream or None)
        if not self.handle:
            raise BscError("bscb200_ctx_create failed on device %d" % device)

    def close(self):
        if self.handle:
            self.lib.bscb200_ctx_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def reserve(self, nbytes):
        return self.lib.bscb200_ctx_reserve(self.handle, nbytes)

    def set_sort_budget(self, nbytes):
        """Bound the forward BWT's working set to about `nbytes` (batched sort above it; 0 = no bound).  Returns 0 or BAD_PARAMETER."""
        return self.lib.bscb200_ctx_set_sort_budget(self.handle, nbytes)

    def launches(self):
        return int(self.lib.bscb200_ctx_kernel_launches(self.handle))

    def set_profile(self, on):
        self.lib.bscb200_ctx_set_profile(self.handle, 1 if on else 0)

    def profile_report(self):
        """{kernel name: (launches, total_ms, algorithmic_bytes)} since set_profile(True)."""
        import re
        buf = ctypes.create_string_buffer(1 << 16)
        n = self.lib.bscb200_ctx_profile_report(self.handle, buf, len(buf))
        out = {}
        for line in buf.raw[:n].decode().splitlines():
            name, cnt, ms, b = line.split("\t")
            name = re.match(r"\(?\s*([A-Za-z_0-9]+)", name).group(1)
            c0, m0, b0 = out.get(name, (0, 0.0, 0.0))
            out[name] = (c0 + int(cnt), m0 + float(ms), b0 + float(b))
        return out

    def compress(self, d_in, d_out, n, sorter=1, coder=1, features=3):
        return self.lib.bscb200_compress_device(self.handle, d_in, d_out, n, sorter, coder, features)

    def decompress(self, d_in, in_size, d_out, out_size, features=3):
        return self.lib.bscb200_decompress_device(self.handle, d_in, in_size, d_out, out_size, features)

    def bwt_encode(self, d_T, n, aux=True):
        idx = (ci * 256)()
        ni = ctypes.c_ubyte(0)
        if aux:
            r = self.lib.bscb200_bwt_encode_device(self.handle, d_T, n, ctypes.cast(ctypes.byref(ni), vp), ctypes.cast(idx, vp))
        else:
            r = self.lib.bscb200_bwt_encode_device(self.handle, d_T, n, None, None)
        return r, [idx[t] for t in range(ni.value)]

    def bwt_decode(self, d_T, n, index):
        return self.lib.bscb200_bwt_decode_device(self.handle, d_T, n, index)

    def st_encode(self, d_T, n, k):
        return self.lib.bscb200_st_encode_device(self.handle, d_T, n, k)

    def st_decode(self, d_T, n, k, index):
        return self.lib.bscb200_st_decode_device(self.handle, d_T, n, k, index)

    def coder_compress(self, d_in, d_out, n, coder=1, features=3):
        return self.lib.bscb200_coder_compress_device(self.handle, d_in, d_out, n, coder, features)

    def coder_decompress(self, d_in, in_size, d_out, out_cap, coder=1, features=3):
        return self.lib.bscb200_coder_decompress_device(self.handle, d_in, in_size, d_out, out_cap, coder, features)

    def adler32(self, d_p, n):
        return int(self.lib.bscb200_adler32_device(self.handle, d_p, n))
