"""finitestateentropy_b200 -- H100-native (sm_90a) block entropy coding: the FSE / Huff0 32 KB block
hot path of Cyan4973/FiniteStateEntropy behind the reference's own C API.

The product is `libfse_b200.so` (hand-written CUDA kernels + a C-ABI, see include/fse_b200.h).  This
package is only the thin Python binding used by tests/ and bench.py: ctypes over the C-ABI, torch for
device memory / streams / torch.distributed.  There is NO CPU implementation here: if the CUDA
library is missing, importing `lib()` raises."""
import ctypes as C
import os

from . import _build

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

c_sz = C.c_size_t
c_vp = C.c_void_p

BLOCK_SIZE = 32768                     # programs/bench.c:98
ERR_MAXCODE = 9                        # lib/error_public.h:55
ERROR_NAMES = {1: "GENERIC", 2: "dstSize_tooSmall", 3: "srcSize_wrong", 4: "corruption_detected",
               5: "tableLog_tooLarge", 6: "maxSymbolValue_tooLarge", 7: "maxSymbolValue_tooSmall",
               8: "workSpace_tooSmall"}


def compress_bound(n):
    """FSE_compressBound (lib/fse.h:290-292): per-block slot size used by programs/bench.c:355,514"""
    return 512 + n + (n >> 7) + 4 + 8


def is_error(code):
    return int(code) > (1 << 64) - ERR_MAXCODE


def error_code(code):
    return ((1 << 64) - int(code)) if is_error(code) else 0


def lib():
    """Loads (building in-tree first if needed) the CUDA library.  Fails loudly; never falls back."""
    global _LIB
    if _LIB is None:
        path = _build.LIB
        if _build.lib_is_stale():
            try:
                path = _build.build_lib()
            except Exception as exc:  # nvcc missing on the box: use the prebuilt .so if there is one
                if not os.path.exists(path):
                    raise RuntimeError("libfse_b200.so is missing and cannot be built: %r -- there is no CPU fallback" % (exc,))
        L = C.CDLL(path)
        _declare(L)
        _LIB = L
    return _LIB


def _declare(L):
    def sig(name, res, *args):
        f = getattr(L, name)
        f.restype = res
        f.argtypes = list(args)

    sig("FSEB200_batch_blocks", c_sz, c_sz, c_sz)
    sig("FSEB200_HUF_decompress_batch", c_sz, c_vp, c_sz, c_sz, c_vp, c_sz, c_vp, c_vp, c_vp, c_vp)
    sig("HUF_decompress", c_sz, c_vp, c_sz, c_vp, c_sz)
    sig("FSEB200_HUF_compress_blocks", c_sz, c_sz, c_vp, c_vp, c_vp, c_vp, c_vp, C.c_uint, C.c_uint, c_vp)
    sig("FSEB200_HUF_decompress_blocks", c_sz, c_sz, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp)
    sig("FSEB200_HUF_compress1X_blocks", c_sz, c_sz, c_vp, c_vp, c_vp, c_vp, c_vp, C.c_uint, C.c_uint, c_vp)
    sig("FSEB200_HUF_decompress1X_blocks", c_sz, c_sz, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp)
    for name in ("FSEB200_HUF_compress4X_repeat_blocks", "FSEB200_HUF_compress1X_repeat_blocks"):
        sig(name, c_sz, c_sz, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, C.c_uint, C.c_uint, c_vp)
    for name in ("FSEB200_HUF_compress4X_repeat_chains", "FSEB200_HUF_compress1X_repeat_chains"):
        sig(name, c_sz, c_sz, c_vp, c_sz, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, C.c_uint, C.c_uint, c_vp)
    for name in ("FSEB200_HUF_compress4X_repeat_chains_packed", "FSEB200_HUF_compress1X_repeat_chains_packed"):
        sig(name, c_sz, c_sz, c_vp, c_sz, c_vp, c_sz, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, C.c_uint, C.c_uint, c_vp)
    for name in ("FSEB200_HUF_decompress4X_repeat_packed", "FSEB200_HUF_decompress1X_repeat_packed"):
        sig(name, c_sz, c_sz, c_vp, c_sz, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp)
    for name in ("FSEB200_HUF_decompress4X_repeat_blocks", "FSEB200_HUF_decompress1X_repeat_blocks"):
        sig(name, c_sz, c_sz, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp)
    sig("FSEB200_HUF_compress_mixed_repeat_chains", c_sz, c_sz, c_vp, c_sz, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
        c_vp, c_vp, c_vp, c_vp, C.c_uint, C.c_uint, c_vp)
    sig("FSEB200_HUF_decompress_mixed_repeat_blocks", c_sz, c_sz, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp)
    sig("FSEB200_HUF_compress_mixed_repeat_chains_packed", c_sz, c_sz, c_vp, c_sz, c_vp, c_sz, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
        c_vp, c_vp, c_vp, c_vp, c_vp, C.c_uint, C.c_uint, c_vp)
    sig("FSEB200_HUF_decompress_mixed_repeat_packed", c_sz, c_sz, c_vp, c_sz, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
        c_vp)
    sig("FSEB200_HUF_compress_literals_chains_packed", c_sz, c_sz, c_vp, c_sz, c_vp, c_sz, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
        c_vp, c_vp, c_vp, c_vp, c_vp, C.c_uint, C.c_uint, C.c_uint, C.c_uint, c_vp)
    for name in ("FSEB200_HUF_compress_packed", "FSEB200_HUF_compress1X_packed"):
        sig(name, c_sz, c_sz, c_vp, c_sz, c_vp, c_vp, c_vp, c_vp, C.c_uint, C.c_uint, c_vp)
    for codec in ("FSE", "FSEU16"):
        sig("FSEB200_%s_compress_blocks" % codec, c_sz, c_sz, c_vp, c_vp, c_vp, c_vp, c_vp, C.c_uint, C.c_uint, c_vp)
        sig("FSEB200_%s_decompress_blocks" % codec, c_sz, c_sz, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp)
        sig("FSEB200_%s_compress_packed" % codec, c_sz, c_sz, c_vp, c_sz, c_vp, c_vp, c_vp, c_vp, C.c_uint, C.c_uint, c_vp, c_sz, c_vp)
        sig("FSEB200_%s_decompress_packed" % codec, c_sz, c_sz, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp)
    sig("FSEB200_FSE_packed_workspace", c_sz, c_sz, c_sz)
    for name in ("FSEB200_HUF_decompress_packed", "FSEB200_HUF_decompress1X_packed"):
        sig(name, c_sz, c_sz, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp)
    sig("FSEB200_compress_host_packed", c_sz, C.c_int, c_vp, c_sz, c_vp, c_vp, c_vp, c_vp, c_sz, C.c_uint, C.c_uint)
    sig("FSEB200_decompress_host_packed", c_sz, C.c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_sz)
    sig("FSEB200_compress_host_repeat_chains_packed", c_sz, C.c_int, c_sz, c_vp, c_sz, c_vp, c_sz, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
        c_vp, c_vp, c_vp, c_vp, C.c_uint, C.c_uint)
    sig("FSEB200_decompress_host_repeat_packed", c_sz, C.c_int, c_sz, c_vp, c_sz, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp)
    sig("FSEB200_compress_host_mixed_repeat_chains_packed", c_sz, c_sz, c_vp, c_sz, c_vp, c_sz, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
        c_vp, c_vp, c_vp, c_vp, C.c_uint, C.c_uint)
    sig("FSEB200_decompress_host_mixed_repeat_packed", c_sz, c_sz, c_vp, c_sz, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp)
    sig("FSEB200_compress_host_literals_chains_packed", c_sz, c_sz, c_vp, c_sz, c_vp, c_sz, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
        c_vp, c_vp, c_vp, c_vp, C.c_uint, C.c_uint, C.c_uint, C.c_uint)
    sig("FSEB200_frame_compressBound", c_sz, c_sz, C.c_uint)
    sig("FSEB200_frame_compress_host", c_sz, C.c_int, C.c_uint, c_vp, c_sz, c_vp, c_sz)
    sig("FSEB200_frame_decompress_bound", c_sz, c_vp, c_sz)
    sig("FSEB200_frame_decompress_host", c_sz, c_vp, c_sz, c_vp, c_sz)
    sig("FSEB200_frame_compress_host_batch", c_sz, C.c_int, C.c_uint, c_sz, c_vp, c_sz, c_vp, c_vp, c_vp, c_vp)
    sig("FSEB200_frame_decompress_host_batch", c_sz, c_sz, c_vp, c_vp, c_vp, c_vp, c_vp)
    sig("FSEB200_frame_compress_device", c_sz, C.c_int, C.c_uint, c_sz, c_vp, c_sz, c_vp, c_vp, c_vp, c_vp, c_vp)
    sig("FSEB200_frame_decompress_bound_device", c_sz, c_sz, c_vp, c_vp, c_vp, c_vp)
    sig("FSEB200_frame_decompress_device", c_sz, c_sz, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp)
    sig("FSEB200_XXH32", C.c_uint, c_vp, c_sz, C.c_uint)
    for name in ("FSEB200_HUF_compress_batch", "FSEB200_FSE_compress_batch", "FSEB200_FSE_decompress_batch",
                 "FSEB200_FSEU16_compress_batch", "FSEB200_FSEU16_decompress_batch"):
        if hasattr(L, name):
            if "decompress" in name:
                sig(name, c_sz, c_vp, c_sz, c_sz, c_vp, c_sz, c_vp, c_vp, c_vp, c_vp)
            else:
                sig(name, c_sz, c_vp, c_sz, c_vp, c_vp, c_sz, c_sz, C.c_uint, C.c_uint, c_vp)


from .batch import (huf_decompress_batch, huf_compress_batch, fse_compress_batch, fse_decompress_batch,  # noqa: E402,F401
                    fseu16_compress_batch, fseu16_decompress_batch, nblocks,
                    huf_compress_blocks, huf_decompress_blocks, block_pointers,
                    huf_compress1x_blocks, huf_decompress1x_blocks,
                    huf_compress_repeat_blocks, huf_compress1x_repeat_blocks,
                    huf_decompress_repeat_blocks, huf_decompress1x_repeat_blocks,
                    huf_compress_repeat_chains, huf_compress1x_repeat_chains,
                    huf_compress_repeat_chains_packed, huf_compress1x_repeat_chains_packed,
                    huf_decompress_repeat_packed, huf_decompress1x_repeat_packed,
                    huf_compress_mixed_repeat_chains, huf_decompress_mixed_repeat_blocks,
                    huf_compress_mixed_repeat_chains_packed, huf_decompress_mixed_repeat_packed,
                    huf_compress_literals_chains_packed, host_compress_literals_chains_packed,
                    huf_compress_packed, huf_compress1x_packed, packed_pointers,
                    fse_compress_blocks, fse_decompress_blocks, fseu16_compress_blocks, fseu16_decompress_blocks,
                    fse_compress_packed, fseu16_compress_packed, fse_decompress_packed, fseu16_decompress_packed,
                    fse_packed_workspace, huf_decompress_packed, huf_decompress1x_packed,
                    host_compress_packed, host_decompress_packed,
                    host_compress_repeat_chains_packed, host_decompress_repeat_packed,
                    host_compress_mixed_repeat_chains_packed, host_decompress_mixed_repeat_packed, frame_compress, frame_decompress,
                    frame_compress_batch, frame_decompress_batch, frame_compress_device, frame_decompress_device)
