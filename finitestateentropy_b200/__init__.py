"""finitestateentropy_b200 -- H100-native (sm_90a) block entropy coding: the FSE / Huff0 32 KB block
hot path of Cyan4973/FiniteStateEntropy behind the reference's own C API.

The product is `libfse_b200.so` (hand-written CUDA kernels + a C-ABI, see include/fse_b200.h).  This
package is only the thin Python binding used by tests/ and bench.py: ctypes over the C-ABI, torch for
device memory / streams / torch.distributed.  There is NO CPU implementation here: if the CUDA
library is missing, importing `lib()` raises."""
import ctypes as C
import os
import re

from . import _build

_HERE = os.path.dirname(os.path.abspath(__file__))
HEADER = os.path.join(os.path.dirname(_HERE), "include", "fse_b200.h")
_LIB = None

# the scalar C types prototypes() maps; any pointer is c_void_p, except a `const char*` return (c_char_p)
_SCALARS = {"size_t": C.c_size_t, "unsigned": C.c_uint, "int": C.c_int, "double": C.c_double, "unsigned char": C.c_ubyte,
            "uint32_t": C.c_uint32, "uint64_t": C.c_uint64}
# words that are part of a type, never a parameter's name: `unsigned long` or `int size_t` raises rather than losing a word
_C_TYPE_WORDS = {"void", "char", "short", "int", "long", "float", "double", "signed", "unsigned", "struct", "union", "enum"} | set(_SCALARS)

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
    """Loads (building in-tree first if needed) the CUDA library, every prototype of include/fse_b200.h declared on it.  Fails
    loudly; never falls back."""
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
        declare(L, HEADER)
        _LIB = L
    return _LIB


def _ctype(decl, name, is_return):
    """ctypes type of a C return type, or of a parameter declaration (its name, if any, last)"""
    t = " ".join(re.sub(r"\bconst\b", " ", decl).split())
    if "*" in t:
        return C.c_char_p if is_return and t.replace(" ", "") == "char*" else C.c_void_p
    if is_return and t == "void":
        return None
    if not is_return and t not in _SCALARS:
        head, _, last = t.rpartition(" ")
        if re.fullmatch(r"[A-Za-z_]\w*", last) and last not in _C_TYPE_WORDS:    # the parameter's name
            t = head
    if t not in _SCALARS:
        raise ValueError("%s: no ctypes mapping for the C type %r" % (name, decl.strip()))
    return _SCALARS[t]


def prototypes(header_path):
    """{name: (restype, argtypes)} of every `ret name(args);` prototype in a C header.  Comments and preprocessor lines are
    ignored; a statement that is not such a prototype, or a type without a mapping, raises."""
    text = open(header_path).read()
    text = re.sub(r"/\*.*?\*/|//[^\n]*", " ", text, flags=re.S)
    text = re.sub(r"^[ \t]*#.*$", " ", text, flags=re.M)
    out = {}
    for stmt in text.split(";"):
        stmt = re.split(r"[{}]", stmt)[-1].strip()    # what follows `extern "C" {` or an enum's braces
        if not stmt:
            continue
        m = re.fullmatch(r"([\w\s*]+?)\s*\b(\w+)\s*\(([^()]*)\)", stmt)
        if not m:
            raise ValueError("%s: not a prototype: %r" % (header_path, stmt))
        ret, name, args = m.groups()
        args = [] if args.strip() in ("", "void") else args.split(",")
        out[name] = (_ctype(ret, name, True), [_ctype(a, name, False) for a in args])
    return out


def declare(lib, header_path, names=None):
    """Sets restype and argtypes on the ctypes.CDLL `lib` for every prototype of `header_path` (only `names`, if given).  A name
    the library does not export raises AttributeError."""
    protos = prototypes(header_path)
    for name in protos if names is None else names:
        f = getattr(lib, name)
        f.restype, f.argtypes = protos[name]
    return lib


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
