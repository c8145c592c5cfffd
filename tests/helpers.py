"""Shared test plumbing: loads the two CPU checkers (oracle port, compiled reference) with ctypes
and builds the input zoo modelled on the reference fuzzers' buffers
(programs/fuzzer.c:157-161: noise, P=1%, 15%, 90%, constant)."""
import ctypes as C
import os
import subprocess
import sys
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:                 # tests/golden/make_golden.py and the scripts put only tests/ on the path
    sys.path.insert(0, ROOT)
import finitestateentropy_b200 as fb     # noqa: E402
ORACLE_DIR = os.path.join(ROOT, "oracle")
PORT_SO = os.path.join(ORACLE_DIR, "_build", "libfse_oracle.so")
REF_SO = os.path.join(ORACLE_DIR, "_ref", "libfse_ref.so")

sz = C.c_size_t
vp = C.c_void_p
u = C.c_uint
ERR_MAX = 9


def is_error(r):
    return r > (2 ** 64 - ERR_MAX)


def err_code(r):
    return (2 ** 64 - r) if is_error(r) else 0


def declared_arity():
    """{name: parameter count} of every prototype the binding reads from include/fse_b200.h"""
    return {n: len(args) for n, (_, args) in fb.prototypes(fb.HEADER).items()}


def _sig(fn, res, *args):
    fn.restype = res
    fn.argtypes = list(args)
    return fn


_port = None
_ref = None


def load_port():
    """our plain-C restatement (always buildable: gcc only), declared from oracle/fse_oracle.h"""
    global _port
    if _port is None:
        src = os.path.join(ORACLE_DIR, "fse_oracle.c")
        if (not os.path.exists(PORT_SO)) or os.path.getmtime(PORT_SO) < os.path.getmtime(src):
            subprocess.check_call(["make", "-s", "-C", ORACLE_DIR, "port"])
        _port = fb.declare(C.CDLL(PORT_SO), os.path.join(ORACLE_DIR, "fse_oracle.h"))
    return _port


def have_ref():
    return os.path.exists(REF_SO) or os.path.isdir("/root/reference/lib")


def load_ref():
    """the unmodified reference library compiled by oracle/Makefile (None if it cannot be had).  Its calls are declared from
    include/fse_b200.h, which states the reference API's prototypes (tests/golden/ref_prototype_arity.json pins their arity);
    the few it does not state are declared here."""
    global _ref
    if _ref is None:
        if not os.path.exists(REF_SO):
            if not os.path.isdir("/root/reference/lib"):
                return None
            subprocess.check_call(["make", "-s", "-C", ORACLE_DIR, "ref"])
        L = C.CDLL(REF_SO)
        fb.declare(L, fb.HEADER, [n for n in fb.prototypes(fb.HEADER) if n.startswith(("FSE_", "HUF_", "HIST_")) and hasattr(L, n)])
        _sig(L.FSE_buildCTableU16, sz, vp, vp, u, u)
        _sig(L.FSE_buildDTableU16, sz, vp, vp, u, u)
        _sig(L.FSE_compressU16_usingCTable, sz, vp, sz, vp, sz, vp)
        for name in ("HUF_decompress4X1_DCtx", "HUF_decompress1X1_DCtx", "HUF_decompress1X_DCtx"):
            _sig(getattr(L, name), sz, vp, vp, sz, vp, sz)
        _sig(L.refshim_compress_blocks, C.c_double, C.c_int, vp, sz, sz, vp, sz, vp, u, u, C.c_int)
        _sig(L.refshim_decompress_blocks, C.c_double, C.c_int, vp, vp, sz, sz, vp, sz, vp, vp, C.c_int)
        _ref = L
    return _ref


def ptr(a):
    """raw pointer of a numpy array / bytearray as c_void_p"""
    if isinstance(a, np.ndarray):
        return a.ctypes.data_as(vp)
    return C.cast((C.c_char * len(a)).from_buffer(a), vp)


def probagen(n, p):
    out = np.empty(n, dtype=np.uint8)
    load_port().orc_probagen(ptr(out), n, float(p))
    return out


def gen_u16(n, start=240, p=0.5, seed=1):
    out = np.empty(n, dtype=np.uint16)
    load_port().orc_gen_u16(ptr(out), n, start, float(p), seed)
    return out


def zoo(rng, n):
    """one random buffer of length n from the fuzzers' buffer zoo (+ a few nastier shapes)"""
    kind = int(rng.integers(0, 9))
    if kind == 0:
        return rng.integers(0, 256, n, dtype=np.uint8)                      # noise
    if kind == 1:
        return np.full(n, int(rng.integers(0, 256)), dtype=np.uint8)        # constant (RLE)
    if kind in (2, 3, 4):
        p = [0.01, 0.15, 0.90][kind - 2]
        off = int(rng.integers(0, 1 << 16))
        return probagen(off + n, p)[off:]
    if kind == 5:                                                          # geometric over a random alphabet
        k = int(rng.integers(2, 257))
        q = float(rng.uniform(0.02, 0.6))
        v = np.minimum(rng.geometric(q, n) - 1, k - 1).astype(np.uint8)
        perm = rng.permutation(256).astype(np.uint8)
        return perm[v]
    if kind == 6:                                                          # few symbols, one dominant
        v = (rng.random(n) < float(rng.uniform(0.001, 0.2))).astype(np.uint8) * rng.integers(1, 256, n, dtype=np.uint8)
        return v
    if kind == 7:                                                          # zipf-like, wide alphabet (deep Huffman trees)
        w = 1.0 / np.arange(1, 257) ** float(rng.uniform(0.8, 2.5))
        return rng.choice(256, n, p=w / w.sum()).astype(np.uint8)
    v = rng.integers(0, int(rng.integers(2, 40)), n, dtype=np.uint8)      # small flat alphabet
    return v


def rand_size(rng, hi=128 * 1024):
    r = rng.random()
    if r < 0.25:
        return int(rng.integers(0, 64))
    if r < 0.5:
        return int(rng.integers(64, 4096))
    return int(rng.integers(4096, hi + 1))
