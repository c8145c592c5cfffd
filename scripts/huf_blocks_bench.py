"""Huff0 through the per-block descriptor calls (FSEB200_HUF_*_blocks) against the uniform batch calls, on one GPU.

  (a) bench layout   1 GiB of probagen P14 in 32 KB blocks: the uniform calls, then the descriptor calls at
                     ptr = base + b * blockSize (same bytes, same kernels, a few descriptor loads per block more);
  (b) ragged layout  the same stream cut into seeded sizes uniform in [1 KiB, 128 KiB], sources back to back: encode into
                     bound-sized destinations, then decode from the compressed blocks packed back to back (packed outside the
                     timed region) into outputs back to back.  Also the share of streams per decode path and emit path.
  (c) small layout   the first 256 MiB of the stream cut into seeded sizes uniform in [64 B, 4 KiB], as (b).

A build with the single-stream descriptor calls (FSEB200_HUF_*1X_blocks) is also timed with them: a1_* in layout (a), b1_* in
(b), c1_* in (c), next to the 4X descriptor calls of the same run (c_* is 4X in layout (c)).

A build with the packed calls (FSEB200_HUF_compress[1X]_packed) times them right after the descriptor encode of the same layout
and format, on the same blocks (*_enc_packed, e.g. a_enc_packed next to a_enc_blocks, b1_enc_packed next to b1_enc), then decodes
every block from the packed buffer with the descriptor decoder and checks the source comes back (*_packed_decoded digests, equal
to a_source).  *_packed_share is packed bytes per source byte.  Layout (d) is 1 GiB of random bytes in 32 KB blocks, every block
raw: d_enc / d1_enc is the descriptor encode (which leaves raw blocks to the caller), d_enc_packed / d1_enc_packed the packed
one (copy included), d_copy a plain device-to-device copy of the same GiB.  Layouts (b) and (c) decode only
the blocks that compressed to a Huffman block (1 < cSize < size); every figure is scaled to ms per GiB of uncompressed bytes
that the call encodes or decodes.  `cpu_ref` is the compiled reference's single-thread HUF_compress1X / HUF_decompress1X_DCtx
on a sample of layout (a) (oracle/_ref/libfse_ref.so, skipped when it is absent), in the same units.

Builds are libraries given as LABEL=PATH (default: this tree's).  Each run of each build is a child process; builds alternate
run by run.  Prints one JSON line with the GPU's name, power limit and SM clock, per build and metric the median and range in
ms per GiB, and digests of the compressed and decoded bytes, so that builds can be checked to compute the same thing.

    python scripts/huf_blocks_bench.py --make-nohead build/variants/libfse_b200_nohead.so
    python scripts/huf_blocks_bench.py --runs 5 --build new=finitestateentropy_b200/libfse_b200.so \
        --build nohead=build/variants/libfse_b200_nohead.so

`--make-nohead PATH` compiles this tree's library with the project's nvcc flags plus -DFSEB200_HUFD_HEAD=0 (descriptor batches
decode misaligned segments per symbol) into PATH, the build the head decode is measured against.
"""
import argparse
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
GIB = 1 << 30
BLOCK = 32768


def ragged_sizes(total, seed=7, lo=1024, hi=128 * 1024):
    import numpy as np
    rng = np.random.default_rng(seed)
    sizes = rng.integers(lo, hi + 1, total // lo)
    ends = np.cumsum(sizes)
    k = int(np.searchsorted(ends, total))
    sizes = sizes[: k + 1].copy()
    sizes[-1] -= int(ends[k] - total)
    return [int(x) for x in sizes if x > 0]


def path_shares(sizes):
    """share of decode streams per path (head+fast / fast / symbol) and of emit streams per group width, for blocks back to back
    from a 512-byte aligned start (every block is a pass-A Huffman block for P14)"""
    from collections import Counter
    from blocks_paths import stream_paths, stream_kind, emit_groups
    dec, emit, off = Counter(), Counter(), 0
    for n in sizes:
        dec.update(stream_kind(*s) for s in stream_paths("A", n, off))
        emit.update(emit_groups(off, n))
        off += n
    nd, ne = sum(dec.values()), sum(emit.values())
    return {k: round(v / nd, 4) for k, v in dec.items()}, {k: round(v / ne, 4) for k, v in emit.items()}


def cpu_ref_rates(src_host, nblocks):
    """the compiled reference's single-thread HUF_compress1X / HUF_decompress1X_DCtx on the first nblocks 32 KB blocks: ms per GiB"""
    import time
    import numpy as np
    from helpers import REF_SO, load_ref
    if not os.path.exists(REF_SO):
        return None
    R = load_ref()
    bound = 129 + BLOCK + (BLOCK >> 8) + 8
    cbuf = np.zeros(nblocks * bound + 64, np.uint8)
    out = np.zeros(BLOCK + 64, np.uint8)
    dt = np.zeros(1 + 4096, np.uint32)
    p = lambda a, o=0: a.ctypes.data + o
    sizes = []
    t0 = time.perf_counter()
    for b in range(nblocks):
        sizes.append(R.HUF_compress1X(p(cbuf, b * bound), bound, p(src_host, b * BLOCK), BLOCK, 255, 12))
    t1 = time.perf_counter()
    for b in range(nblocks):
        dt[0] = 12 * 0x01000001
        assert R.HUF_decompress1X_DCtx(p(dt), p(out), BLOCK, p(cbuf, b * bound), sizes[b]) == BLOCK
    t2 = time.perf_counter()
    scale = GIB / (nblocks * BLOCK) * 1e3
    return {"enc1x": round((t1 - t0) * scale, 1), "dec1x": round((t2 - t1) * scale, 1), "sample_blocks": nblocks}


def child(lib_path, reps):
    import numpy as np
    import torch
    import finitestateentropy_b200 as fb
    L = C.CDLL(lib_path)
    fb.declare(L, fb.HEADER, [n for n in fb.prototypes(fb.HEADER) if hasattr(L, n)])   # an older build lacks the later calls
    have, have1x, have_packed = (hasattr(L, n) for n in ("FSEB200_HUF_compress_blocks", "FSEB200_HUF_compress1X_blocks",
                                                         "FSEB200_HUF_compress_packed"))
    dev = torch.device("cuda")
    stream = torch.cuda.current_stream().cuda_stream
    slot = 512 + BLOCK + (BLOCK >> 7) + 12
    src = torch.empty(GIB + 64, dtype=torch.uint8, device=dev)
    assert L.FSEB200_probagen(src.data_ptr(), GIB, 0, 0.14, stream) == 0
    nb = GIB // BLOCK

    def timed(fn):
        fn()                                                            # warm-up (module load, scratch growth)
        ts = []
        for _ in range(reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(); fn(); b.record(); b.synchronize()
            ts.append(a.elapsed_time(b))
        return sorted(ts)[len(ts) // 2]

    def t64(a):
        return torch.tensor(np.asarray(a, dtype=np.int64), device=dev)

    out = {}
    cbuf = torch.empty(nb * slot + 64, dtype=torch.uint8, device=dev)
    cs = torch.empty(nb, dtype=torch.int64, device=dev)
    dst = torch.empty(GIB, dtype=torch.uint8, device=dev)
    res = torch.empty(nb, dtype=torch.int64, device=dev)
    out["a_enc_uniform"] = timed(lambda: L.FSEB200_HUF_compress_batch(cbuf.data_ptr(), slot, cs.data_ptr(), src.data_ptr(), GIB, BLOCK, 255, 12, stream))
    out["a_dec_uniform"] = timed(lambda: L.FSEB200_HUF_decompress_batch(dst.data_ptr(), GIB, BLOCK, cbuf.data_ptr(), slot, cs.data_ptr(), res.data_ptr(), None, stream))
    assert torch.equal(dst, src[:GIB])
    used = torch.arange(slot, device=dev)[None, :] < cs[:, None]          # bytes [0, cSize) of each slot: the rest is unspecified
    digest = {"a_cbuf": hashlib.sha256(cbuf[: nb * slot].view(nb, slot)[used].cpu().numpy().tobytes()).hexdigest()[:16]}
    del used
    if have:
        b = np.arange(nb, dtype=np.int64)
        sp, sn = t64(src.data_ptr() + b * BLOCK), t64(np.full(nb, BLOCK))
        dp, dc = t64(cbuf.data_ptr() + b * slot), t64(np.full(nb, slot))
        cs2 = torch.empty_like(cs)
        out["a_enc_blocks"] = timed(lambda: L.FSEB200_HUF_compress_blocks(nb, dp.data_ptr(), dc.data_ptr(), cs2.data_ptr(), sp.data_ptr(), sn.data_ptr(), 255, 12, stream))
        assert torch.equal(cs, cs2)
        op = t64(dst.data_ptr() + b * BLOCK)
        dst.zero_()
        out["a_dec_blocks"] = timed(lambda: L.FSEB200_HUF_decompress_blocks(nb, op.data_ptr(), sn.data_ptr(), res.data_ptr(), dp.data_ptr(), cs2.data_ptr(), stream))
        assert torch.equal(dst, src[:GIB]) and bool((res == BLOCK).all())
        if have1x:                                                      # (a) in the single-stream format, into the same slots
            cs1 = torch.empty_like(cs)
            out["a1_enc"] = timed(lambda: L.FSEB200_HUF_compress1X_blocks(nb, dp.data_ptr(), dc.data_ptr(), cs1.data_ptr(), sp.data_ptr(), sn.data_ptr(), 255, 12, stream))
            assert bool(((cs1 > 1) & (cs1 < BLOCK)).all())
            used = torch.arange(slot, device=dev)[None, :] < cs1[:, None]
            digest["a1_cbuf"] = hashlib.sha256(cbuf[: nb * slot].view(nb, slot)[used].cpu().numpy().tobytes()).hexdigest()[:16]
            del used
            dst.zero_()
            out["a1_dec"] = timed(lambda: L.FSEB200_HUF_decompress1X_blocks(nb, op.data_ptr(), sn.data_ptr(), res.data_ptr(), dp.data_ptr(), cs1.data_ptr(), stream))
            assert torch.equal(dst, src[:GIB]) and bool((res == BLOCK).all())
        del cbuf

        def sha(t):
            return hashlib.sha256(t.cpu().numpy().tobytes()).hexdigest()[:16]

        def pack_run(key, fn, dec, sp, sn, offs, total):
            """the packed call on blocks (sp, sn) into one buffer, then every block decoded from it with the descriptor decoder"""
            n = sn.numel()
            pout = torch.empty(total + 32, dtype=torch.uint8, device=dev)
            poffs = torch.empty(n + 1, dtype=torch.int64, device=dev)
            pcs = torch.empty(n, dtype=torch.int64, device=dev)
            out[key + "_enc_packed"] = timed(lambda: fn(n, pout.data_ptr(), pout.numel(), poffs.data_ptr(), pcs.data_ptr(), sp.data_ptr(),
                                                        sn.data_ptr(), 255, 12, stream)) * GIB / total
            used = int(poffs[-1])
            out[key + "_packed_share"] = round(used / total, 4)           # packed bytes per source byte
            digest[key + "_packed_out"] = sha(pout[:used])
            dst.zero_()
            pres = torch.empty(n, dtype=torch.int64, device=dev)
            # the descriptor arrays stay referenced until the call is enqueued: a temporary freed while the argument list is built
            # would hand its memory to the next one
            od, cp, cl = t64(dst.data_ptr() + offs), poffs[:-1] + pout.data_ptr(), poffs[1:] - poffs[:-1]
            assert dec(n, od.data_ptr(), sn.data_ptr(), pres.data_ptr(), cp.data_ptr(), cl.data_ptr(), stream) == 0
            assert torch.equal(pres, sn) and torch.equal(dst[:total], src[:total])
            digest[key + "_packed_decoded"] = sha(dst[:total])

        if have_packed:                                                 # (a) packed, next to a_enc_blocks / a1_enc of this run
            pack_run("a", L.FSEB200_HUF_compress_packed, L.FSEB200_HUF_decompress_blocks, sp, sn, b * BLOCK, GIB)
            pack_run("a1", L.FSEB200_HUF_compress1X_packed, L.FSEB200_HUF_decompress1X_blocks, sp, sn, b * BLOCK, GIB)
            digest["a_source"] = sha(src[:GIB])

        def ragged(key, enc, dec, sizes, pk=None):
            """encode blocks back to back into bound-sized destinations, pack the Huffman blocks back to back, decode them"""
            n = len(sizes)
            total = int(sum(sizes))
            offs = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.int64)
            bounds = np.array([129 + s + (s >> 8) + 8 for s in sizes], np.int64)
            boffs = np.concatenate([[0], np.cumsum(bounds)[:-1]]).astype(np.int64)
            carena = torch.empty(int(bounds.sum()) + 64, dtype=torch.uint8, device=dev)
            rsp, rsn = t64(src.data_ptr() + offs), t64(sizes)
            rdp, rdc = t64(carena.data_ptr() + boffs), t64(bounds)
            rcs = torch.empty(n, dtype=torch.int64, device=dev)
            out[key + "_enc"] = timed(lambda: enc(n, rdp.data_ptr(), rdc.data_ptr(), rcs.data_ptr(), rsp.data_ptr(), rsn.data_ptr(), 255, 12, stream)) * GIB / total
            csz = rcs.cpu().numpy()
            sz_np = np.array(sizes, np.int64)
            keep = np.nonzero((csz > 1) & (csz < sz_np))[0]             # Huffman blocks (error codes are huge as u64, negative here)
            kc, kn = csz[keep], sz_np[keep]
            poffs = np.concatenate([[0], np.cumsum(kc)[:-1]]).astype(np.int64)
            src_idx = torch.repeat_interleave(t64(boffs[keep] - poffs), t64(kc)) + torch.arange(int(kc.sum()), device=dev)
            packed = torch.empty(int(kc.sum()) + 64, dtype=torch.uint8, device=dev)
            packed[: int(kc.sum())] = carena[src_idx]                   # packing: outside the timed region
            del carena, src_idx
            digest[key + "_packed"] = hashlib.sha256(packed[: int(kc.sum())].cpu().numpy().tobytes()).hexdigest()[:16]
            pp, pcs = t64(packed.data_ptr() + poffs), t64(kc)
            od, on = t64(dst.data_ptr() + offs[keep]), t64(kn)
            rres = torch.empty(len(keep), dtype=torch.int64, device=dev)
            dst.zero_()
            out[key + "_dec"] = timed(lambda: dec(len(keep), od.data_ptr(), on.data_ptr(), rres.data_ptr(), pp.data_ptr(), pcs.data_ptr(), stream)) * GIB / int(kn.sum())
            assert torch.equal(rres, on)
            ok = torch.zeros(GIB, dtype=torch.bool, device=dev)
            ok[torch.repeat_interleave(t64(offs[keep]), t64(kn)) + torch.arange(int(kn.sum()), device=dev) - torch.repeat_interleave(t64(np.concatenate([[0], np.cumsum(kn)[:-1]])), t64(kn))] = True
            assert torch.equal(dst[ok], src[:GIB][ok])
            out[key + "_count"] = n
            out[key + "_huffman_share"] = round(float(kn.sum()) / total, 4)
            if pk is not None:
                del ok
                pack_run(key, pk, dec, rsp, rsn, offs, total)

        layouts = {"b": ragged_sizes(GIB), "c": ragged_sizes(GIB // 4, seed=9, lo=64, hi=4096)}
        for lay, sizes in layouts.items():
            ragged(lay, L.FSEB200_HUF_compress_blocks, L.FSEB200_HUF_decompress_blocks, sizes,
                   L.FSEB200_HUF_compress_packed if have_packed else None)
            if have1x:
                ragged(lay + "1", L.FSEB200_HUF_compress1X_blocks, L.FSEB200_HUF_decompress1X_blocks, sizes,
                       L.FSEB200_HUF_compress1X_packed if have_packed else None)
        if have1x:
            out["cpu_ref"] = cpu_ref_rates(src[: 512 * BLOCK].cpu().numpy(), 512)
        if have_packed:                                                 # (d) 1 GiB of random bytes in 32 KB blocks: every block raw
            gen = torch.Generator(device=dev)
            gen.manual_seed(11)
            src[:GIB] = torch.randint(0, 256, (GIB,), dtype=torch.uint8, device=dev, generator=gen)
            cbuf = torch.empty(nb * slot + 64, dtype=torch.uint8, device=dev)
            ddp = t64(cbuf.data_ptr() + b * slot)
            for key, enc, pk, dec in (("d", L.FSEB200_HUF_compress_blocks, L.FSEB200_HUF_compress_packed, L.FSEB200_HUF_decompress_blocks),
                                      ("d1", L.FSEB200_HUF_compress1X_blocks, L.FSEB200_HUF_compress1X_packed, L.FSEB200_HUF_decompress1X_blocks)):
                out[key + "_enc"] = timed(lambda: enc(nb, ddp.data_ptr(), dc.data_ptr(), cs2.data_ptr(), sp.data_ptr(), sn.data_ptr(), 255, 12, stream))
                assert bool((cs2 == 0).all())                           # the descriptor call leaves the raw blocks to its caller
                pack_run(key, pk, dec, sp, sn, b * BLOCK, GIB)
            out["d_copy"] = timed(lambda: dst.copy_(src[:GIB]))           # a plain device-to-device copy of the same bytes
            del cbuf
    print(json.dumps({"ms": out, "digest": digest}))


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--build", action="append", default=[], help="LABEL=path/to/libfse_b200.so (repeatable)")
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3, help="timed calls per metric and run (median taken)")
    ap.add_argument("--child", default=None)
    ap.add_argument("--make-nohead", metavar="PATH", default=None, help="build the library without the head decode into PATH and exit")
    a = ap.parse_args()
    if a.make_nohead:
        sys.path.insert(0, ROOT)
        from finitestateentropy_b200 import _build
        import glob
        os.makedirs(os.path.dirname(os.path.abspath(a.make_nohead)), exist_ok=True)
        nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
        srcs = sorted(glob.glob(os.path.join(_build.CSRC, "*.cu")))
        subprocess.check_call([nvcc] + _build.NVCC_FLAGS + ["-DFSEB200_HUFD_HEAD=0", "-I", os.path.join(ROOT, "include"),
                               "-o", a.make_nohead] + srcs)
        return
    if a.child:
        child(a.child, a.reps)
        return
    builds = [b.split("=", 1) for b in a.build] or [["this", os.path.join(ROOT, "finitestateentropy_b200", "libfse_b200.so")]]
    runs = {lab: [] for lab, _ in builds}
    info_before = gpu_info()
    for _ in range(a.runs):
        for lab, path in builds:
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", os.path.abspath(path), "--reps", str(a.reps)],
                               capture_output=True, text=True)
            assert r.returncode == 0, (lab, r.stderr[-3000:])
            runs[lab].append(json.loads(r.stdout.strip().splitlines()[-1]))
            print(lab, r.stdout.strip().splitlines()[-1], file=sys.stderr)   # every run's raw figures
    summary = {}
    for lab, rs in runs.items():
        ms = {}
        for k in rs[0]["ms"]:
            if k.endswith("_count") or k.endswith("_share"):                 # block counts and Huffman shares: the same every run
                ms[k] = rs[0]["ms"][k]
                continue
            if k == "cpu_ref":                                              # medians of the reference's rates
                ms[k] = rs[0]["ms"][k] and {m: sorted(x["ms"][k][m] for x in rs)[len(rs) // 2] for m in rs[0]["ms"][k]}
                continue
            v = sorted(x["ms"][k] for x in rs)                           # per GiB: every layout moves 1 GiB uncompressed
            ms[k] = {"median": round(v[len(v) // 2], 3), "min": round(v[0], 3), "max": round(v[-1], 3)}
        summary[lab] = {"ms_per_gib": ms, "digests": sorted({json.dumps(x["digest"], sort_keys=True) for x in rs})}
    dec, emit = path_shares(ragged_sizes(GIB))
    print(json.dumps({"gpu": info_before, "gpu_after": gpu_info(), "runs": a.runs, "builds": summary,
                      "ragged_blocks": len(ragged_sizes(GIB)), "ragged_decode_stream_paths": dec, "ragged_emit_stream_groups": emit}))


if __name__ == "__main__":
    main()
