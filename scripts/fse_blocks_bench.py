"""FSE and FSE-U16 through the per-block descriptor calls (FSEB200_FSE{,U16}_*_blocks) against the uniform batch calls, on one GPU.

  (a) bench layout   1 GiB of the bench.py inputs -- FSE: probagen P80, (255, 12), slot FSE_compressBound(32768); U16:
                     generateU16(240, 0.50, 1), (0, 12), slot 32768 -- in 32 KB blocks: the uniform calls, then the descriptor
                     calls at ptr = base + b * blockSize;
  (b) ragged layout  the same stream cut into seeded sizes uniform in [1 KiB, 128 KiB] (U16: even byte counts), sources back
                     to back: encode into bound-sized destinations, then decode from the compressed blocks packed back to back
                     (packed outside the timed region) into outputs back to back.  Also the share of blocks per encode kernel.
  (c) random layout  FSE only: 1 GiB of random bytes in 32 KB blocks, every block raw.  c_enc_blocks is the descriptor encode
                     (which leaves raw blocks to the caller), c_copy a plain device-to-device copy of the same GiB.  (A U16
                     block is never raw: its symbols hold at most log2(287) bits of 16.)

The packed calls (FSEB200_FSE{,U16}_{compress,decompress}_packed) are timed alternated with the descriptor calls on the same
blocks: *_pk_enc_packed next to *_pk_enc_blocks (descriptor encode into bound-sized destinations), *_pk_dec_packed next to
*_pk_dec_blocks (descriptor decode of the same compressed bytes); c_enc_packed / c_dec_packed for layout (c).  The packed buffer
must equal the compressed blocks packed back to back (a_compressed, b_packed digests) and decode to the source.

Each run is a child process per codec; within a child the uniform and descriptor calls alternate, each metric the median of
--reps timed calls.  Prints one JSON line with the GPU's name, power limit and SM clock, per codec and metric the median and
range over runs in ms per GiB, and digests of the compressed and decoded bytes.

    python scripts/fse_blocks_bench.py --runs 5 [--codecs fse]
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


def fbound(n):
    return 512 + n + (n >> 7) + 12


def ragged_sizes(total, wide, seed=7):
    import numpy as np
    rng = np.random.default_rng(seed)
    sizes = rng.integers(1024, 128 * 1024 + 1, total // 1024)
    if wide:
        sizes &= ~1
    ends = np.cumsum(sizes)
    k = int(np.searchsorted(ends, total))
    sizes = sizes[: k + 1].copy()
    sizes[-1] -= int(ends[k] - total)
    if sizes[-1] < 1024:                                                # no tiny last block: every block compresses
        sizes[-2] += sizes[-1]
        sizes = sizes[:-1]
    return [int(x) for x in sizes]


def encoder_shares(sizes, wide):
    """share of blocks per encode kernel for sources back to back from a 256-byte aligned start (fse_blocks_paths.encode_route)"""
    from collections import Counter
    from fse_blocks_paths import encode_route
    c, off = Counter(), 0
    for n in sizes:
        c[encode_route(off, n // 2 if wide else n, wide)] += 1
        off += n
    return {k: round(v / len(sizes), 4) for k, v in c.items()}


def child(codec, reps):
    import numpy as np
    import torch
    import finitestateentropy_b200 as fb
    L = fb.declare(C.CDLL(os.path.join(ROOT, "finitestateentropy_b200", "libfse_b200.so")), fb.HEADER)
    wide = codec == "u16"
    w = 2 if wide else 1
    name = "FSEU16" if wide else "FSE"
    msv = 0 if wide else 255
    slot = 32768 if wide else fbound(BLOCK)
    dev = torch.device("cuda")
    stream = torch.cuda.current_stream().cuda_stream
    src = torch.empty(GIB + 64, dtype=torch.uint8, device=dev)
    gen = (lambda: L.FSEB200_genU16(src.data_ptr(), GIB // 2, 0, 240, 0.5, 1, stream)) if wide else \
          (lambda: L.FSEB200_probagen(src.data_ptr(), GIB, 0, 0.80, stream))
    assert gen() == 0
    nb = GIB // BLOCK
    f = {k: getattr(L, "FSEB200_%s_%s" % (name, k)) for k in ("compress_batch", "decompress_batch", "compress_blocks", "decompress_blocks",
                                                               "compress_packed", "decompress_packed")}

    def t64(a):
        return torch.tensor(np.asarray(a, dtype=np.int64), device=dev)

    def timed_pair(fa, fb_):
        fa(); fb_()                                                     # warm-up (module load, scratch growth)
        ta, tb = [], []
        for _ in range(reps):
            for fn, ts in ((fa, ta), (fb_, tb)):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(); fn(); b.record(); b.synchronize()
                ts.append(a.elapsed_time(b))
        return sorted(ta)[len(ta) // 2], sorted(tb)[len(tb) // 2]

    class Packed:
        """one packed buffer for n blocks of `nbytes` source bytes in all, and its calls"""
        def __init__(self, n, sp, sn, nbytes):
            self.n, self.sp, self.sn = n, sp, sn
            self.out = torch.empty(nbytes + 32, dtype=torch.uint8, device=dev)
            self.wsz = L.FSEB200_FSE_packed_workspace(n, nbytes)
            self.work = torch.empty(self.wsz, dtype=torch.uint8, device=dev)
            self.offs = torch.empty(n + 1, dtype=torch.int64, device=dev)
            self.cs = torch.empty(n, dtype=torch.int64, device=dev)
            self.res = torch.empty(n, dtype=torch.int64, device=dev)

        def enc(self):
            assert f["compress_packed"](self.n, self.out.data_ptr(), self.out.numel(), self.offs.data_ptr(), self.cs.data_ptr(),
                                        self.sp.data_ptr(), self.sn.data_ptr(), msv, 12, self.work.data_ptr(), self.wsz, stream) == 0

        def dec(self, dptrs):
            assert f["decompress_packed"](self.n, dptrs.data_ptr(), self.sn.data_ptr(), self.res.data_ptr(), self.out.data_ptr(),
                                          self.offs.data_ptr(), stream) == 0

        def digest(self):
            return hashlib.sha256(self.out[: int(self.offs[-1])].cpu().numpy().tobytes()).hexdigest()[:16]

    out, digest = {}, {}
    cbuf = torch.zeros(nb * slot + 64, dtype=torch.uint8, device=dev)
    cbuf2 = torch.zeros_like(cbuf)
    cs, cs2 = torch.empty(nb, dtype=torch.int64, device=dev), torch.empty(nb, dtype=torch.int64, device=dev)
    b = np.arange(nb, dtype=np.int64)
    sp, sn = t64(src.data_ptr() + b * BLOCK), t64(np.full(nb, BLOCK // w))
    dp, dc = t64(cbuf2.data_ptr() + b * slot), t64(np.full(nb, slot))
    out["a_enc_uniform"], out["a_enc_blocks"] = timed_pair(
        lambda: f["compress_batch"](cbuf.data_ptr(), slot, cs.data_ptr(), src.data_ptr(), GIB, BLOCK, msv, 12, stream),
        lambda: f["compress_blocks"](nb, dp.data_ptr(), dc.data_ptr(), cs2.data_ptr(), sp.data_ptr(), sn.data_ptr(), msv, 12, stream))
    assert torch.equal(cs, cs2) and bool((cs > 1).all())
    used = torch.arange(slot, device=dev)[None, :] < cs[:, None]          # bytes [0, cSize) of each slot: the rest is unspecified
    h1 = hashlib.sha256(cbuf[: nb * slot].view(nb, slot)[used].cpu().numpy().tobytes()).hexdigest()[:16]
    h2 = hashlib.sha256(cbuf2[: nb * slot].view(nb, slot)[used].cpu().numpy().tobytes()).hexdigest()[:16]
    assert h1 == h2
    digest["a_compressed"] = h1
    pka = Packed(nb, sp, sn, GIB)
    out["a_pk_enc_blocks"], out["a_pk_enc_packed"] = timed_pair(
        lambda: f["compress_blocks"](nb, dp.data_ptr(), dc.data_ptr(), cs2.data_ptr(), sp.data_ptr(), sn.data_ptr(), msv, 12, stream), pka.enc)
    assert torch.equal(pka.cs, cs) and pka.digest() == h1
    del used, cbuf2, pka.work
    dst = torch.zeros(GIB, dtype=torch.uint8, device=dev)
    dst2 = torch.zeros(GIB, dtype=torch.uint8, device=dev)
    res, res2 = torch.empty(nb, dtype=torch.int64, device=dev), torch.empty(nb, dtype=torch.int64, device=dev)
    cp, op = t64(cbuf.data_ptr() + b * slot), t64(dst2.data_ptr() + b * BLOCK)
    out["a_dec_uniform"], out["a_dec_blocks"] = timed_pair(
        lambda: f["decompress_batch"](dst.data_ptr(), GIB, BLOCK, cbuf.data_ptr(), slot, cs.data_ptr(), res.data_ptr(), None, stream),
        lambda: f["decompress_blocks"](nb, op.data_ptr(), sn.data_ptr(), res2.data_ptr(), cp.data_ptr(), cs.data_ptr(), stream))
    assert torch.equal(dst, src[:GIB]) and torch.equal(dst2, src[:GIB]) and torch.equal(res // w, res2)
    digest["a_decoded"] = hashlib.sha256(dst.cpu().numpy().tobytes()).hexdigest()[:16]
    dst.zero_()
    da = t64(dst.data_ptr() + b * BLOCK)
    out["a_pk_dec_blocks"], out["a_pk_dec_packed"] = timed_pair(
        lambda: f["decompress_blocks"](nb, op.data_ptr(), sn.data_ptr(), res2.data_ptr(), cp.data_ptr(), cs.data_ptr(), stream),
        lambda: pka.dec(da))
    assert torch.equal(dst, src[:GIB]) and torch.equal(pka.res, sn)
    digest["a_pk_decoded"] = hashlib.sha256(dst.cpu().numpy().tobytes()).hexdigest()[:16]
    del cbuf, dst2, pka
    # (b) ragged
    sizes = ragged_sizes(GIB, wide)
    n = len(sizes)
    offs = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.int64)
    bounds = np.array([fbound(s) for s in sizes], np.int64)
    boffs = np.concatenate([[0], np.cumsum(bounds)[:-1]]).astype(np.int64)
    carena = torch.empty(int(bounds.sum()) + 64, dtype=torch.uint8, device=dev)
    rsp, rsn = t64(src.data_ptr() + offs), t64(np.array(sizes) // w)
    rdp, rdc = t64(carena.data_ptr() + boffs), t64(bounds)
    rcs = torch.empty(n, dtype=torch.int64, device=dev)
    enc = lambda: f["compress_blocks"](n, rdp.data_ptr(), rdc.data_ptr(), rcs.data_ptr(), rsp.data_ptr(), rsn.data_ptr(), msv, 12, stream)   # noqa: E731
    out["b_enc"], _ = timed_pair(enc, lambda: None)
    pkb = Packed(n, rsp, rsn, GIB)
    out["b_pk_enc_blocks"], out["b_pk_enc_packed"] = timed_pair(enc, pkb.enc)
    assert torch.equal(pkb.cs, rcs)
    del pkb.work
    csz = rcs.cpu().numpy()
    assert (csz > 1).all() and (csz < np.array(sizes)).all()
    poffs = np.concatenate([[0], np.cumsum(csz)[:-1]]).astype(np.int64)
    packed = torch.empty(int(csz.sum()) + 64, dtype=torch.uint8, device=dev)
    for i in range(n):                                                  # packing: outside the timed region
        packed[poffs[i]: poffs[i] + csz[i]].copy_(carena[boffs[i]: boffs[i] + csz[i]])
    del carena
    digest["b_packed"] = hashlib.sha256(packed[: int(csz.sum())].cpu().numpy().tobytes()).hexdigest()[:16]
    pp, od = t64(packed.data_ptr() + poffs), t64(dst.data_ptr() + offs)
    rres = torch.empty(n, dtype=torch.int64, device=dev)
    dst.zero_()
    dec = lambda: f["decompress_blocks"](n, od.data_ptr(), rsn.data_ptr(), rres.data_ptr(), pp.data_ptr(), rcs.data_ptr(), stream)   # noqa: E731
    out["b_dec"], _ = timed_pair(dec, lambda: None)
    assert torch.equal(dst, src[:GIB]) and torch.equal(rres, rsn)
    dst.zero_()
    out["b_pk_dec_blocks"], out["b_pk_dec_packed"] = timed_pair(dec, lambda: pkb.dec(od))
    assert torch.equal(dst, src[:GIB]) and torch.equal(pkb.res, rsn) and pkb.digest() == digest["b_packed"]
    digest["b_pk_decoded"] = hashlib.sha256(dst.cpu().numpy().tobytes()).hexdigest()[:16]
    del pkb, packed
    if not wide:                                                        # (c) random bytes: every block raw
        rnd = torch.randint(0, 256, (GIB,), dtype=torch.uint8, device=dev, generator=torch.Generator(device=dev).manual_seed(5))
        rp = t64(rnd.data_ptr() + b * BLOCK)
        cbuf = torch.empty(nb * slot + 64, dtype=torch.uint8, device=dev)
        dp = t64(cbuf.data_ptr() + b * slot)
        pkc = Packed(nb, rp, sn, GIB)
        out["c_enc_blocks"], out["c_enc_packed"] = timed_pair(
            lambda: f["compress_blocks"](nb, dp.data_ptr(), dc.data_ptr(), cs2.data_ptr(), rp.data_ptr(), sn.data_ptr(), msv, 12, stream), pkc.enc)
        assert bool((cs2 == 0).all()) and bool((pkc.cs == 0).all()) and torch.equal(pkc.out[:GIB], rnd)
        del cbuf, pkc.work
        out["c_copy"], out["c_dec_packed"] = timed_pair(lambda: dst.copy_(rnd), lambda: pkc.dec(da))
        assert torch.equal(dst, rnd) and torch.equal(pkc.res, sn)
        digest["c_source"] = hashlib.sha256(rnd.cpu().numpy().tobytes()).hexdigest()[:16]
        digest["c_pk_decoded"] = hashlib.sha256(dst.cpu().numpy().tobytes()).hexdigest()[:16]
    print(json.dumps({"ms": out, "digest": digest, "blocks": n}))


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3, help="timed calls per metric and run (median taken)")
    ap.add_argument("--child", default=None, choices=("fse", "u16"))
    ap.add_argument("--codecs", default="fse,u16", help="comma-separated subset of fse,u16")
    a = ap.parse_args()
    if a.child:
        child(a.child, a.reps)
        return
    runs = {c: [] for c in a.codecs.split(",")}
    info_before = gpu_info()
    for _ in range(a.runs):
        for codec in runs:
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", codec, "--reps", str(a.reps)], capture_output=True, text=True)
            assert r.returncode == 0, (codec, r.stderr[-3000:])
            runs[codec].append(json.loads(r.stdout.strip().splitlines()[-1]))
    summary = {}
    for codec, rs in runs.items():
        ms = {}
        for k in rs[0]["ms"]:
            v = sorted(x["ms"][k] for x in rs)                           # per GiB: every layout moves 1 GiB uncompressed
            ms[k] = {"median": round(v[len(v) // 2], 3), "min": round(v[0], 3), "max": round(v[-1], 3)}
        ratio = {op: round(ms["a_%s_blocks" % op]["median"] / ms["a_%s_uniform" % op]["median"], 4) for op in ("enc", "dec")}
        sizes = ragged_sizes(GIB, codec == "u16")
        summary[codec] = {"ms_per_gib": ms, "a_blocks_over_uniform": ratio, "digests": sorted({json.dumps(x["digest"], sort_keys=True) for x in rs}),
                          "ragged_blocks": len(sizes), "ragged_encoder_shares": encoder_shares(sizes, codec == "u16")}
    print(json.dumps({"gpu": info_before, "gpu_after": gpu_info(), "runs": a.runs, "codecs": summary}))


if __name__ == "__main__":
    main()
