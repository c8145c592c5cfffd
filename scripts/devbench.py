"""Developer micro-benchmark (not the judged bench.py): times one batched kernel on HBM-resident data.
usage: python scripts/devbench.py {huf_enc|huf_dec|fse_enc|fse_dec|u16_enc|u16_dec} [MiB] [p] [iters]"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import finitestateentropy_b200 as fb

what = sys.argv[1] if len(sys.argv) > 1 else "huf_dec"
mib = int(sys.argv[2]) if len(sys.argv) > 2 else 256
p = float(sys.argv[3]) if len(sys.argv) > 3 else 0.14
iters = int(sys.argv[4]) if len(sys.argv) > 4 else 10
n = mib << 20
L = fb.lib()
BLOCK = 32768
codec, op = what.split("_")
src = torch.empty(n, dtype=torch.uint8, device="cuda")
st = torch.cuda.current_stream().cuda_stream
if codec == "u16":
    assert L.FSEB200_genU16(src.data_ptr(), n // 2, 0, 240, p, 1, st) == 0
    SLOT = 32768; enc = lambda **k: fb.fseu16_compress_batch(src, BLOCK, SLOT, 0, 12, **k); dec = fb.fseu16_decompress_batch
else:
    assert L.FSEB200_probagen(src.data_ptr(), n, 0, p, st) == 0
    SLOT = fb.compress_bound(BLOCK)
    e = fb.huf_compress_batch if codec == "huf" else fb.fse_compress_batch
    enc = lambda **k: e(src, BLOCK, SLOT, 255, 12, **k); dec = fb.huf_decompress_batch if codec == "huf" else fb.fse_decompress_batch
cbuf, cs = enc()
out, res = dec(cbuf, cs, n, BLOCK, SLOT, orig=src)
torch.cuda.synchronize()
ok = bool(torch.equal(out, src))
csum = int(cs.sum())
run = (lambda: enc(cbuf=cbuf, csizes=cs)) if op == "enc" else (lambda: dec(cbuf, cs, n, BLOCK, SLOT, out=out, results=res, orig=src))
for _ in range(3): run()
torch.cuda.synchronize()
ts = []
for _ in range(iters):
    e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
    e0.record(); run(); e1.record(); torch.cuda.synchronize(); ts.append(e0.elapsed_time(e1))
best = min(ts); med = sorted(ts)[len(ts) // 2]; alg = n + csum
print("%s %d MiB p=%.2f roundtrip_ok=%s ratio %.4f best %.3f ms med %.3f ms -> %.1f GB/s uncompressed, %.1f GB/s algorithmic (%.1f%% of 6566)" %
      (what, mib, p, ok, csum / n, best, med, n / best / 1e6, alg / best / 1e6, alg / best / 1e6 / 65.66))
