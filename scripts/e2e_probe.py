"""Developer probe: PCIe copy rates and the two host-API phases timed separately (wall clock, host buffers pinned)."""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import finitestateentropy_b200 as fb
L = fb.lib()
n = 1 << 30; BLOCK = 32768; SLOT = fb.compress_bound(BLOCK); nb = n // BLOCK
src = torch.empty(n, dtype=torch.uint8, device="cuda")
L.FSEB200_probagen(src.data_ptr(), n, 0, 0.14, torch.cuda.current_stream().cuda_stream); torch.cuda.synchronize()
h_src = torch.empty(n, dtype=torch.uint8, pin_memory=True); h_src.copy_(src)
h_c = torch.empty(nb * SLOT + 64, dtype=torch.uint8, pin_memory=True)
h_cs = torch.empty(nb, dtype=torch.int64, pin_memory=True); h_out = torch.empty(n, dtype=torch.uint8, pin_memory=True); h_res = torch.empty(nb, dtype=torch.int64, pin_memory=True)
def t(f, reps=3):
    best = 1e9
    for _ in range(reps):
        torch.cuda.synchronize(); a = time.perf_counter(); f(); torch.cuda.synchronize(); best = min(best, time.perf_counter() - a)
    return best * 1e3
d = torch.empty(n, dtype=torch.uint8, device="cuda")
print("H2D 1 GiB   %.2f ms" % t(lambda: d.copy_(h_src, non_blocking=True)))
print("D2H 1 GiB   %.2f ms" % t(lambda: h_out.copy_(d, non_blocking=True)))
s2 = torch.cuda.Stream()
def both():
    d.copy_(h_src, non_blocking=True)
    with torch.cuda.stream(s2): h_out.copy_(src, non_blocking=True)
print("H2D+D2H concurrently 1 GiB each  %.2f ms" % t(both))
print("compress_host   %.2f ms" % t(lambda: L.FSEB200_compress_host(1, h_c.data_ptr(), SLOT, h_cs.data_ptr(), h_src.data_ptr(), n, BLOCK, 255, 12)))
print("decompress_host %.2f ms" % t(lambda: L.FSEB200_decompress_host(1, h_out.data_ptr(), n, BLOCK, h_c.data_ptr(), SLOT, h_cs.data_ptr(), h_res.data_ptr(), h_src.data_ptr())))
print("ok", bool(torch.equal(h_out, h_src)), "csum", int(h_cs.sum()))
