import sys, os
sys.path.insert(0, "/root/repo")
import torch
import finitestateentropy_b200 as fb
L = fb.lib()
n = 4 << 20
src = torch.empty(n, dtype=torch.uint8, device="cuda")
L.FSEB200_probagen(src.data_ptr(), n, 0, 0.14, torch.cuda.current_stream().cuda_stream)
ts=[]
cb, cs = fb.huf_compress_batch(src, 32768, fb.compress_bound(32768), 255, 12)
ref = (cb.clone(), cs.clone())
for i in range(int(sys.argv[1]) if len(sys.argv)>1 else 3):
    e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
    e0.record(); cb, cs = fb.huf_compress_batch(src, 32768, fb.compress_bound(32768), 255, 12); e1.record(); torch.cuda.synchronize()
    ts.append(round(e0.elapsed_time(e1),3))
    assert torch.equal(cs, ref[1])
print(ts, int(cs.sum()))
