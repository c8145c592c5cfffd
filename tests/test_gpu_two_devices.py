"""One process, every GPU it sees (-m gpu): per-device launcher state (ADVICE round 1: the opt-in shared-memory attribute, SM
count, tier-2 workspace and host pipeline used to be process-wide singletons bound to the first device).  With two or more GPUs
device 1 runs first, so nothing may be bound to device 0; with one GPU the same sequence re-uses that device's cached state.
The middle pass runs on a side stream, so state kept per (device, stream) is exercised on any number of GPUs."""

import numpy as np
import pytest
import torch

from helpers import probagen, ptr
from gpu_common import cpu_compress, BLOCK, SLOT
import finitestateentropy_b200 as fb

pytestmark = pytest.mark.gpu


def test_both_devices_from_one_process():
    n = torch.cuda.device_count()
    assert n >= 1
    L = fb.lib()
    data = probagen(64 * BLOCK + 777, 0.14)
    for codec, enc, dec, one in (("huf", fb.huf_compress_batch, fb.huf_decompress_batch, L.HUF_compress2),
                                 ("fse", fb.fse_compress_batch, fb.fse_decompress_batch, L.FSE_compress2)):
        want_c, want_cs, _ = cpu_compress(codec, data, slot=SLOT)
        other = min(n - 1, 1)                                       # device 1, or device 0 on a one-GPU box
        for k, d in enumerate((other, 0, other)):                   # the second device first: nothing may be bound to device 0
            side = torch.cuda.Stream(d) if k == 1 else torch.cuda.default_stream(d)
            with torch.cuda.device(d), torch.cuda.stream(side):
                src = torch.from_numpy(data).cuda(d)
                cbuf, cs = enc(src, BLOCK, SLOT, 255, 12)
                out, res = dec(cbuf, cs, len(data), BLOCK, SLOT, orig=src)
                torch.cuda.synchronize(d)
                assert np.array_equal(cs.cpu().numpy().view(np.uint64), want_cs), (codec, d)
                assert torch.equal(out, src), (codec, d)
                blk = np.ascontiguousarray(data[:BLOCK]); o = np.zeros(SLOT, np.uint8)
                r = one(ptr(o), SLOT, ptr(blk), BLOCK, 255, 12)      # tier 2 (host pointers) on the current device
                assert r == want_cs[0] and np.array_equal(o[:r], want_c[:r]), (codec, d)
