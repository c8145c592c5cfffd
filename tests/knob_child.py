"""One parity sweep under whatever FSEB200_* tuning knobs the environment sets (the library reads them once per process, so
tests/test_gpu_knobs.py runs this script in a child process per setting).  Exits 0 when everything matched the compiled
reference, non-zero (with the assertion) otherwise.

Sweep: Huff0, FSE and U16 batches of mixed fixtures at two block sizes and three placements through gpu_common.placed_check,
and the host-buffer tier (FSEB200_compress_host / decompress_host) for the three codecs with raw / RLE blocks and a ragged
last block."""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from helpers import ptr, probagen, gen_u16, zoo, is_error  # noqa: E402
from gpu_common import arena, placed_check, cpu_compress, cpu_decompress, checker, CANARY  # noqa: E402
import layout_fixtures as F  # noqa: E402
import paths as P  # noqa: E402
import finitestateentropy_b200 as fb  # noqa: E402


def _env_int(name):
    v = os.environ.get(name)
    return int(v) if v is not None else None


def batch_sweep():
    optin = getattr(torch.cuda.get_device_properties(0), "shared_memory_per_block_optin", 232448)
    rows = P.row_budgets(_env_int("FSEB200_HUFD_ROWS"), _env_int("FSEB200_HUFD_ROWS_B"), optin)
    for codec in ("huf", "fse", "u16"):
        for kind in ("aligned", "ragged"):
            blk = F.block_size(codec, kind)
            data = F.layout_data(codec, blk)
            slot = F.slot_for(codec, data, blk, "odd" if kind == "ragged" else "bound")
            want = cpu_compress(codec, data, block=blk, slot=slot, **F.MSV_TL[codec])[:2]
            if codec == "huf" and kind == "aligned":
                kinds, _ = P.summarize(P.huf_decode_paths(want[0], want[1], len(data), blk, slot, 0, rows))
                print("rows", rows, "block kinds", dict(kinds))
                assert kinds["A"] > 0
                if rows[1] > rows[0]:
                    assert kinds["B"] > 0
                if max(rows) < 813:
                    assert kinds["hard"] > 0
            for offs in ((0, 0, 0), (1, 8, 64), (4, 97, 1)):
                if codec == "u16":
                    offs = tuple(o + (o & 1) for o in offs)
                views = []
                for k, o in zip((len(data), len(want[1]) * slot, len(data)), offs):
                    views.append((arena(k + 128), CANARY + o))
                placed_check(codec, data, blk, slot, want, *views, **F.MSV_TL[codec])
            torch.cuda.empty_cache()


def host_tier():
    """FSEB200_compress_host / decompress_host against the reference: at FSEB200_HOST_CHUNK_BLOCKS=64 the 400 blocks below are
    seven chunks, more than the pipeline's four streams"""
    L = fb.lib()
    rng = np.random.default_rng(44)
    block = 4096
    for codec, cid in (("huf", 1), ("fse", 0), ("u16", 2)):
        parts = []
        for b in range(400):
            r = b % 10
            if codec == "u16":
                parts.append(gen_u16(block // 2, 240, 0.5, 1 + b).view(np.uint8) if r < 8 else np.full(block // 2, b, np.uint16).view(np.uint8))
            elif r < 6:
                parts.append(probagen(block + b, 0.14 if codec == "huf" else 0.8)[b:])
            elif r < 8:
                parts.append(rng.integers(0, 256, block, dtype=np.uint8))        # not compressible: stored raw (cSize 0)
            elif r < 9:
                parts.append(np.full(block, b & 0xFF, np.uint8))                 # RLE (cSize 1)
            else:
                parts.append(zoo(rng, block))
        parts.append(probagen(1234, 0.2) if codec != "u16" else gen_u16(617, 240, 0.5, 3).view(np.uint8))   # ragged last block
        data = np.concatenate(parts)
        n = len(data)
        nb = (n + block - 1) // block
        slot = F.bound(block) + (2 if codec == "u16" else 1)
        wc, wcs, _ = cpu_compress(codec, data, block=block, slot=slot, **F.MSV_TL[codec])
        want_out, want_res = cpu_decompress(codec, wc, wcs.copy(), data, block=block, slot=slot)
        assert (wcs == 0).sum() + (wcs == 1).sum() > 20 or codec == "u16"
        hc = np.full(nb * slot + CANARY, 0x5A, np.uint8)
        hcs = np.zeros(nb, np.uint64)
        m = F.MSV_TL[codec]
        assert L.FSEB200_compress_host(cid, ptr(hc), slot, ptr(hcs), ptr(data), n, block, m["msv"], m["tl"]) == 0
        assert np.array_equal(hcs, wcs), [(b, int(hcs[b]), int(wcs[b])) for b in range(nb) if hcs[b] != wcs[b]][:5]
        for b in range(nb):
            k = int(wcs[b])
            if is_error(k) or (k <= 1 and codec != "huf") or k == 0:
                continue
            assert np.array_equal(hc[b * slot: b * slot + k], wc[b * slot: b * slot + k]), (codec, b)
        assert (hc[nb * slot:] == 0x5A).all()
        out = np.concatenate([~want_out, np.full(CANARY, 0x5A, np.uint8)])
        res = np.zeros(nb, np.uint64)
        assert L.FSEB200_decompress_host(cid, ptr(out), n, block, ptr(wc), slot, ptr(wcs), ptr(res), ptr(data)) == 0
        keep = np.array([not is_error(int(c)) for c in wcs])
        assert np.array_equal(res[keep], want_res[keep]), [(b, int(res[b]), int(want_res[b])) for b in range(nb) if keep[b] and res[b] != want_res[b]][:5]
        for b in range(nb):
            if keep[b] and not is_error(int(want_res[b])):
                assert np.array_equal(out[b * block: min(n, (b + 1) * block)], want_out[b * block: min(n, (b + 1) * block)]), (codec, b)
        assert (out[n:] == 0x5A).all()


if __name__ == "__main__":
    assert checker()[1], "needs the compiled reference"
    batch_sweep()
    host_tier()
    print("knob sweep ok:", {k: v for k, v in os.environ.items() if k.startswith("FSEB200_")})
