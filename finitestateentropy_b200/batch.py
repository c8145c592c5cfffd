"""Batched, device-resident entry points on torch CUDA tensors (thin wrappers over FSEB200_*_batch).

Geometry is the one programs/bench.c:530-548 builds: a flat uncompressed buffer split into
`block_size` blocks (last one shorter), compressed block b in the fixed slot `cbuf[b*slot : (b+1)*slot]`,
`csizes[b]` = the reference's return value for that block (0 = stored raw, 1 = RLE, error codes in-band).

The `*_blocks` calls take per-block descriptors instead (FSEB200_{HUF,HUF_*1X,FSE,FSEU16}_*_blocks): int64 CUDA tensors of device
addresses and sizes, one entry per block, so blocks of any size may sit anywhere -- e.g. packed back to back.  As in the
reference's functions, the U16 calls count uncompressed sizes in 16-bit symbols (`block_pointers` gives bytes: halve them)."""
import torch


def nblocks(total, block_size):
    return (total + block_size - 1) // block_size


def _stream_ptr():
    return torch.cuda.current_stream().cuda_stream


def _check(t, dtype):
    assert t.is_cuda and t.is_contiguous() and t.dtype == dtype, (t.device, t.dtype, t.is_contiguous())


def _ret(code, what):
    from . import is_error, error_code, ERROR_NAMES
    if is_error(code):
        raise RuntimeError("%s failed: %s" % (what, ERROR_NAMES.get(error_code(code), code)))


def _compress(fn_name, src, block_size, slot, msv, tlog, cbuf=None, csizes=None):
    from . import lib
    _check(src, torch.uint8)
    nb = nblocks(src.numel(), block_size)
    if cbuf is None:
        cbuf = torch.empty(nb * slot + 64, dtype=torch.uint8, device=src.device)
    if csizes is None:
        csizes = torch.empty(nb, dtype=torch.int64, device=src.device)
    _check(cbuf, torch.uint8); _check(csizes, torch.int64)
    assert cbuf.numel() >= nb * slot and csizes.numel() >= nb
    r = getattr(lib(), fn_name)(cbuf.data_ptr(), slot, csizes.data_ptr(), src.data_ptr(), src.numel(), block_size,
                                msv, tlog, _stream_ptr())
    _ret(r, fn_name)
    return cbuf, csizes


def _decompress(fn_name, cbuf, csizes, total, block_size, slot, out=None, results=None, orig=None):
    from . import lib
    _check(cbuf, torch.uint8); _check(csizes, torch.int64)
    nb = nblocks(total, block_size)
    if out is None:
        out = torch.empty(total, dtype=torch.uint8, device=cbuf.device)
    if results is None:
        results = torch.empty(nb, dtype=torch.int64, device=cbuf.device)
    _check(out, torch.uint8); _check(results, torch.int64)
    assert out.numel() >= total and results.numel() >= nb and csizes.numel() >= nb
    r = getattr(lib(), fn_name)(out.data_ptr(), total, block_size, cbuf.data_ptr(), slot, csizes.data_ptr(),
                                results.data_ptr(), orig.data_ptr() if orig is not None else None, _stream_ptr())
    _ret(r, fn_name)
    return out, results


def huf_compress_batch(src, block_size=32768, slot=None, max_symbol_value=255, table_log=12, cbuf=None, csizes=None):
    from . import compress_bound
    return _compress("FSEB200_HUF_compress_batch", src, block_size, slot or compress_bound(block_size),
                     max_symbol_value, table_log, cbuf, csizes)


def huf_decompress_batch(cbuf, csizes, total, block_size=32768, slot=None, out=None, results=None, orig=None):
    from . import compress_bound
    return _decompress("FSEB200_HUF_decompress_batch", cbuf, csizes, total, block_size,
                       slot or compress_bound(block_size), out, results, orig)


def fse_compress_batch(src, block_size=32768, slot=None, max_symbol_value=255, table_log=12, cbuf=None, csizes=None):
    from . import compress_bound
    return _compress("FSEB200_FSE_compress_batch", src, block_size, slot or compress_bound(block_size),
                     max_symbol_value, table_log, cbuf, csizes)


def fse_decompress_batch(cbuf, csizes, total, block_size=32768, slot=None, out=None, results=None, orig=None):
    from . import compress_bound
    return _decompress("FSEB200_FSE_decompress_batch", cbuf, csizes, total, block_size,
                       slot or compress_bound(block_size), out, results, orig)


def fseu16_compress_batch(src, block_size=32768, slot=32768, max_symbol_value=0, table_log=12, cbuf=None, csizes=None):
    """src: uint8 view of little-endian uint16 symbols; block_size in BYTES (programs/bench.c:221 halves it)"""
    return _compress("FSEB200_FSEU16_compress_batch", src, block_size, slot, max_symbol_value, table_log, cbuf, csizes)


def fseu16_decompress_batch(cbuf, csizes, total, block_size=32768, slot=32768, out=None, results=None, orig=None):
    return _decompress("FSEB200_FSEU16_decompress_batch", cbuf, csizes, total, block_size, slot, out, results, orig)


def block_pointers(views):
    """(ptrs, sizes): int64 tensors of the device addresses and lengths of a list of 1-D uint8 CUDA views, on their device"""
    dev = views[0].device if views else torch.device("cuda")
    for v in views:
        assert v.is_cuda and v.dtype == torch.uint8 and v.dim() == 1 and v.is_contiguous() and v.device == dev, (v.device, v.dtype)
    ptrs = torch.tensor([v.data_ptr() for v in views], dtype=torch.int64).to(dev)
    sizes = torch.tensor([v.numel() for v in views], dtype=torch.int64).to(dev)
    return ptrs, sizes


def _blocks_args(*arrays):
    n = arrays[0].numel()
    for a in arrays:
        _check(a, torch.int64)
        assert a.numel() == n and a.device == arrays[0].device, (a.numel(), n, a.device)
    return n


def huf_compress_blocks(src_ptrs, src_sizes, dst_ptrs, dst_caps, csizes=None, max_symbol_value=255, table_log=12):
    """HUF_compress2 on every block b: src_ptrs[b] / src_sizes[b] into dst_ptrs[b] of capacity dst_caps[b], on the current
    stream.  Returns csizes (int64; the reference's value per block, error codes as their two's-complement)."""
    return _codec_blocks("FSEB200_HUF_compress_blocks", src_ptrs, (src_ptrs, src_sizes, dst_ptrs, dst_caps), csizes,
                         (max_symbol_value, table_log))


def huf_decompress_blocks(csrc_ptrs, csrc_sizes, dst_ptrs, dst_sizes, results=None):
    """HUF_decompress on every block b: csrc_ptrs[b] / csrc_sizes[b] into dst_ptrs[b] of dst_sizes[b] bytes, on the current
    stream.  Returns results (int64; regenerated size or error code per block)."""
    return _codec_blocks("FSEB200_HUF_decompress_blocks", csrc_ptrs, (csrc_ptrs, csrc_sizes, dst_ptrs, dst_sizes), results)


def huf_compress1x_blocks(src_ptrs, src_sizes, dst_ptrs, dst_caps, csizes=None, max_symbol_value=255, table_log=12):
    """HUF_compress1X (single-stream format) on every block b: src_ptrs[b] / src_sizes[b] into dst_ptrs[b] of capacity
    dst_caps[b], on the current stream.  Returns csizes (int64; the reference's value per block, error codes as their
    two's-complement)."""
    return _codec_blocks("FSEB200_HUF_compress1X_blocks", src_ptrs, (src_ptrs, src_sizes, dst_ptrs, dst_caps), csizes,
                         (max_symbol_value, table_log))


def huf_decompress1x_blocks(csrc_ptrs, csrc_sizes, dst_ptrs, dst_sizes, results=None):
    """HUF_decompress1X_DCtx (single-stream format) on every block b: csrc_ptrs[b] / csrc_sizes[b] into dst_ptrs[b] of
    dst_sizes[b] bytes, on the current stream.  Returns results (int64; regenerated size or error code per block)."""
    return _codec_blocks("FSEB200_HUF_decompress1X_blocks", csrc_ptrs, (csrc_ptrs, csrc_sizes, dst_ptrs, dst_sizes), results)


def huf_compress_repeat_blocks(src_ptrs, src_sizes, dst_ptrs, dst_caps, ctables, repeats, prefer, csizes=None,
                               max_symbol_value=255, table_log=12):
    """HUF_compress4X_repeat on every block b: src_ptrs[b] / src_sizes[b] into dst_ptrs[b] of capacity dst_caps[b], with the
    table at ctables[b] (int64 device address of 256 uint32 cells), the flag repeats[b] (int32 HUF_repeat: none 0, check 1,
    valid 2) and prefer[b] (int32 preferRepeat), on the current stream.  Updates the tables and flags where the reference does.
    Returns csizes (int64).  A block of 2 or more bytes with repeats[b] != 0 afterwards carries no tree header."""
    return _repeat_blocks("FSEB200_HUF_compress4X_repeat_blocks", src_ptrs, src_sizes, dst_ptrs, dst_caps, ctables, repeats,
                          prefer, csizes, max_symbol_value, table_log)


def huf_compress1x_repeat_blocks(src_ptrs, src_sizes, dst_ptrs, dst_caps, ctables, repeats, prefer, csizes=None,
                                 max_symbol_value=255, table_log=12):
    """huf_compress_repeat_blocks in the single-stream format (HUF_compress1X_repeat per block)"""
    return _repeat_blocks("FSEB200_HUF_compress1X_repeat_blocks", src_ptrs, src_sizes, dst_ptrs, dst_caps, ctables, repeats,
                          prefer, csizes, max_symbol_value, table_log)


def _repeat_blocks(fn_name, src_ptrs, src_sizes, dst_ptrs, dst_caps, ctables, repeats, prefer, csizes, msv, tlog):
    from . import lib
    if csizes is None:
        csizes = torch.empty(src_ptrs.numel(), dtype=torch.int64, device=src_ptrs.device)
    n = _blocks_args(src_ptrs, src_sizes, dst_ptrs, dst_caps, csizes, ctables)
    _arrays(n, src_ptrs.device, (repeats, torch.int32), (prefer, torch.int32))
    r = getattr(lib(), fn_name)(n, dst_ptrs.data_ptr(), dst_caps.data_ptr(), csizes.data_ptr(), src_ptrs.data_ptr(),
                                src_sizes.data_ptr(), ctables.data_ptr(), repeats.data_ptr(), prefer.data_ptr(), msv, tlog,
                                _stream_ptr())
    _ret(r, fn_name)
    return csizes


def huf_compress_repeat_chains(chain_starts, src_ptrs, src_sizes, dst_ptrs, dst_caps, prefer, ctables, repeats, chain_hdr_ptrs,
                               chain_hdr_sizes, csizes=None, hdr_ptrs=None, hdr_sizes=None, max_symbol_value=255, table_log=12):
    """HUF_compress4X_repeat block after block along each chain, on the current stream: chain c is blocks
    [chain_starts[c], chain_starts[c + 1]) (int64, n_chains + 1 entries), coded into dst_ptrs[b] of capacity dst_caps[b] with
    prefer[b] (int32); the stream's state is ctables[c] (int64 device address of 256 uint32 cells), repeats[c] (int32 HUF_repeat)
    and its header chain_hdr_ptrs[c] / chain_hdr_sizes[c] (int64), read at the start and updated at the end of the chain.
    Returns (csizes, hdr_ptrs, hdr_sizes) (int64): block b's value and the header it was coded with (0 / 0: its own, or none),
    as FSEB200_HUF_decompress4X_repeat_blocks takes them."""
    return _repeat_chains("FSEB200_HUF_compress4X_repeat_chains", chain_starts, src_ptrs, src_sizes, dst_ptrs, dst_caps, prefer, None,
                          ctables, repeats, chain_hdr_ptrs, chain_hdr_sizes, csizes, hdr_ptrs, hdr_sizes, max_symbol_value, table_log)


def huf_compress1x_repeat_chains(chain_starts, src_ptrs, src_sizes, dst_ptrs, dst_caps, prefer, ctables, repeats, chain_hdr_ptrs,
                                 chain_hdr_sizes, csizes=None, hdr_ptrs=None, hdr_sizes=None, max_symbol_value=255, table_log=12):
    """huf_compress_repeat_chains in the single-stream format (HUF_compress1X_repeat per block)"""
    return _repeat_chains("FSEB200_HUF_compress1X_repeat_chains", chain_starts, src_ptrs, src_sizes, dst_ptrs, dst_caps, prefer, None,
                          ctables, repeats, chain_hdr_ptrs, chain_hdr_sizes, csizes, hdr_ptrs, hdr_sizes, max_symbol_value, table_log)


def _arrays(n, dev, *arrays):
    """the device addresses of (tensor, dtype) pairs, each checked to be a contiguous CUDA tensor of that dtype with n entries on
    `dev`; a None tensor (the form flags of a call that has none) is left out"""
    ptrs = []
    for a, dtype in arrays:
        if a is not None:
            _check(a, dtype)
            assert a.numel() == n and a.device == dev, (a.numel(), n, a.device)
            ptrs.append(a.data_ptr())
    return ptrs


def _chain_args(chain_starts, dev, *per_chain):
    """(n_chains, addresses of the per-chain arrays) after checking chain_starts (int64, n_chains + 1) and each array"""
    _check(chain_starts, torch.int64)
    n_chains = chain_starts.numel() - 1
    assert n_chains >= 0 and chain_starts.device == dev, (chain_starts.numel(), chain_starts.device)
    return n_chains, _arrays(n_chains, dev, *per_chain)


def _state_args(chain_starts, dev, ctables, repeats, chain_hdr_ptrs, chain_hdr_sizes):
    return _chain_args(chain_starts, dev, (ctables, torch.int64), (repeats, torch.int32), (chain_hdr_ptrs, torch.int64),
                       (chain_hdr_sizes, torch.int64))


def _repeat_chains(fn_name, chain_starts, src_ptrs, src_sizes, dst_ptrs, dst_caps, prefer, single, ctables, repeats, chain_hdr_ptrs,
                   chain_hdr_sizes, csizes, hdr_ptrs, hdr_sizes, msv, tlog):
    """the pointer-form chain compress; `single` the per-block forms of the mixed call, None for the 4X and 1X calls"""
    from . import lib
    n = src_ptrs.numel()
    dev = src_ptrs.device
    if csizes is None:
        csizes = torch.empty(n, dtype=torch.int64, device=dev)
    if hdr_ptrs is None:
        hdr_ptrs = torch.empty(n, dtype=torch.int64, device=dev)
    if hdr_sizes is None:
        hdr_sizes = torch.empty(n, dtype=torch.int64, device=dev)
    _blocks_args(src_ptrs, src_sizes, dst_ptrs, dst_caps, csizes, hdr_ptrs, hdr_sizes)
    per_block = _arrays(n, dev, (prefer, torch.int32), (single, torch.uint8))
    n_chains, state = _state_args(chain_starts, dev, ctables, repeats, chain_hdr_ptrs, chain_hdr_sizes)
    r = getattr(lib(), fn_name)(n_chains, chain_starts.data_ptr(), n, dst_ptrs.data_ptr(), dst_caps.data_ptr(), csizes.data_ptr(),
                                src_ptrs.data_ptr(), src_sizes.data_ptr(), *per_block, *state, hdr_ptrs.data_ptr(),
                                hdr_sizes.data_ptr(), msv, tlog, _stream_ptr())
    _ret(r, fn_name)
    return csizes, hdr_ptrs, hdr_sizes


def huf_compress_repeat_chains_packed(chain_starts, src_ptrs, src_sizes, prefer, ctables, repeats, chain_hdr_ptrs, chain_hdr_sizes,
                                      out=None, offsets=None, csizes=None, kinds=None, max_symbol_value=255, table_log=12):
    """huf_compress_repeat_chains at capacities HUF_compressBound with every block stored back to back in `out` (capacity
    out.numel()), on the current stream.  The chain and state arguments are huf_compress_repeat_chains's; a chain header that
    comes back points into `out`.  Returns (out, offsets, csizes, kinds): offsets (int64, n + 1 entries) the prefix sum of the
    stored lengths, csizes the loop's value per block (dstSize_tooSmall for a block that does not fit `out`), kinds (uint8) 0 raw,
    1 RLE, 2 own tree header, 3 the previous table's header, 4 nothing stored.  With out=None, `out` is allocated at
    sum(src_sizes) + 32 bytes, always enough: reading that sum costs one host synchronisation."""
    return _repeat_chains_packed("FSEB200_HUF_compress4X_repeat_chains_packed", chain_starts, src_ptrs, src_sizes, prefer, None, ctables,
                                 repeats, chain_hdr_ptrs, chain_hdr_sizes, out, offsets, csizes, kinds, (max_symbol_value, table_log))


def huf_compress1x_repeat_chains_packed(chain_starts, src_ptrs, src_sizes, prefer, ctables, repeats, chain_hdr_ptrs, chain_hdr_sizes,
                                        out=None, offsets=None, csizes=None, kinds=None, max_symbol_value=255, table_log=12):
    """huf_compress_repeat_chains_packed in the single-stream format (HUF_compress1X_repeat per block)"""
    return _repeat_chains_packed("FSEB200_HUF_compress1X_repeat_chains_packed", chain_starts, src_ptrs, src_sizes, prefer, None, ctables,
                                 repeats, chain_hdr_ptrs, chain_hdr_sizes, out, offsets, csizes, kinds, (max_symbol_value, table_log))


def _repeat_chains_packed(fn_name, chain_starts, src_ptrs, src_sizes, prefer, single, ctables, repeats, chain_hdr_ptrs, chain_hdr_sizes,
                          out, offsets, csizes, kinds, scalars, forms_out=False):
    """the packed chain compress; `single` the per-block forms (None for the 4X and 1X calls), which with forms_out the call
    writes, allocated here when None and returned last; `scalars` the C call's arguments between the chain headers and the stream"""
    from . import lib
    n = _blocks_args(src_ptrs, src_sizes)
    dev = src_ptrs.device
    if forms_out and single is None:
        single = torch.empty(n, dtype=torch.uint8, device=dev)
    per_block = _arrays(n, dev, (prefer, torch.int32), (single, torch.uint8))
    n_chains, state = _state_args(chain_starts, dev, ctables, repeats, chain_hdr_ptrs, chain_hdr_sizes)
    if out is None:
        out = torch.empty(int(src_sizes.sum().item()) + 32, dtype=torch.uint8, device=dev)    # .item(): the host sync
    if offsets is None:
        offsets = torch.empty(n + 1, dtype=torch.int64, device=dev)
    if csizes is None:
        csizes = torch.empty(n, dtype=torch.int64, device=dev)
    if kinds is None:
        kinds = torch.empty(n, dtype=torch.uint8, device=dev)
    _check(out, torch.uint8); _check(offsets, torch.int64); _check(csizes, torch.int64); _check(kinds, torch.uint8)
    assert offsets.numel() == n + 1 and csizes.numel() == n and kinds.numel() == n and out.device == dev, (offsets.numel(), n)
    r = getattr(lib(), fn_name)(n_chains, chain_starts.data_ptr(), n, out.data_ptr(), out.numel(), offsets.data_ptr(),
                                csizes.data_ptr(), kinds.data_ptr(), src_ptrs.data_ptr(), src_sizes.data_ptr(), *per_block, *state,
                                *scalars, _stream_ptr())
    _ret(r, fn_name)
    return (out, offsets, csizes, kinds) + ((single,) if forms_out else ())


def huf_decompress_repeat_packed(chain_starts, packed, offsets, kinds, chain_hdr_ptrs, chain_hdr_sizes, dst_ptrs, dst_sizes,
                                 results=None):
    """every block of a packed chain buffer (huf_compress_repeat_chains_packed's out, offsets and kinds) into dst_ptrs[b],
    regenerating dst_sizes[b] bytes, on the current stream: a kind-3 block takes the header of the last kind-2 block before it
    in its chain, or chain_hdr_ptrs[c] / chain_hdr_sizes[c] (int64, the headers the chains entered the compress call with).
    Returns results (int64; the regenerated size or an error code per block)."""
    return _repeat_unpack("FSEB200_HUF_decompress4X_repeat_packed", chain_starts, packed, offsets, kinds, None, chain_hdr_ptrs,
                          chain_hdr_sizes, dst_ptrs, dst_sizes, results)


def huf_decompress1x_repeat_packed(chain_starts, packed, offsets, kinds, chain_hdr_ptrs, chain_hdr_sizes, dst_ptrs, dst_sizes,
                                   results=None):
    """huf_decompress_repeat_packed in the single-stream format (huf_compress1x_repeat_chains_packed's buffers)"""
    return _repeat_unpack("FSEB200_HUF_decompress1X_repeat_packed", chain_starts, packed, offsets, kinds, None, chain_hdr_ptrs,
                          chain_hdr_sizes, dst_ptrs, dst_sizes, results)


def _repeat_unpack(fn_name, chain_starts, packed, offsets, kinds, single, chain_hdr_ptrs, chain_hdr_sizes, dst_ptrs, dst_sizes,
                   results):
    """the packed chain decompress; `single` the per-block forms of the mixed call, None for the 4X and 1X calls"""
    from . import lib
    n = _blocks_args(dst_ptrs, dst_sizes)
    dev = dst_ptrs.device
    n_chains, headers = _chain_args(chain_starts, dev, (chain_hdr_ptrs, torch.int64), (chain_hdr_sizes, torch.int64))
    forms = _arrays(n, dev, (single, torch.uint8))
    if results is None:
        results = torch.empty(n, dtype=torch.int64, device=dev)
    _check(packed, torch.uint8); _check(offsets, torch.int64); _check(kinds, torch.uint8); _check(results, torch.int64)
    assert offsets.numel() == n + 1 and kinds.numel() == n and results.numel() == n and packed.device == dev, (offsets.numel(), n)
    r = getattr(lib(), fn_name)(n_chains, chain_starts.data_ptr(), n, dst_ptrs.data_ptr(), dst_sizes.data_ptr(), results.data_ptr(),
                                packed.data_ptr(), offsets.data_ptr(), kinds.data_ptr(), *forms, *headers, _stream_ptr())
    _ret(r, fn_name)
    return results


def huf_decompress_repeat_blocks(csrc_ptrs, csrc_sizes, dst_ptrs, dst_sizes, hdr_ptrs, hdr_sizes, results=None):
    """Every block b of csrc_ptrs[b] / csrc_sizes[b] into dst_ptrs[b] of dst_sizes[b] bytes, on the current stream: with
    hdr_sizes[b] == 0, HUF_decompress4X1_DCtx (the block's own tree header); otherwise HUF_readDTableX1 on hdr_ptrs[b] /
    hdr_sizes[b] and HUF_decompress4X1_usingDTable on the block.  Returns results (int64)."""
    return _header_blocks("FSEB200_HUF_decompress4X_repeat_blocks", csrc_ptrs, csrc_sizes, dst_ptrs, dst_sizes, hdr_ptrs,
                          hdr_sizes, results)


def huf_decompress1x_repeat_blocks(csrc_ptrs, csrc_sizes, dst_ptrs, dst_sizes, hdr_ptrs, hdr_sizes, results=None):
    """huf_decompress_repeat_blocks in the single-stream format (HUF_decompress1X1_DCtx / HUF_decompress1X1_usingDTable)"""
    return _header_blocks("FSEB200_HUF_decompress1X_repeat_blocks", csrc_ptrs, csrc_sizes, dst_ptrs, dst_sizes, hdr_ptrs,
                          hdr_sizes, results)


def _header_blocks(fn_name, csrc_ptrs, csrc_sizes, dst_ptrs, dst_sizes, hdr_ptrs, hdr_sizes, results, single=None):
    """the header-taking blocks decompress; `single` the per-block forms of the mixed call, None for the 4X and 1X calls"""
    from . import lib
    if results is None:
        results = torch.empty(csrc_ptrs.numel(), dtype=torch.int64, device=csrc_ptrs.device)
    n = _blocks_args(csrc_ptrs, csrc_sizes, dst_ptrs, dst_sizes, results, hdr_ptrs, hdr_sizes)
    forms = _arrays(n, csrc_ptrs.device, (single, torch.uint8))
    r = getattr(lib(), fn_name)(n, dst_ptrs.data_ptr(), dst_sizes.data_ptr(), results.data_ptr(), csrc_ptrs.data_ptr(),
                                csrc_sizes.data_ptr(), hdr_ptrs.data_ptr(), hdr_sizes.data_ptr(), *forms, _stream_ptr())
    _ret(r, fn_name)
    return results


def huf_compress_mixed_repeat_chains(chain_starts, src_ptrs, src_sizes, dst_ptrs, dst_caps, prefer, single_stream, ctables, repeats,
                                     chain_hdr_ptrs, chain_hdr_sizes, csizes=None, hdr_ptrs=None, hdr_sizes=None, max_symbol_value=255,
                                     table_log=12):
    """huf_compress_repeat_chains with each block's form chosen by single_stream[b] (uint8): 0 HUF_compress4X_repeat, anything
    else HUF_compress1X_repeat.  Both forms share the stream's table, flag and header.  Returns (csizes, hdr_ptrs, hdr_sizes),
    as huf_decompress_mixed_repeat_blocks takes them with the same single_stream."""
    return _repeat_chains("FSEB200_HUF_compress_mixed_repeat_chains", chain_starts, src_ptrs, src_sizes, dst_ptrs, dst_caps, prefer,
                          single_stream, ctables, repeats, chain_hdr_ptrs, chain_hdr_sizes, csizes, hdr_ptrs, hdr_sizes,
                          max_symbol_value, table_log)


def huf_decompress_mixed_repeat_blocks(csrc_ptrs, csrc_sizes, dst_ptrs, dst_sizes, hdr_ptrs, hdr_sizes, single_stream, results=None):
    """huf_decompress_repeat_blocks (single_stream[b] == 0) or huf_decompress1x_repeat_blocks (otherwise) on every block b, in
    one call on the current stream.  Returns results (int64)."""
    return _header_blocks("FSEB200_HUF_decompress_mixed_repeat_blocks", csrc_ptrs, csrc_sizes, dst_ptrs, dst_sizes, hdr_ptrs,
                          hdr_sizes, results, single_stream)


def huf_compress_mixed_repeat_chains_packed(chain_starts, src_ptrs, src_sizes, prefer, single_stream, ctables, repeats, chain_hdr_ptrs,
                                            chain_hdr_sizes, out=None, offsets=None, csizes=None, kinds=None, max_symbol_value=255,
                                            table_log=12):
    """huf_compress_repeat_chains_packed with each block's form chosen by single_stream[b] (uint8, 0 = 4X).  Kinds keep their
    numbering whatever the form, so the stream is (out, offsets, kinds) plus single_stream.  Returns (out, offsets, csizes, kinds)."""
    return _repeat_chains_packed("FSEB200_HUF_compress_mixed_repeat_chains_packed", chain_starts, src_ptrs, src_sizes, prefer,
                                 single_stream, ctables, repeats, chain_hdr_ptrs, chain_hdr_sizes, out, offsets, csizes, kinds,
                                 (max_symbol_value, table_log))


def huf_compress_literals_chains_packed(chain_starts, src_ptrs, src_sizes, prefer, ctables, repeats, chain_hdr_ptrs, chain_hdr_sizes,
                                        out=None, offsets=None, csizes=None, kinds=None, single_stream=None, max_symbol_value=255,
                                        table_log=11, min_literals=64, min_gain_log=6):
    """huf_compress_mixed_repeat_chains_packed under zstd's literal-coding policy (FSEB200_HUF_compress_literals_chains_packed): the
    device chooses each block's form from the stream's flag, skips blocks below the size threshold (min_literals, or 6 bytes with
    a valid table), stores a block raw when it fails the minimum gain (n >> min_gain_log) + 2 and RLE only when its bytes are
    equal, and keeps a step's table and flag only for a block stored with its own header.  The other arguments are the mixed
    call's.  Returns (out, offsets, csizes, kinds, single_stream): single_stream (uint8) holds the forms it chose, so the stream
    decodes with huf_decompress_mixed_repeat_packed."""
    return _repeat_chains_packed("FSEB200_HUF_compress_literals_chains_packed", chain_starts, src_ptrs, src_sizes, prefer,
                                 single_stream, ctables, repeats, chain_hdr_ptrs, chain_hdr_sizes, out, offsets, csizes, kinds,
                                 (max_symbol_value, table_log, min_literals, min_gain_log), forms_out=True)


def huf_decompress_mixed_repeat_packed(chain_starts, packed, offsets, kinds, single_stream, chain_hdr_ptrs, chain_hdr_sizes, dst_ptrs,
                                       dst_sizes, results=None):
    """huf_decompress_repeat_packed over a buffer huf_compress_mixed_repeat_chains_packed wrote, each block in the form
    single_stream[b] names.  Returns results (int64)."""
    return _repeat_unpack("FSEB200_HUF_decompress_mixed_repeat_packed", chain_starts, packed, offsets, kinds, single_stream,
                          chain_hdr_ptrs, chain_hdr_sizes, dst_ptrs, dst_sizes, results)


def huf_compress_packed(src_ptrs, src_sizes, out=None, offsets=None, csizes=None, max_symbol_value=255, table_log=12):
    """HUF_compress2 on every block b (src_ptrs[b] / src_sizes[b]) at capacity HUF_compressBound, the results stored back to
    back in `out` (capacity out.numel()), on the current stream.  Returns (out, offsets, csizes): offsets (int64, n + 1 entries)
    is the prefix sum of the stored lengths, csizes the reference's value per block (dstSize_tooSmall for a block that does not
    fit `out`).  With out=None, `out` is allocated at sum(src_sizes) + 32 bytes, always enough: reading that sum costs one host
    synchronisation.  `packed_pointers(out, offsets)` gives the arrays huf_decompress_blocks decodes the buffer with."""
    return _compress_packed("FSEB200_HUF_compress_packed", 1, src_ptrs, src_sizes, out, offsets, csizes, max_symbol_value, table_log)


def huf_compress1x_packed(src_ptrs, src_sizes, out=None, offsets=None, csizes=None, max_symbol_value=255, table_log=12):
    """huf_compress_packed in the single-stream format (HUF_compress1X per block); decode with huf_decompress1x_blocks"""
    return _compress_packed("FSEB200_HUF_compress1X_packed", 1, src_ptrs, src_sizes, out, offsets, csizes, max_symbol_value, table_log)


def _compress_packed(fn_name, unit, src_ptrs, src_sizes, out, offsets, csizes, msv, tlog, fse=False, work=None):
    """the packed compress of blocks of `unit` bytes per symbol; FSE (`fse`) also takes the staging workspace `work`.  out and
    work, when None, are sized from the source bytes"""
    from . import lib
    n = _blocks_args(src_ptrs, src_sizes)
    dev = src_ptrs.device
    if out is None or (fse and work is None):
        src_bytes = unit * int(src_sizes.sum().item())                                  # .item(): the host sync
        if out is None:
            out = torch.empty(src_bytes + 32, dtype=torch.uint8, device=dev)
        if fse and work is None:
            work = torch.empty(max(fse_packed_workspace(n, src_bytes), 1), dtype=torch.uint8, device=dev)
    if offsets is None:
        offsets = torch.empty(n + 1, dtype=torch.int64, device=dev)
    if csizes is None:
        csizes = torch.empty(n, dtype=torch.int64, device=dev)
    _check(out, torch.uint8)
    if fse:
        _check(work, torch.uint8)
    _check(offsets, torch.int64); _check(csizes, torch.int64)
    assert offsets.numel() == n + 1 and csizes.numel() == n and out.device == dev and (not fse or work.device == dev), \
        (offsets.numel(), csizes.numel(), n)
    workspace = (work.data_ptr(), work.numel()) if fse else ()
    r = getattr(lib(), fn_name)(n, out.data_ptr(), out.numel(), offsets.data_ptr(), csizes.data_ptr(), src_ptrs.data_ptr(),
                                src_sizes.data_ptr(), msv, tlog, *workspace, _stream_ptr())
    _ret(r, fn_name)
    return out, offsets, csizes


def packed_pointers(out, offsets):
    """(ptrs, sizes) of the blocks of a packed buffer: int64 device addresses out + offsets[b] and stored lengths
    offsets[b + 1] - offsets[b], the compressed-source arrays of huf_decompress_blocks / huf_decompress1x_blocks"""
    _check(offsets, torch.int64)
    return offsets[:-1] + out.data_ptr(), offsets[1:] - offsets[:-1]


def _codec_blocks(fn_name, n_ptrs, arrays, out, extra=()):
    from . import lib
    if out is None:
        out = torch.empty(n_ptrs.numel(), dtype=torch.int64, device=n_ptrs.device)
    src_ptrs, src_sizes, dst_ptrs, dst_caps = arrays
    n = _blocks_args(src_ptrs, src_sizes, dst_ptrs, dst_caps, out)
    r = getattr(lib(), fn_name)(n, dst_ptrs.data_ptr(), dst_caps.data_ptr(), out.data_ptr(), src_ptrs.data_ptr(),
                                src_sizes.data_ptr(), *extra, _stream_ptr())
    _ret(r, fn_name)
    return out


def fse_compress_blocks(src_ptrs, src_sizes, dst_ptrs, dst_caps, csizes=None, max_symbol_value=255, table_log=12):
    """FSE_compress2 on every block b: src_ptrs[b] / src_sizes[b] bytes into dst_ptrs[b] of capacity dst_caps[b], on the current
    stream.  Returns csizes (int64; the reference's value per block, error codes as their two's-complement)."""
    return _codec_blocks("FSEB200_FSE_compress_blocks", src_ptrs, (src_ptrs, src_sizes, dst_ptrs, dst_caps), csizes,
                         (max_symbol_value, table_log))


def fse_decompress_blocks(csrc_ptrs, csrc_sizes, dst_ptrs, dst_caps, results=None):
    """FSE_decompress on every block b: csrc_ptrs[b] / csrc_sizes[b] into dst_ptrs[b] of capacity dst_caps[b] bytes, on the
    current stream.  Returns results (int64; regenerated size or error code per block)."""
    return _codec_blocks("FSEB200_FSE_decompress_blocks", csrc_ptrs, (csrc_ptrs, csrc_sizes, dst_ptrs, dst_caps), results)


def fseu16_compress_blocks(src_ptrs, src_symbols, dst_ptrs, dst_caps, csizes=None, max_symbol_value=0, table_log=12):
    """FSE_compressU16 on every block b: src_symbols[b] 16-bit symbols at src_ptrs[b] (2-byte aligned) into dst_ptrs[b] of
    dst_caps[b] bytes, on the current stream.  Returns csizes (int64, bytes or error codes)."""
    return _codec_blocks("FSEB200_FSEU16_compress_blocks", src_ptrs, (src_ptrs, src_symbols, dst_ptrs, dst_caps), csizes,
                         (max_symbol_value, table_log))


def fseu16_decompress_blocks(csrc_ptrs, csrc_sizes, dst_ptrs, dst_symbols, results=None):
    """FSE_decompressU16 on every block b: csrc_ptrs[b] / csrc_sizes[b] bytes into dst_ptrs[b] (2-byte aligned) of room for
    dst_symbols[b] symbols, on the current stream.  Returns results (int64; regenerated symbols or error code per block)."""
    return _codec_blocks("FSEB200_FSEU16_decompress_blocks", csrc_ptrs, (csrc_ptrs, csrc_sizes, dst_ptrs, dst_symbols), results)


def fse_compress_packed(src_ptrs, src_sizes, out=None, offsets=None, csizes=None, work=None, max_symbol_value=255, table_log=12):
    """FSE_compress2 on every block b (src_ptrs[b] / src_sizes[b] bytes) at capacity FSE_compressBound, the results stored back
    to back in `out` (capacity out.numel()), raw and RLE blocks included, on the current stream.  `work` (uint8) holds each
    block's staging slot.  Returns (out, offsets, csizes): offsets (int64, n + 1 entries) is the prefix sum of the stored lengths,
    csizes the reference's value per block (dstSize_tooSmall / workSpace_tooSmall for a block that does not fit `out` / `work`).
    With out or work None they are sized from sum(src_sizes) -- out at that sum + 32 bytes, work by fse_packed_workspace, both
    always enough: reading the sum costs one host synchronisation.  Decode with fse_decompress_packed."""
    return _compress_packed("FSEB200_FSE_compress_packed", 1, src_ptrs, src_sizes, out, offsets, csizes, max_symbol_value, table_log,
                            fse=True, work=work)


def fseu16_compress_packed(src_ptrs, src_symbols, out=None, offsets=None, csizes=None, work=None, max_symbol_value=0, table_log=12):
    """fse_compress_packed for FSE_compressU16: src_symbols[b] 16-bit symbols at src_ptrs[b] (2-byte aligned); `out` and `work`
    default to 2 * sum(src_symbols) + 32 bytes and the workspace of 2 * sum(src_symbols) source bytes"""
    return _compress_packed("FSEB200_FSEU16_compress_packed", 2, src_ptrs, src_symbols, out, offsets, csizes, max_symbol_value,
                            table_log, fse=True, work=work)


def fse_packed_workspace(n_blocks, src_bytes):
    """bytes of workspace that never run short for n_blocks blocks of src_bytes source bytes in all (U16: 2 * symbols)"""
    from . import lib
    return int(lib().FSEB200_FSE_packed_workspace(n_blocks, src_bytes))


def fse_decompress_packed(packed, offsets, dst_ptrs, dst_sizes, results=None):
    """every block of a packed FSE buffer (fse_compress_packed's out and offsets) into dst_ptrs[b], regenerating dst_sizes[b]
    bytes, on the current stream: a stored length equal to the size is a raw copy, one byte an RLE block, anything else is
    FSE_decompress'ed.  Returns results (int64; the regenerated size or an error code per block)."""
    return _decompress_packed("FSEB200_FSE_decompress_packed", packed, offsets, dst_ptrs, dst_sizes, results)


def fseu16_decompress_packed(packed, offsets, dst_ptrs, dst_symbols, results=None):
    """fse_decompress_packed for FSE-U16: dst_symbols[b] 16-bit symbols into dst_ptrs[b] (2-byte aligned); results in symbols"""
    return _decompress_packed("FSEB200_FSEU16_decompress_packed", packed, offsets, dst_ptrs, dst_symbols, results)


def huf_decompress_packed(packed, offsets, dst_ptrs, dst_sizes, results=None):
    """every block of a packed Huff0 buffer (huf_compress_packed's out and offsets) into dst_ptrs[b], regenerating dst_sizes[b]
    bytes, on the current stream: exactly huf_decompress_blocks on packed_pointers(packed, offsets), except that an empty block
    (size 0, nothing stored) gives 0.  Returns results (int64; the regenerated size or an error code per block)."""
    return _decompress_packed("FSEB200_HUF_decompress_packed", packed, offsets, dst_ptrs, dst_sizes, results)


def huf_decompress1x_packed(packed, offsets, dst_ptrs, dst_sizes, results=None):
    """huf_decompress_packed in the single-stream format (huf_compress1x_packed's buffers, huf_decompress1x_blocks per block)"""
    return _decompress_packed("FSEB200_HUF_decompress1X_packed", packed, offsets, dst_ptrs, dst_sizes, results)


def _decompress_packed(fn_name, packed, offsets, dst_ptrs, dst_sizes, results):
    from . import lib
    n = _blocks_args(dst_ptrs, dst_sizes)
    if results is None:
        results = torch.empty(n, dtype=torch.int64, device=dst_ptrs.device)
    _check(packed, torch.uint8); _check(offsets, torch.int64); _check(results, torch.int64)
    assert offsets.numel() == n + 1 and results.numel() == n and packed.device == dst_ptrs.device, (offsets.numel(), results.numel(), n)
    r = getattr(lib(), fn_name)(n, dst_ptrs.data_ptr(), dst_sizes.data_ptr(), results.data_ptr(), packed.data_ptr(),
                                offsets.data_ptr(), _stream_ptr())
    _ret(r, fn_name)
    return results


# Host-buffer packed calls (FSEB200_{compress,decompress}_host_packed): name -> (C codec number, bytes per symbol, default
# maxSymbolValue)
HOST_CODECS = {"fse": (0, 1, 255), "huf": (1, 1, 255), "fseu16": (2, 2, 0), "huf1x": (3, 1, 255)}
_NONEMPTY = None


def _host_ptr(t):
    """t's address; an empty tensor has none, and the C calls refuse NULL, so it stands in with a 1-byte buffer"""
    global _NONEMPTY
    if t.numel():
        return t.data_ptr()
    if _NONEMPTY is None:
        _NONEMPTY = torch.zeros(8, dtype=torch.uint8)
    return _NONEMPTY.data_ptr()


def _host_check(t, dtype):
    assert t.device.type == "cpu" and t.is_contiguous() and t.dtype == dtype, (t.device, t.dtype, t.is_contiguous())


def _host_sizes(sizes):
    sizes = torch.as_tensor(sizes, dtype=torch.int64)
    _host_check(sizes, torch.int64)
    return sizes


def host_compress_packed(src, sizes, codec, out=None, offsets=None, csizes=None, max_symbol_value=None, table_log=12):
    """The packed compress of `codec` ("fse", "huf", "huf1x" or "fseu16") on HOST memory: block b is sizes[b] symbols of `src`
    (a CPU uint8 tensor, pinned or pageable; U16 symbols as little-endian byte pairs) right after block b - 1.  `out` (capacity
    out.numel()), offsets (int64, n + 1 entries) and csizes (int64) are what the device packed call gives for the same blocks;
    with out=None it is allocated at unit * sum(sizes) + 32 bytes, always enough.  Synchronous.  Returns (out, offsets, csizes)."""
    from . import lib
    cid, unit, msv = HOST_CODECS[codec]
    msv = msv if max_symbol_value is None else max_symbol_value
    sizes = _host_sizes(sizes)
    n = sizes.numel()
    total = unit * int(sizes.sum())
    _host_check(src, torch.uint8)
    assert src.numel() >= total, (src.numel(), total)
    if out is None:
        out = torch.empty(total + 32, dtype=torch.uint8)
    if offsets is None:
        offsets = torch.empty(n + 1, dtype=torch.int64)
    if csizes is None:
        csizes = torch.empty(n, dtype=torch.int64)
    _host_check(out, torch.uint8); _host_check(offsets, torch.int64); _host_check(csizes, torch.int64)
    assert offsets.numel() == n + 1 and csizes.numel() == n, (offsets.numel(), csizes.numel(), n)
    r = lib().FSEB200_compress_host_packed(cid, _host_ptr(out), out.numel(), offsets.data_ptr(), _host_ptr(csizes), _host_ptr(src),
                                           _host_ptr(sizes), n, msv, table_log)
    _ret(r, "FSEB200_compress_host_packed")
    return out, offsets, csizes


def host_decompress_packed(packed, offsets, dst_sizes, codec, out=None, results=None):
    """The packed decompress of `codec` on HOST memory: every block of `packed` (a CPU uint8 tensor, host_compress_packed's out)
    located by `offsets`, regenerating dst_sizes[b] symbols; block b lands in `out` right after block b - 1, as in the source.
    With out=None it is allocated at unit * sum(dst_sizes) bytes.  results (int64) equals the device packed decompress's.
    Synchronous.  Returns (out, results)."""
    from . import lib
    cid, unit, _ = HOST_CODECS[codec]
    dst_sizes = _host_sizes(dst_sizes)
    n = dst_sizes.numel()
    total = unit * int(dst_sizes.sum())
    _host_check(packed, torch.uint8); _host_check(offsets, torch.int64)
    assert offsets.numel() == n + 1 and packed.numel() >= int(offsets[-1]), (offsets.numel(), n, packed.numel())
    if out is None:
        out = torch.empty(total, dtype=torch.uint8)
    if results is None:
        results = torch.empty(n, dtype=torch.int64)
    _host_check(out, torch.uint8); _host_check(results, torch.int64)
    assert out.numel() >= total and results.numel() == n, (out.numel(), total, results.numel(), n)
    r = lib().FSEB200_decompress_host_packed(cid, _host_ptr(out), _host_ptr(dst_sizes), _host_ptr(results), _host_ptr(packed),
                                             offsets.data_ptr(), n)
    _ret(r, "FSEB200_decompress_host_packed")
    return out, results


# Host-buffer packed chains of table reuse (FSEB200_{compress_host_repeat_chains,decompress_host_repeat}_packed): name -> C codec
HOST_CHAIN_CODECS = {"huf": 1, "huf1x": 3}


def _host_chain_args(chain_starts, per_chain):
    chain_starts = _host_sizes(chain_starts)
    n_chains = chain_starts.numel() - 1
    assert n_chains >= 0, chain_starts.numel()
    for a, dtype, shape in per_chain:
        _host_check(a, dtype)
        assert tuple(a.shape) == (n_chains,) + shape, (tuple(a.shape), n_chains)
    return chain_starts, n_chains


def host_compress_repeat_chains_packed(src, sizes, chain_starts, prefer, ctables, repeats, chain_hdr_ptrs, chain_hdr_sizes,
                                       codec="huf", out=None, max_symbol_value=255, table_log=12):
    """The packed chain compress of `codec` ("huf" or "huf1x") on HOST memory: block b is sizes[b] bytes of `src` (a CPU uint8
    tensor, pinned or pageable) right after block b - 1, chain c is blocks [chain_starts[c], chain_starts[c + 1]), and prefer (int32,
    one per block) is each block's preferRepeat.  The streams' state is in-out, in CPU tensors: ctables (uint32 or int32, n_chains x
    256 HUF_CElt cells), repeats (int32 HUF_repeat), chain_hdr_ptrs (int64 host addresses) and chain_hdr_sizes (int64); it is
    updated only when the whole stream fits `out`, and a header that comes back points into `out`.  `out` (capacity out.numel(),
    allocated at sum(sizes) + 32 bytes if None, always enough), offsets, csizes and kinds are what the device call
    huf_compress_repeat_chains_packed gives.  Synchronous.  Returns (out, offsets, csizes, kinds, (ctables, repeats,
    chain_hdr_ptrs, chain_hdr_sizes))."""
    return _host_chains_compress(HOST_CHAIN_CODECS[codec], None, src, sizes, chain_starts, prefer, ctables, repeats, chain_hdr_ptrs,
                                 chain_hdr_sizes, out, max_symbol_value, table_log)


def host_compress_mixed_repeat_chains_packed(src, sizes, chain_starts, prefer, single_stream, ctables, repeats, chain_hdr_ptrs,
                                             chain_hdr_sizes, out=None, max_symbol_value=255, table_log=12):
    """host_compress_repeat_chains_packed with each block's form chosen by single_stream[b] (a CPU uint8 tensor: 0 4X, else 1X),
    byte for byte what huf_compress_mixed_repeat_chains_packed gives.  Synchronous.  Returns (out, offsets, csizes, kinds,
    (ctables, repeats, chain_hdr_ptrs, chain_hdr_sizes))."""
    return _host_chains_compress(None, single_stream, src, sizes, chain_starts, prefer, ctables, repeats, chain_hdr_ptrs,
                                 chain_hdr_sizes, out, max_symbol_value, table_log)


def host_compress_literals_chains_packed(src, sizes, chain_starts, prefer, ctables, repeats, chain_hdr_ptrs, chain_hdr_sizes, out=None,
                                         max_symbol_value=255, table_log=11, min_literals=64, min_gain_log=6):
    """huf_compress_literals_chains_packed on HOST memory (FSEB200_compress_host_literals_chains_packed), with the arguments and
    state of host_compress_mixed_repeat_chains_packed but no forms in: byte for byte what the device call gives.  Synchronous.
    Returns (out, offsets, csizes, kinds, single_stream, (ctables, repeats, chain_hdr_ptrs, chain_hdr_sizes)); the stream decodes
    with host_decompress_mixed_repeat_packed and that single_stream."""
    single = torch.empty(_host_sizes(sizes).numel(), dtype=torch.uint8)
    out, offsets, csizes, kinds, state = _host_chains_compress(None, single, src, sizes, chain_starts, prefer, ctables, repeats,
                                                               chain_hdr_ptrs, chain_hdr_sizes, out, max_symbol_value, table_log,
                                                               (min_literals, min_gain_log))
    return out, offsets, csizes, kinds, single, state


def _host_chains_compress(cid, single, src, sizes, chain_starts, prefer, ctables, repeats, chain_hdr_ptrs, chain_hdr_sizes, out,
                          max_symbol_value, table_log, literals=None):
    """cid: the C codec of the 4X / 1X call, or None for the mixed call with the per-block forms `single`, or for the literal-policy
    call with literals = (min_literals, min_gain_log), which writes the forms into `single`"""
    from . import lib
    sizes = _host_sizes(sizes)
    n = sizes.numel()
    _host_check(src, torch.uint8)
    _host_check(prefer, torch.int32)
    assert src.numel() >= int(sizes.sum()) and prefer.numel() == n, (src.numel(), prefer.numel(), n)
    assert ctables.dtype in (torch.int32, torch.uint32), ctables.dtype
    chain_starts, n_chains = _host_chain_args(chain_starts, ((ctables, ctables.dtype, (256,)), (repeats, torch.int32, ()),
                                                             (chain_hdr_ptrs, torch.int64, ()), (chain_hdr_sizes, torch.int64, ())))
    if out is None:
        out = torch.empty(int(sizes.sum()) + 32, dtype=torch.uint8)
    _host_check(out, torch.uint8)
    offsets = torch.empty(n + 1, dtype=torch.int64)
    csizes = torch.empty(n, dtype=torch.int64)
    kinds = torch.empty(n, dtype=torch.uint8)
    table_ptrs = torch.tensor([ctables.data_ptr() + 1024 * c for c in range(n_chains)], dtype=torch.int64)
    head = (n_chains, chain_starts.data_ptr(), n, _host_ptr(out), out.numel(), offsets.data_ptr(), _host_ptr(csizes), _host_ptr(kinds),
            _host_ptr(src), _host_ptr(sizes), _host_ptr(prefer))
    state = (_host_ptr(table_ptrs), _host_ptr(repeats), _host_ptr(chain_hdr_ptrs), _host_ptr(chain_hdr_sizes), max_symbol_value,
             table_log)
    if literals is not None:
        fn_name = "FSEB200_compress_host_literals_chains_packed"
        r = getattr(lib(), fn_name)(*head, _host_ptr(single), *state, *literals)
    elif cid is None:
        _host_check(single, torch.uint8)
        assert single.numel() == n, (single.numel(), n)
        fn_name = "FSEB200_compress_host_mixed_repeat_chains_packed"
        r = getattr(lib(), fn_name)(*head, _host_ptr(single), *state)
    else:
        fn_name = "FSEB200_compress_host_repeat_chains_packed"
        r = getattr(lib(), fn_name)(cid, *head, *state)
    _ret(r, fn_name)
    return out, offsets, csizes, kinds, (ctables, repeats, chain_hdr_ptrs, chain_hdr_sizes)


def host_decompress_repeat_packed(packed, offsets, kinds, chain_starts, dst_sizes, chain_hdr_ptrs, chain_hdr_sizes, codec="huf",
                                  out=None, results=None):
    """The packed chain decompress of `codec` on HOST memory: every block of `packed` (a CPU uint8 tensor,
    host_compress_repeat_chains_packed's out) located by `offsets` and `kinds`, regenerating dst_sizes[b] bytes; block b lands in
    `out` right after block b - 1.  chain_hdr_ptrs / chain_hdr_sizes (int64 CPU tensors, host addresses) are the headers the chains
    entered the compress with.  With out=None it is allocated at sum(dst_sizes) bytes.  results (int64) equals the device call
    huf_decompress_repeat_packed's.  Synchronous.  Returns (out, results)."""
    return _host_chains_decompress(HOST_CHAIN_CODECS[codec], None, packed, offsets, kinds, chain_starts, dst_sizes, chain_hdr_ptrs,
                                   chain_hdr_sizes, out, results)


def host_decompress_mixed_repeat_packed(packed, offsets, kinds, single_stream, chain_starts, dst_sizes, chain_hdr_ptrs, chain_hdr_sizes,
                                        out=None, results=None):
    """host_decompress_repeat_packed over host_compress_mixed_repeat_chains_packed's stream, each block in the form single_stream[b]
    (a CPU uint8 tensor) names; results equals huf_decompress_mixed_repeat_packed's.  Synchronous.  Returns (out, results)."""
    return _host_chains_decompress(None, single_stream, packed, offsets, kinds, chain_starts, dst_sizes, chain_hdr_ptrs,
                                   chain_hdr_sizes, out, results)


def _host_chains_decompress(cid, single, packed, offsets, kinds, chain_starts, dst_sizes, chain_hdr_ptrs, chain_hdr_sizes, out, results):
    from . import lib
    dst_sizes = _host_sizes(dst_sizes)
    n = dst_sizes.numel()
    total = int(dst_sizes.sum())
    _host_check(packed, torch.uint8); _host_check(offsets, torch.int64); _host_check(kinds, torch.uint8)
    assert offsets.numel() == n + 1 and kinds.numel() == n and packed.numel() >= int(offsets[-1]), (offsets.numel(), kinds.numel(), n)
    chain_starts, n_chains = _host_chain_args(chain_starts, ((chain_hdr_ptrs, torch.int64, ()), (chain_hdr_sizes, torch.int64, ())))
    if out is None:
        out = torch.empty(total, dtype=torch.uint8)
    if results is None:
        results = torch.empty(n, dtype=torch.int64)
    _host_check(out, torch.uint8); _host_check(results, torch.int64)
    assert out.numel() >= total and results.numel() == n, (out.numel(), total, results.numel(), n)
    head = (n_chains, chain_starts.data_ptr(), n, _host_ptr(out), _host_ptr(dst_sizes), _host_ptr(results), _host_ptr(packed),
            offsets.data_ptr(), _host_ptr(kinds))
    tail = (_host_ptr(chain_hdr_ptrs), _host_ptr(chain_hdr_sizes))
    if cid is None:
        _host_check(single, torch.uint8)
        assert single.numel() == n, (single.numel(), n)
        fn_name = "FSEB200_decompress_host_mixed_repeat_packed"
        r = getattr(lib(), fn_name)(*head, _host_ptr(single), *tail)
    else:
        fn_name = "FSEB200_decompress_host_repeat_packed"
        r = getattr(lib(), fn_name)(cid, *head, *tail)
    _ret(r, fn_name)
    return out, results


# .fse frames (FSEB200_frame_{compress,decompress}_host): codec name -> C codec number
FRAME_CODECS = {"fse": 0, "huf": 1}


def frame_compress(src, codec="fse", block_size_id=5):
    """src (a CPU uint8 tensor, pinned or pageable) as one .fse frame, byte for byte what the reference's `fse -e` ("fse") or
    `fse -h` ("huf") with -B<block_size_id> writes (blocks of 1 KB << block_size_id).  Synchronous.  Returns the frame as a CPU
    uint8 tensor."""
    from . import lib
    cid = FRAME_CODECS[codec]
    _host_check(src, torch.uint8)
    bound = lib().FSEB200_frame_compressBound(src.numel(), block_size_id)
    _ret(bound, "FSEB200_frame_compressBound")
    out = torch.empty(bound, dtype=torch.uint8)
    r = lib().FSEB200_frame_compress_host(cid, block_size_id, out.data_ptr(), out.numel(), _host_ptr(src), src.numel())
    _ret(r, "FSEB200_frame_compress_host")
    return out[:r]


def frame_decompress(frame):
    """the data of an .fse frame (a CPU uint8 tensor), exactly what the reference's `fse -d` writes for it; a frame it rejects
    raises.  Synchronous.  Returns a CPU uint8 tensor."""
    from . import lib
    _host_check(frame, torch.uint8)
    bound = lib().FSEB200_frame_decompress_bound(_host_ptr(frame), frame.numel())
    _ret(bound, "FSEB200_frame_decompress_bound")
    out = torch.empty(bound, dtype=torch.uint8)
    r = lib().FSEB200_frame_decompress_host(_host_ptr(out), out.numel(), _host_ptr(frame), frame.numel())
    _ret(r, "FSEB200_frame_decompress_host")
    return out[:r]


def frame_compress_batch(src, sizes, codec="fse", block_size_id=5):
    """Many .fse frames in one synchronous call: frame f is sizes[f] bytes of `src` (a CPU uint8 tensor, pinned or pageable)
    right after frame f - 1, each coded exactly as frame_compress codes it.  Returns (frames, offsets, results): frame f is
    frames[offsets[f]:offsets[f + 1]] (offsets: int64, n + 1 entries) and results[f] its size or error code (int64)."""
    from . import lib
    cid = FRAME_CODECS[codec]
    sizes = _host_sizes(sizes)
    n = sizes.numel()
    _host_check(src, torch.uint8)
    assert bool((sizes >= 0).all()), "sizes must not be negative"
    assert src.numel() >= int(sizes.sum()), (src.numel(), int(sizes.sum()))
    assert 0 <= block_size_id <= 6, block_size_id
    cap = sum(int(lib().FSEB200_frame_compressBound(int(x), block_size_id)) for x in sizes.tolist())
    frames = torch.empty(cap, dtype=torch.uint8)
    offsets = torch.zeros(n + 1, dtype=torch.int64)                 # nFrames == 0 writes nothing
    results = torch.empty(n, dtype=torch.int64)
    r = lib().FSEB200_frame_compress_host_batch(cid, block_size_id, n, _host_ptr(frames), cap, offsets.data_ptr(), _host_ptr(results),
                                                _host_ptr(src), _host_ptr(sizes))
    _ret(r, "FSEB200_frame_compress_host_batch")
    return frames[:int(offsets[-1])], offsets, results


def frame_decompress_batch(frames, offsets, capacities=None):
    """Many .fse frames in one synchronous call: frame f is frames[offsets[f]:offsets[f + 1]] (a CPU uint8 tensor; offsets int64,
    n + 1 entries, non-decreasing).  Frame f decodes into out[start_f : start_f + capacities[f]], start_f the sum of the earlier
    capacities; capacities default to each frame's FSEB200_frame_decompress_bound (0 for a frame its header walk rejects).
    Returns (out, results): results[f] (int64) is what frame_decompress's C call returns for frame f -- its size or error code;
    a failing frame does not stop the others."""
    from . import lib, is_error
    _host_check(frames, torch.uint8)
    offsets = _host_sizes(offsets)
    n = offsets.numel() - 1
    assert n >= 0, "offsets needs n + 1 entries"
    o = offsets.tolist()
    assert all(o[i] <= o[i + 1] for i in range(n)) and (n == 0 or (o[0] >= 0 and o[-1] <= frames.numel())), "offsets"
    if capacities is None:
        caps = []
        for f in range(n):
            b = lib().FSEB200_frame_decompress_bound(frames.data_ptr() + o[f] if o[f + 1] > o[f] else None, o[f + 1] - o[f])
            caps.append(0 if is_error(b) else int(b))
        capacities = caps
    capacities = _host_sizes(capacities)
    assert capacities.numel() == n and bool((capacities >= 0).all()), (capacities.numel(), n)
    out = torch.empty(int(capacities.sum()), dtype=torch.uint8)
    results = torch.empty(n, dtype=torch.int64)
    r = lib().FSEB200_frame_decompress_host_batch(n, _host_ptr(out), _host_ptr(capacities), _host_ptr(results), _host_ptr(frames),
                                                  offsets.data_ptr())
    _ret(r, "FSEB200_frame_decompress_host_batch")
    return out, results


def _device_check(t, dtype):
    """the device frame calls' tensor check: the dtype, then a contiguous CUDA tensor"""
    assert t.dtype == dtype, ("dtype", t.dtype, dtype)
    assert t.is_cuda and t.is_contiguous(), ("device", t.device, t.is_contiguous())


def _device_sizes(sizes):
    """host int64 sizes or offsets: the device calls take their geometry from the host"""
    if isinstance(sizes, torch.Tensor):
        assert sizes.dtype == torch.int64, sizes.dtype
        sizes = sizes.cpu()
    return _host_sizes(sizes)


def frame_compress_device(src, sizes, codec="fse", block_size_id=5, out=None):
    """Many .fse frames of DEVICE data in one call on the current stream, each exactly what frame_compress_batch gives for it:
    frame f is sizes[f] bytes of `src` (a CUDA uint8 tensor) right after frame f - 1.  `sizes`: int64, on the host or read back
    from a tensor.  With out=None the output holds the sum of the frames' compressBound, always enough; a frame that does not
    fit `out` is not written and its result is dstSize_tooSmall.  Asynchronous.  Returns (out, offsets, results), CUDA int64
    offsets (n + 1 entries) and results (each frame's size or error code)."""
    from . import lib
    cid = FRAME_CODECS[codec]
    sizes = _device_sizes(sizes)
    n = sizes.numel()
    _device_check(src, torch.uint8)
    assert bool((sizes >= 0).all()), "sizes must not be negative"
    assert src.numel() >= int(sizes.sum()), (src.numel(), int(sizes.sum()))
    assert 0 <= block_size_id <= 6, block_size_id
    if out is None:
        cap = sum(int(lib().FSEB200_frame_compressBound(int(x), block_size_id)) for x in sizes.tolist())
        out = torch.empty(cap, dtype=torch.uint8, device=src.device)
    _device_check(out, torch.uint8)
    assert out.device == src.device, (out.device, src.device)
    offsets = torch.zeros(n + 1, dtype=torch.int64, device=src.device)  # nFrames == 0 writes nothing
    results = torch.empty(n, dtype=torch.int64, device=src.device)
    with torch.cuda.device(src.device):
        r = lib().FSEB200_frame_compress_device(cid, block_size_id, n, out.data_ptr() if out.numel() else offsets.data_ptr(), out.numel(),
                                                offsets.data_ptr(), results.data_ptr(), src.data_ptr() if src.numel() else None,
                                                _host_ptr(sizes), _stream_ptr())
    _ret(r, "FSEB200_frame_compress_device")
    return out, offsets, results


def frame_decompress_device(frames, offsets, capacities=None, out=None):
    """Many .fse frames of DEVICE data in one call on the current stream, each exactly what frame_decompress_batch gives for it:
    frame f is frames[offsets[f]:offsets[f + 1]] (a CUDA uint8 tensor; offsets int64 on the host or read back from a tensor,
    n + 1 entries, non-decreasing).  Frame f decodes into out[start_f : start_f + capacities[f]], start_f the sum of the earlier
    capacities; capacities default to each frame's decompress bound (0 for a frame its header walk rejects), from the device's
    header walk.  Synchronises the stream once, after the walk.  Returns (out, results): results (CUDA int64) as
    frame_decompress_batch's."""
    from . import lib, is_error
    offsets = _device_sizes(offsets)
    _device_check(frames, torch.uint8)
    n = offsets.numel() - 1
    assert n >= 0, "offsets needs n + 1 entries"
    o = offsets.tolist()
    assert all(o[i] <= o[i + 1] for i in range(n)) and (n == 0 or (o[0] >= 0 and o[-1] <= frames.numel())), "offsets"
    # every frame empty: no byte is read, but the C call refuses NULL, so a 1-byte buffer stands in (as _host_ptr does)
    stand_in = None if frames.numel() else torch.zeros(1, dtype=torch.uint8, device=frames.device)
    live = (frames if stand_in is None else stand_in).data_ptr()
    with torch.cuda.device(frames.device):
        if capacities is None:
            bounds = torch.zeros(n, dtype=torch.int64)
            if n:
                r = lib().FSEB200_frame_decompress_bound_device(n, bounds.data_ptr(), live, offsets.data_ptr(), _stream_ptr())
                _ret(r, "FSEB200_frame_decompress_bound_device")
            capacities = [0 if is_error(b % (1 << 64)) else int(b) for b in bounds.tolist()]
        capacities = _device_sizes(capacities)
        assert capacities.numel() == n and bool((capacities >= 0).all()), (capacities.numel(), n)
        total = int(capacities.sum())
        if out is None:
            out = torch.empty(max(total, 1), dtype=torch.uint8, device=frames.device)
        _device_check(out, torch.uint8)
        assert out.device == frames.device and out.numel() >= total, (out.device, out.numel(), total)
        results = torch.empty(n, dtype=torch.int64, device=frames.device)
        if n:
            r = lib().FSEB200_frame_decompress_device(n, out.data_ptr(), _host_ptr(capacities), results.data_ptr(), live,
                                                      offsets.data_ptr(), _stream_ptr())
            _ret(r, "FSEB200_frame_decompress_device")
    return out[:total], results
