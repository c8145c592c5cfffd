"""Host-side predicates for the FSE / FSE-U16 per-block descriptor calls (FSEB200_FSE{,U16}_{compress,decompress}_blocks).  They
restate the guards of csrc/fse_codec.cu one to one:

  encode_route   fse_route_kernel: the verdict the route kernel settles, or the encode kernel a block goes to ('cta': a whole
                 number of 64-byte groups, at least one, at a 16-byte aligned source; 'warp': everything else);
  cta_groups     fse_encode_cta_kernel: ring groups per block, and the CTA's hand-over count (its largest block's);
  decode_path    fse_decode_cta_kernel: whether a block's lane starts in the check-free windowed loop or on the exact
                 byte-granular model, including sameHi computed from the block's own compressed extent;
  read_range     the addresses the decoder may read for a block: from its first aligned 16-byte piece up to its last byte
                 rounded up to a word -- inside the 32-byte sectors the call's contract makes readable.

The GPU tests assert with them that their fixtures reach both encoders, CTAs of mixed sizes and both decode paths;
tests/test_fse_blocks_model.py pins them on the CPU."""
FSE_BLOCK_MAX = 1 << 30
ERR_GENERIC = 2 ** 64 - 1
ERR_SRC_WRONG = 2 ** 64 - 3
MARGIN = 24                         # container bytes the windowed loop leaves unread below a chunk


def fse_bytes(size, wide):
    """a descriptor size in bytes (U16 sizes count symbols); FSE_BLOCK_MAX + 1 for anything above the limit"""
    if wide:
        return FSE_BLOCK_MAX + 1 if size > FSE_BLOCK_MAX // 2 else 2 * size
    return FSE_BLOCK_MAX + 1 if size > FSE_BLOCK_MAX else size


def encode_route(src_addr, size, wide):
    """'cta' | 'warp' | the block's settled value (int)"""
    if wide and src_addr & 1:
        return ERR_GENERIC
    if wide and size <= 1:
        return size
    n = fse_bytes(size, wide)
    if n > FSE_BLOCK_MAX:
        return ERR_SRC_WRONG
    return "cta" if n >= 64 and n % 64 == 0 and src_addr % 16 == 0 else "warp"


def cta_groups(block_bytes):
    """(groups per block, the CTA's ring hand-over count) for the coded blocks of one CTA"""
    groups = [n // 64 for n in block_bytes]
    return groups, max(groups, default=0)


def same_hi(out_addr, out_bytes, c_addr, csize):
    return ((out_addr + out_bytes) >> 32) == (out_addr >> 32) and ((c_addr + csize + 3) >> 32) == ((c_addr & ~15) >> 32)


def _hibit(v):
    return v.bit_length() - 1


def decode_path(cblock, csize, hsize, tl, out_addr, c_addr, out_symbols, wide):
    """'windowed' or 'exact' for a block whose header (hsize bytes, table log tl) was accepted: the first chunk test of
    fse_decode_cta_kernel after bs_open and the initial state reads"""
    if out_addr % (8 if wide else 4) or not same_hi(out_addr, out_symbols * (2 if wide else 1), c_addr, csize):
        return "exact"
    length = csize - hsize
    if length < 8:
        return "exact"
    last = int(cblock[csize - 1])
    if last == 0:
        return "exact"
    at, used = length - 8, 8 - _hibit(last)
    for _ in range(1 if wide else 2):                 # BIT_readBits(tl) + BIT_reloadDStream per initial state
        used += tl
        if used > 64 or at < 8:
            return "exact"
        at -= used >> 3
        used &= 7
    if at < MARGIN:
        return "exact"
    chunks = min((at - MARGIN) // (7 if wide else 6), out_symbols // 4)
    return "windowed" if chunks > 0 else "exact"


def read_range(c_addr, csize):
    """[lo, hi): every address the decoder may read for a block of csize compressed bytes at c_addr"""
    return c_addr & ~15, (c_addr + csize + 3) & ~3     # window words below the top; header, bs_open and ld64u stay in the block


def readable_range(c_addr, csize):
    """[lo, hi): what the contract makes readable -- the 32-byte sectors holding the block's first and last bytes"""
    last = c_addr + max(csize, 1) - 1
    return c_addr & ~31, (last | 31) + 1
