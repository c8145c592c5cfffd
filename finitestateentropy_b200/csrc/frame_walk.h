// frame_walk.h -- the .fse frame header walk, one step at a time, for the host (host_pipeline.cu walk_frame) and the device
// (frame_device.cu: one frame per thread).  The layout is described in frame.cu; the verdicts are the exit codes of the
// reference's FIO_decompressFilename (programs/fileio.c), and blocks that would overrun its buffers are corruption_detected.
#pragma once
#include "common.cuh"

namespace fseb {
namespace fmt {

constexpr u32 MAGIC_FSE = 0x183E2309u, MAGIC_HUF = 0x183E3309u;
constexpr u64 FRAME_HEADER = 5, FRAME_TRAILER = 3;
enum { BT_COMPRESSED = 0, BT_RAW = 1, BT_RLE = 2, BT_END = 3 };
// A block's role in a frame body (frame.cu's Body::role): it starts the frame, ends it, and carries the trailer written on the
// device with the frame's index into the hashes in the upper 32 bits
enum : u64 { ROLE_FIRST = 1, ROLE_LAST = 2, ROLE_HASHED = 4 };

struct FrameBlock { u64 head, payload, rSize, cSize; int type; };   // header and payload offsets in the frame

// Where a walk is: the next header byte (0 before the frame header), and what the frame header said
struct WalkState { u64 pos = 0, bs = 0; int codec = 0; u32 checksum = 0; };
// walk_step's answers besides a verdict (an error value): block k was read, or the trailer was (its 22 bits in s.checksum)
constexpr u64 WALK_BLOCK = 1, WALK_END = 2;

__host__ __device__ __forceinline__ u64 be16(const u8* p) { return (u64)p[0] << 8 | p[1]; }

// The next step of the walk of frame f (size bytes): at pos 0 the frame header and then the first block, else one block or the
// trailer.  Returns WALK_BLOCK with k filled, WALK_END, or the verdict where the walk stops (nothing more may be read).
__host__ __device__ inline u64 walk_step(const u8* f, u64 size, WalkState& s, FrameBlock& k)
{
    if (s.pos == 0) {
        if (size < FRAME_HEADER) return err(E_SRC_WRONG);                                       // exit 30
        u32 const magic = (u32)f[0] | (u32)f[1] << 8 | (u32)f[2] << 16 | (u32)f[3] << 24;
        if (magic != MAGIC_FSE && magic != MAGIC_HUF) return err(E_GENERIC);                  // 31 (zlibh too)
        if (f[4] > 6) return err(E_GENERIC);                                                   // 32
        s.codec = magic == MAGIC_HUF;
        s.bs = (u64)1024 << f[4];
        s.pos = FRAME_HEADER;
        if (s.pos >= size) return err(E_SRC_WRONG);                                            // 34
    }
    u64 pos = s.pos;
    k.head = pos;
    k.type = f[pos] >> 6;
    if (k.type == BT_END) {
        if (pos + FRAME_TRAILER > size) return err(E_SRC_WRONG);                              // 43
        s.checksum = (u32)be16(f + pos + 1) | (u32)(f[pos] & 0x3F) << 16;
        return WALK_END;
    }
    bool const full = f[pos] & 0x20;
    pos++;
    k.rSize = s.bs;
    if (!full) {
        if (pos + 2 > size) return err(E_SRC_WRONG);                                           // 35
        k.rSize = be16(f + pos); pos += 2;
    }
    if (k.type == BT_COMPRESSED) {
        if (pos + 2 > size) return err(E_SRC_WRONG);                                           // 36
        k.cSize = be16(f + pos); pos += 2;
    } else k.cSize = k.type == BT_RAW ? k.rSize : 1;
    if (k.cSize > s.bs + 4) return err(E_CORRUPT);                                             // past its input buffer
    if (pos + k.cSize + 1 > size) return err(E_SRC_WRONG);                                     // 38: payload + next header byte
    if (k.type != BT_RAW && k.rSize > s.bs) return err(E_CORRUPT);                             // past its output buffer
    k.payload = pos;
    s.pos = pos + k.cSize;
    return WALK_BLOCK;
}

__host__ __device__ __forceinline__ u32 trailer_checksum(u32 h) { return (h >> 5) & ((1u << 22) - 1); }

}  // namespace fmt
}  // namespace fseb
