// micro.h -- op codes and scratch layout of the single-CTA table kernels (micro.cu) shared with the C-ABI layer (capi.cu).
#pragma once
#include <stdint.h>
namespace fseb {
struct MicroArgs { unsigned long long a[6]; };
enum {
    MOP_NORMALIZE = 1, MOP_WRITE_NCOUNT, MOP_READ_NCOUNT, MOP_BUILD_CTABLE, MOP_BUILD_DTABLE,
    MOP_HUF_BUILD_CTABLE, MOP_HUF_WRITE_CTABLE, MOP_HUF_READ_STATS, MOP_HUF_READ_DTABLE_X1,
    MOP_FSE_ENCODE_CT, MOP_FSE_DECODE_DT, MOP_HUF_ENCODE4X_CT, MOP_HUF_DECODE4X1_DT,
    MOP_HUF_ENCODE1X_CT, MOP_HUF_DECODE1X1_DT, MOP_HUF_READ_DTABLE_X2, MOP_HUF_DECODE4X2_DT, MOP_HUF_DECODE1X2_DT
};
// Byte offsets into the kernel's scratch buffer.  Every op reads its input at 0.  Payload ops (the *_usingCTable /
// *_usingDTable calls) take the caller's table image at 0, their input at MICRO_PAYLOAD and write at an offset passed in a3.
constexpr unsigned MICRO_OUT = 4096;                 // results of the table ops
constexpr unsigned MICRO_META = 8192;                // FSE_readNCount: msv, tableLog ; HUF_readStats: rankStats u32[13]
constexpr unsigned MICRO_META_HUF = MICRO_META + 64; // HUF_readStats: nbSymbols, tableLog
constexpr unsigned MICRO_DTABLE_X1 = 16384;          // HUF_readDTableX1 result, u32[1 + 2048]
constexpr unsigned MICRO_DTABLE_X2 = 32768;          // HUF_readDTableX2 result, u32[1 + 4096]
constexpr unsigned MICRO_PAYLOAD = 32768;            // above the largest table image (an FSE or X2 DTable, 16,388 bytes)
constexpr unsigned MICRO_WORK = 65536;               // work area of the serial FSE table builders
}
