// gen.cu -- measurement inputs on the device: size-parametric restatements of the reference's
// generators, so that bench.py can build a 1 GiB (or a rank's shard of an 8 GiB) input in HBM.
//   generate()    programs/probaGenerator.c:95-126  (4096-cell table, 32-bit LCG, seed 1)
//   generateU16() programs/fuzzerU16.c:107-134
// The LCG  seed' = seed*2654435761 + 2246822519 (mod 2^32), draw = (seed' >> 11) & 4095  is
// jumped ahead per thread by composing affine maps (square-and-multiply), so every thread can
// start anywhere in the stream; the byte at stream position i is identical to the reference's.
#include "common.cuh"
#include "launchers.h"

namespace fseb {

__device__ __forceinline__ u32 lcg_at(u64 i, u32 seed0)       // state after i+1 steps from seed0 (the draw for position i uses it)
{
    u32 A = 2654435761u, Cc = 2246822519u;                    // map for 1 step
    u32 accA = 1, accC = 0;                                   // identity
    u64 k = i + 1;
    while (k) {
        if (k & 1) { accC = accC * A + Cc; accA = accA * A; } // acc = step_map o acc
        Cc = Cc * A + Cc; A = A * A;                          // square the map
        k >>= 1;
    }
    return accA * seed0 + accC;
}

template <typename T>
__global__ void gen_kernel(T* __restrict__ out, u64 n, u64 offset, const T* __restrict__ table, u32 seed0, u32 run)
{
    __shared__ T tab[4096];
    for (int i = threadIdx.x; i < 4096; i += blockDim.x) tab[i] = table[i];
    __syncthreads();
    u64 const first = ((u64)blockIdx.x * blockDim.x + threadIdx.x) * run;
    if (first >= n) return;
    u32 s = lcg_at(offset + first, seed0);
    u64 const last = first + run < n ? first + run : n;
    for (u64 i = first; i < last; i++) {
        out[i] = tab[(s >> 11) & 4095];
        s = s * 2654435761u + 2246822519u;
    }
}

cudaError_t launch_gen8(void* out, u64 n, u64 offset, const void* dTable, u32 seed0, cudaStream_t st)
{
    if (!n) return cudaSuccess;
    u32 const run = 64; u64 const threads = (n + run - 1) / run;
    gen_kernel<u8><<<(unsigned)((threads + 255) / 256), 256, 0, st>>>((u8*)out, n, offset, (const u8*)dTable, seed0, run);
    return cudaGetLastError();
}
cudaError_t launch_gen16(void* out, u64 n, u64 offset, const void* dTable, u32 seed0, cudaStream_t st)
{
    if (!n) return cudaSuccess;
    u32 const run = 32; u64 const threads = (n + run - 1) / run;
    gen_kernel<u16><<<(unsigned)((threads + 255) / 256), 256, 0, st>>>((u16*)out, n, offset, (const u16*)dTable, seed0, run);
    return cudaGetLastError();
}

}  // namespace fseb
