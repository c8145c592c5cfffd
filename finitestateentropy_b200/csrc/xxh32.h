// xxh32.h -- XXH32, streaming, on the host: the checksum of the .fse frame's trailer (22 bits of XXH32(data, seed 0) >> 5).
// Written from the public xxHash specification (doc/xxhash_spec.md of the xxHash project): four lanes of 32-bit accumulators
// over 16-byte stripes, a merge, the remaining 4-byte words and bytes, and the avalanche.  update() may be fed any split of the
// input; digest() equals the one-shot hash of everything fed so far.
#pragma once
#include <stddef.h>
#include <stdint.h>
#include <string.h>

namespace fseb {

class Xxh32 {
public:
    explicit Xxh32(uint32_t seed = 0) { reset(seed); }
    void reset(uint32_t seed)
    {
        v_[0] = seed + P1 + P2; v_[1] = seed + P2; v_[2] = seed; v_[3] = seed - P1;
        seed_ = seed; total_ = 0; held_ = 0;
    }
    // One scalar stripe loop, out of line, for every caller.  GCC otherwise packs the four lanes into SSE2 vectors, which have no
    // 32-bit multiply, at about half the speed.  Inlined into the frame decompress's finish step, 1 GiB hashed in 480-490 ms
    // there against 250 ms through FSEB200_XXH32 (host of an H100 80GB HBM3 machine); this loop keeps both at the latter.
    __attribute__((noinline, optimize("no-tree-vectorize"))) void update(const void* data, size_t len)
    {
        const unsigned char* p = static_cast<const unsigned char*>(data);
        total_ += len;
        if (held_) {                                                    // complete the held stripe first
            size_t const take = len < 16 - held_ ? len : 16 - held_;
            memcpy(buf_ + held_, p, take);
            held_ += (unsigned)take; p += take; len -= take;
            if (held_ < 16) return;
            stripe(v_, buf_);
            held_ = 0;
        }
        uint32_t v[4] = { v_[0], v_[1], v_[2], v_[3] };   // lanes in registers: the input, read as bytes, might alias *this
        for (; len >= 16; p += 16, len -= 16) stripe(v, p);
        memcpy(v_, v, sizeof(v));
        memcpy(buf_, p, len);
        held_ = (unsigned)len;
    }
    uint32_t digest() const
    {
        uint32_t h = total_ >= 16 ? rotl(v_[0], 1) + rotl(v_[1], 7) + rotl(v_[2], 12) + rotl(v_[3], 18) : seed_ + P5;
        h += (uint32_t)total_;
        const unsigned char* p = buf_;
        const unsigned char* const end = buf_ + held_;
        for (; p + 4 <= end; p += 4) h = rotl(h + rd32(p) * P3, 17) * P4;
        for (; p < end; p++) h = rotl(h + *p * P5, 11) * P1;
        h ^= h >> 15; h *= P2; h ^= h >> 13; h *= P3; h ^= h >> 16;
        return h;
    }

private:
    static constexpr uint32_t P1 = 2654435761u, P2 = 2246822519u, P3 = 3266489917u, P4 = 668265263u, P5 = 374761393u;
    static uint32_t rotl(uint32_t x, int r) { return (x << r) | (x >> (32 - r)); }
    static uint32_t rd32(const unsigned char* p) { return (uint32_t)p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16 | (uint32_t)p[3] << 24; }
    static void stripe(uint32_t* v, const unsigned char* p)
    {
        for (int i = 0; i < 4; i++) v[i] = rotl(v[i] + rd32(p + 4 * i) * P2, 13) * P1;
    }
    uint32_t v_[4], seed_;
    uint64_t total_;
    unsigned char buf_[16];
    unsigned held_;
};

}  // namespace fseb
