// bm25x_keys.cuh — 16-byte token keys on the device, shared by the builds from documents (bm25x_documents.cu) and the
// tsvector casts (bm25x_tsvector.cu).
#pragma once

#include <stdint.h>

#include <cuda/std/tuple>

namespace {

// A 16-byte Element.key as two big-endian words: (hi, lo) order is the bytewise order of the key.
struct Key128 {
    uint64_t hi, lo;
};
__host__ __device__ __forceinline__ bool operator==(const Key128 &a, const Key128 &b) { return a.hi == b.hi && a.lo == b.lo; }
struct Key128Bits {  // CUB's radix decomposer, most significant word first
    __host__ __device__ ::cuda::std::tuple<uint64_t &, uint64_t &> operator()(Key128 &k) const { return {k.hi, k.lo}; }
};

__device__ __forceinline__ uint64_t bswap64(uint64_t x) {
    return ((uint64_t)__byte_perm((uint32_t)x, 0, 0x0123) << 32) | __byte_perm((uint32_t)(x >> 32), 0, 0x0123);
}
// The key's bytes as loaded from memory (two little-endian words) → Key128, and back.
__device__ __forceinline__ Key128 key_of(ulonglong2 raw) { return {bswap64(raw.x), bswap64(raw.y)}; }
__device__ __forceinline__ ulonglong2 raw_of(Key128 k) { return make_ulonglong2(bswap64(k.hi), bswap64(k.lo)); }

}  // namespace
