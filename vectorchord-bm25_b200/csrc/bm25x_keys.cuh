// bm25x_keys.cuh — 16-byte token keys on the device, shared by the builds from documents (bm25x_documents.cu) and the
// tsvector casts (bm25x_tsvector.cu): the Key128 format, its conversions, the search of a sorted device vocabulary and
// its upload.  The host's search of sorted key bytes is key_ordinal (bm25x_build.h).
#pragma once

#include <stdint.h>

#include <cuda/std/tuple>

#include "bm25x_build.h"

namespace {

constexpr unsigned TPB = 256;  // threads per block of every kernel of both files

unsigned grid_of(uint64_t n) { return (unsigned)((n + TPB - 1) / TPB); }

// A 16-byte Element.key as two big-endian words: (hi, lo) order is the bytewise order of the key.
struct Key128 {
    uint64_t hi, lo;
};
__host__ __device__ __forceinline__ bool operator==(const Key128 &a, const Key128 &b) { return a.hi == b.hi && a.lo == b.lo; }
struct Key128Bits {  // CUB's radix decomposer, most significant word first
    __host__ __device__ ::cuda::std::tuple<uint64_t &, uint64_t &> operator()(Key128 &k) const { return {k.hi, k.lo}; }
};

__host__ __device__ __forceinline__ uint64_t bswap64(uint64_t x) {
#ifdef __CUDA_ARCH__
    return ((uint64_t)__byte_perm((uint32_t)x, 0, 0x0123) << 32) | __byte_perm((uint32_t)(x >> 32), 0, 0x0123);
#else
    return __builtin_bswap64(x);
#endif
}
// The key's bytes as loaded from memory (two little-endian words) → Key128, and back.
__device__ __forceinline__ Key128 key_of(ulonglong2 raw) { return {bswap64(raw.x), bswap64(raw.y)}; }
__host__ __device__ __forceinline__ ulonglong2 raw_of(Key128 k) { return make_ulonglong2(bswap64(k.hi), bswap64(k.lo)); }

// The rank of k in the ascending vocab[0..T): the number of entries below it.
__device__ __forceinline__ uint32_t key_rank(const Key128 *__restrict__ vocab, uint32_t T, Key128 k) {
    uint32_t lo = 0, hi = T;
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        const Key128 v = vocab[mid];
        if (v.hi < k.hi || (v.hi == k.hi && v.lo < k.lo)) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

// Raw keys (as uploaded) → Key128 in place; cnt[i] = 1 when cnt is given (the vocabulary pass's appended entries).
__global__ void k_keys_be(Key128 *__restrict__ keys, uint32_t *__restrict__ cnt, uint64_t n) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const ulonglong2 raw = reinterpret_cast<const ulonglong2 *>(keys)[i];
    keys[i] = key_of(raw);
    if (cnt) cnt[i] = 1u;
}

// A sorted vocabulary (host bytes, T keys) on the current device as Key128, owned by sc.
Key128 *upload_vocab(Scratch &sc, const std::vector<uint8_t> &keys, uint32_t T) {
    Key128 *v = sc.alloc<Key128>(T);
    if (sc.e == cudaSuccess && T) sc.e = cudaMemcpy(v, keys.data(), 16 * (size_t)T, cudaMemcpyHostToDevice);
    if (sc.e == cudaSuccess && T) {
        k_keys_be<<<grid_of(T), TPB>>>(v, nullptr, T);
        sc.e = cudaGetLastError();
    }
    return v;
}

}  // namespace
