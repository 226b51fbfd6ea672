// bm25x_blocks.cuh — GPU decoder for the reference's posting-block codec (SURVEY §8 f1: ingest of the stored format).
//
// What is decoded: the payload of a BlockTuple (crates/bm25/src/tuples.rs:973-983) as compression.rs:36-136 wrote it —
//   * full blocks (128 postings): 4-lane vertical bit packing (crates/simd/src/bitpacking.rs:14-98); doc ids are
//     delta-coded against the previous id, the first against SummaryTuple.min_document_id
//     (bitpacking_u32_ordered.rs:82-91); bit width 32 stores raw values (:119-121); term frequencies are not delta-coded;
//   * a token's last, shorter block: 1..4 little-endian bytes per value (bytepacking_u32_ordered.rs / _unordered.rs).
// One warp decodes one block: lane `it` owns input vector `it` of the macro, i.e. values 4*it .. 4*it+3, so the delta
// prefix sum is a 4-element local scan plus one warp scan.  The result is written straight into the engine's posting
// layout {doc, tf << 8 | fieldnorm(doc)}.
#pragma once

#include "bm25x_common.h"

namespace {

#define BM25X_BLKERR_RANGE 1u  // doc id >= n_docs, ids not strictly ascending or wrapped past 2^32, tf == 0
#define BM25X_BLKERR_TF 2u     // tf >= 2^24

__device__ __forceinline__ uint32_t sm_u32(const uint8_t *p) {  // payloads are byte-aligned only
    return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
}

// The four values of input vector `it` from a bit-packed payload of width bw (1..31).
__device__ __forceinline__ void unpack4(const uint8_t *sm, uint32_t bw, uint32_t it, uint32_t v[4]) {
    const uint32_t bit = it * bw, j = bit >> 5, cur = bit & 31u, mask = 0xFFFFFFFFu >> (32u - bw);
#pragma unroll
    for (uint32_t l = 0; l < 4; l++) {
        uint32_t x = sm_u32(sm + 4u * (4u * j + l)) >> cur;
        if (cur + bw > 32u) x |= sm_u32(sm + 4u * (4u * (j + 1u) + l)) << (32u - cur);
        v[l] = x & mask;
    }
}

// Decodes one stream of a block into v[0..3] (values 4*lane .. 4*lane+3).  `delta`: doc ids.  Returns whether the values
// are a running sum seeded with min_doc (false: stored as is).
__device__ __forceinline__ bool decode_stream(const uint8_t *sm, uint8_t meta, uint32_t n, uint32_t lane, bool delta,
                                              uint32_t min_doc, uint32_t v[4]) {
    const uint32_t width = meta & 0x7Fu;
    bool raw = !delta;
    if ((meta >> 7) == 0) {
        if (width == 0) {
            v[0] = v[1] = v[2] = v[3] = 0u;
        } else if (width == 32) {
            raw = true;  // stored as is, even for doc ids
#pragma unroll
            for (uint32_t l = 0; l < 4; l++) v[l] = sm_u32(sm + 4u * (4u * lane + l));
        } else {
            unpack4(sm, width, lane, v);
        }
    } else {
        // a token's last block: 1..4 little-endian bytes per value; width 4 = the values themselves, even for doc ids
        // (crates/simd/src/bytepacking_u32_ordered.rs:195,211: `4 => copy_from_slice`, no delta)
        if (width == 4) raw = true;
#pragma unroll
        for (uint32_t l = 0; l < 4; l++) {
            const uint32_t i = 4u * lane + l;
            uint32_t x = 0;
            if (i < n)
                for (uint32_t k = 0; k < width; k++) x |= (uint32_t)sm[i * width + k] << (8u * k);
            v[l] = x;
        }
    }
    if (!raw) {  // running sum seeded with min_document_id
        v[1] += v[0];
        v[2] += v[1];
        v[3] += v[2];
        uint32_t incl = v[3];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t up = __shfl_up_sync(0xFFFFFFFFu, incl, o);
            if ((int)lane >= o) incl += up;
        }
        const uint32_t base = min_doc + (incl - v[3]);
#pragma unroll
        for (uint32_t l = 0; l < 4; l++) v[l] += base;
    }
    return !raw;
}

constexpr int DEC_WARPS = 8;

__global__ void __launch_bounds__(DEC_WARPS * 32)
k_decode_blocks(uint64_t n_blocks, const uint64_t *__restrict__ term_blk_off, uint32_t n_terms,
                const uint32_t *__restrict__ blk_min, const uint32_t *__restrict__ blk_n,
                const uint8_t *__restrict__ meta_doc, const uint8_t *__restrict__ meta_tf,
                const uint64_t *__restrict__ doc_off, const uint64_t *__restrict__ tf_off,
                const uint8_t *__restrict__ bytes, const uint64_t *__restrict__ off_pad,
                const uint8_t *__restrict__ fieldnorm, uint32_t n_docs, Posting *__restrict__ post,
                uint32_t *__restrict__ err) {
    __shared__ __align__(16) uint8_t stage[DEC_WARPS][2][512];
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
    const uint64_t g = (uint64_t)blockIdx.x * DEC_WARPS + warp;
    if (g >= n_blocks) return;  // whole warps leave; no block-wide barrier below
    uint32_t lo = 0, hi = n_terms;  // token of this block: last t with term_blk_off[t] <= g
    while (lo < hi) {
        const uint32_t mid = (lo + hi + 1) >> 1;
        if (term_blk_off[mid] <= g) lo = mid;
        else hi = mid - 1;
    }
    const uint32_t n = blk_n[g];
    const uint8_t md = meta_doc[g], mt = meta_tf[g];
    const uint32_t nbd = (md >> 7) ? (md & 0x7Fu) * n : (md & 0x7Fu) * 16u;
    const uint32_t nbt = (mt >> 7) ? (mt & 0x7Fu) * n : (mt & 0x7Fu) * 16u;
    const uint8_t *sd = bytes + doc_off[g], *stf = bytes + tf_off[g];
    for (uint32_t i = lane; i < nbd; i += 32) stage[warp][0][i] = sd[i];
    for (uint32_t i = lane; i < nbt; i += 32) stage[warp][1][i] = stf[i];
    __syncwarp();
    uint32_t doc[4], tf[4];
    const uint32_t min_doc = blk_min[g];
    const bool summed = decode_stream(stage[warp][0], md, n, lane, true, min_doc, doc);
    decode_stream(stage[warp][1], mt, n, lane, false, 0u, tf);
    // the reference trusts its pages ("data corruption" panics); here bad blocks are reported, never dereferenced.  A
    // running sum below its seed wrapped past 2^32 (a first delta the encoder never writes: it always starts at 0).
    const uint32_t prev_last = __shfl_up_sync(0xFFFFFFFFu, doc[3], 1);
    uint32_t bad = 0;
    Posting *dst = post + off_pad[lo] + (g - term_blk_off[lo]) * BM25X_BLOCK;
#pragma unroll
    for (uint32_t l = 0; l < 4; l++) {
        const uint32_t i = 4u * lane + l;
        if (i >= n) continue;
        const uint32_t before = l ? doc[l - 1] : prev_last;
        if (doc[l] >= n_docs || (i > 0 && doc[l] <= before) || (summed && doc[l] < min_doc) || tf[l] == 0u)
            bad |= BM25X_BLKERR_RANGE;
        if (tf[l] >= (1u << 24)) bad |= BM25X_BLKERR_TF;
        Posting p;
        p.doc = doc[l];
        p.w = (tf[l] << 8) | (doc[l] < n_docs ? fieldnorm[doc[l]] : 0u);
        dst[i] = p;
    }
    if (bad) atomicOr(err, bad);
}

// Doc ids must also ascend across the blocks of a token (the reference's cursor assumes it, search.rs:440-470).
__global__ void k_check_block_order(const uint64_t *__restrict__ blk_off, uint32_t n_terms, uint64_t n_blocks,
                                    const uint2 *__restrict__ blk, uint32_t *__restrict__ err) {
    const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g == 0 || g >= n_blocks) return;
    uint32_t lo = 0, hi = n_terms;
    while (lo < hi) {
        const uint32_t mid = (lo + hi + 1) >> 1;
        if (blk_off[mid] <= g) lo = mid;
        else hi = mid - 1;
    }
    if (blk_off[lo] == g) return;  // first block of its token
    if (blk[g].x <= blk[g - 1].y) atomicOr(err, BM25X_BLKERR_RANGE);
}

}  // namespace
