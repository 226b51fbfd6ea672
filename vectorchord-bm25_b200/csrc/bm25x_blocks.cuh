// bm25x_blocks.cuh — GPU decoder for the reference's posting-block codec (SURVEY §8 f1: ingest of the stored format).
//
// What is decoded: the payload of a BlockTuple (crates/bm25/src/tuples.rs:973-983) as compression.rs:36-136 wrote it —
//   * full blocks (128 postings): 4-lane vertical bit packing (crates/simd/src/bitpacking.rs:14-98); doc ids are
//     delta-coded against the previous id, the first against SummaryTuple.min_document_id
//     (bitpacking_u32_ordered.rs:82-91); bit width 32 stores raw values (:119-121); term frequencies are not delta-coded;
//   * a token's last, shorter block: 1..4 little-endian bytes per value (bytepacking_u32_ordered.rs / _unordered.rs).
// One warp decodes one block: lane `it` owns input vector `it` of the macro, i.e. values 4*it .. 4*it+3, so the delta
// prefix sum is a 4-element local scan plus one warp scan.  The result is written straight into the engine's posting
// layout {doc, tf << 8 | fieldnorm(doc)}.  The encoder of the same codec (bm25x_index_export_blocks) is at the end of
// this file, with the same lane mapping.
#pragma once

#include "bm25x_build.h"

namespace {

#define BM25X_BLKERR_RANGE 1u  // doc id >= n_docs, ids not strictly ascending or wrapped past 2^32, tf == 0
#define BM25X_BLKERR_TF 2u     // tf >= 2^24
#define BM25X_BLKERR_DIR 4u    // a staged directory entry that does not describe a payload inside the staged bytes
#define BM25X_BLKERR_WAND 8u   // SummaryTuple.wand_* is not the block's arg-max

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

// The posting-check rule of the decoder: error bits of decoded posting i (doc, tf) of a block, `before` the id ahead of it.
// A running sum below its seed wrapped past 2^32 (a first delta the encoder never writes: it always starts at 0).
__device__ __forceinline__ uint32_t posting_errors(uint32_t doc, uint32_t tf, uint32_t i, uint32_t before, bool summed,
                                                   uint32_t min_doc, uint32_t n_docs) {
    uint32_t bad = 0;
    if (doc >= n_docs || (i > 0 && doc <= before) || (summed && doc < min_doc) || tf == 0u) bad |= BM25X_BLKERR_RANGE;
    if (tf >= (1u << 24)) bad |= BM25X_BLKERR_TF;
    return bad;
}

// The stored SummaryTuple.(wand_fieldnorm, wand_term_frequency) of a block against the block's bound blk_ub (k_block_desc's
// block_bound): tf() and Cache::evaluate round differently, so the last f32 ulp either way is allowed.  wand_tf is a full
// u32 and is never packed into a posting word.
__device__ __forceinline__ bool wand_pair_ok(uint32_t wand_tf, uint8_t wand_fn, double s0, const double *__restrict__ s1d,
                                             float blk_ub) {
    const float ub = block_bound(tf_score(wand_tf, wand_fn, s0, s1d));
    return ub <= blk_ub * 1.0000003f && ub >= blk_ub * 0.9999997f;
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
    const uint32_t t = owner_of(term_blk_off, n_terms, g);  // token of this block
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
    // the reference trusts its pages ("data corruption" panics); here bad blocks are reported, never dereferenced
    const uint32_t prev_last = __shfl_up_sync(0xFFFFFFFFu, doc[3], 1);
    uint32_t bad = 0;
    Posting *dst = post + off_pad[t] + (g - term_blk_off[t]) * BM25X_BLOCK;
#pragma unroll
    for (uint32_t l = 0; l < 4; l++) {
        const uint32_t i = 4u * lane + l;
        if (i >= n) continue;
        bad |= posting_errors(doc[l], tf[l], i, l ? doc[l - 1] : prev_last, summed, min_doc, n_docs);
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
    if (blk_off[owner_of(blk_off, n_terms, g)] == g) return;  // first block of its token
    if (blk[g].x <= blk[g - 1].y) atomicOr(err, BM25X_BLKERR_RANGE);
}

// ---- document-sharded index from stored blocks (bm25x_index_create_sharded_from_blocks, DESIGN §4.7): the kernels below
// read blocks gathered from the caller's directory into a staging buffer, back to back with rebased offsets ----

// Bytes of one stream of an n-posting block: bit packing (flag 0) only for full blocks, 16 words of `width` <= 32 bits; byte
// packing 1..4 bytes per value (compression.rs:43-62).  ~0u: a layout the encoder never writes.
__host__ __device__ __forceinline__ uint32_t stream_bytes(uint8_t meta, uint32_t n) {
    const uint32_t w = meta & 0x7Fu;
    if ((meta >> 7) == 0) return w <= 32u && n == BM25X_BLOCK ? w * 16u : ~0u;
    return w >= 1u && w <= 4u && n >= 1u && n <= BM25X_BLOCK ? w * n : ~0u;
}

// Copies one stream of a staged block into the warp's 512-byte stage.  False (the warp leaves, the caller reports
// BM25X_BLKERR_DIR) when the entry does not describe a payload inside bytes[0, n_bytes).
__device__ __forceinline__ bool stage_stream(uint8_t *stage, uint32_t lane, const uint8_t *__restrict__ bytes,
                                             uint64_t n_bytes, uint8_t meta, uint32_t n, uint64_t off) {
    const uint32_t nb = stream_bytes(meta, n);
    if (nb == ~0u || off > n_bytes || nb > n_bytes - off) return false;
    for (uint32_t i = lane; i < nb; i += 32) stage[i] = bytes[off + i];
    return true;
}

// Whole-segment check: one warp per stored block of the chunk [g0, g0 + n_blocks) (directory arrays chunk-local).  Exactly
// k_decode_blocks' posting checks against the segment's n_docs, without writing postings, and per block its decoded (first,
// last) doc id: k_check_block_order's rule and the shards' block selection run on these on the host.  With wand_fn:
// k_check_block_wand's test against the bound k_block_desc computes from the same postings (needs the segment's fieldnorm,
// s0d, s1d).  With doc_count: every posting counted on its document (the balanced shard bounds).
__global__ void __launch_bounds__(DEC_WARPS * 32)
k_check_blocks(uint64_t g0, uint64_t n_blocks, const uint64_t *__restrict__ term_blk_off, uint32_t n_terms,
               const uint32_t *__restrict__ blk_min, const uint32_t *__restrict__ blk_n,
               const uint8_t *__restrict__ meta_doc, const uint8_t *__restrict__ meta_tf,
               const uint64_t *__restrict__ doc_off, const uint64_t *__restrict__ tf_off, const uint8_t *__restrict__ bytes,
               uint64_t n_bytes, const uint8_t *__restrict__ fieldnorm, uint32_t n_docs,
               const uint8_t *__restrict__ wand_fn, const uint32_t *__restrict__ wand_tf, const double *__restrict__ s0d,
               const double *__restrict__ s1d, uint2 *__restrict__ first_last, uint32_t *__restrict__ doc_count,
               uint32_t *__restrict__ err) {
    __shared__ __align__(16) uint8_t stage[DEC_WARPS][2][512];
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
    const uint64_t j = (uint64_t)blockIdx.x * DEC_WARPS + warp;
    if (j >= n_blocks) return;  // whole warps leave; no block-wide barrier below
    const uint32_t n = blk_n[j];
    const uint8_t md = meta_doc[j], mt = meta_tf[j];
    if (!stage_stream(stage[warp][0], lane, bytes, n_bytes, md, n, doc_off[j]) ||
        !stage_stream(stage[warp][1], lane, bytes, n_bytes, mt, n, tf_off[j])) {
        if (lane == 0) {
            first_last[j] = make_uint2(BM25X_DOC_INF, BM25X_DOC_INF);
            atomicOr(err, BM25X_BLKERR_DIR);
        }
        return;
    }
    __syncwarp();
    uint32_t doc[4], tf[4];
    const uint32_t min_doc = blk_min[j];
    const bool summed = decode_stream(stage[warp][0], md, n, lane, true, min_doc, doc);
    decode_stream(stage[warp][1], mt, n, lane, false, 0u, tf);
    const bool wand = wand_fn != nullptr;
    const double s0 = wand ? s0d[owner_of(term_blk_off, n_terms, g0 + j)] : 0.0;  // of the block's token
    const uint32_t prev_last = __shfl_up_sync(0xFFFFFFFFu, doc[3], 1);
    uint32_t bad = 0, last_mine = doc[0];
    double best = 0.0;
#pragma unroll
    for (uint32_t l = 0; l < 4; l++) {
        const uint32_t i = 4u * lane + l;
        if (i >= n) continue;
        bad |= posting_errors(doc[l], tf[l], i, l ? doc[l - 1] : prev_last, summed, min_doc, n_docs);
        if (i == n - 1) last_mine = doc[l];
        const bool in = doc[l] < n_docs;
        if (wand) {
            const double v = posting_score((tf[l] << 8) | (in ? fieldnorm[doc[l]] : 0u), s0, s1d);
            best = v > best ? v : best;
        }
        if (doc_count && in) atomicAdd(doc_count + doc[l], 1u);
    }
    const uint32_t first = __shfl_sync(0xFFFFFFFFu, doc[0], 0), last = __shfl_sync(0xFFFFFFFFu, last_mine, (n - 1) >> 2);
    if (wand)
        for (int o = 16; o > 0; o >>= 1) {
            const double v = __shfl_xor_sync(0xFFFFFFFFu, best, o);
            best = v > best ? v : best;
        }
    if (bad) atomicOr(err, bad);
    if (lane == 0) {
        first_last[j] = make_uint2(first, last);
        if (wand && !wand_pair_ok(wand_tf[j], wand_fn[j], s0, s1d, block_bound(best)))
            atomicOr(err, BM25X_BLKERR_WAND);
    }
}

// Per-shard count: one warp per selected block (its decoded (first, last) from the check pass): of its postings, how many
// fall in the shard's documents [lo, hi) (.x) and how many lie below lo (.y; ids ascend inside a block, so those in range
// are one run after them).  A block inside [lo, hi) counts n without decoding; only the blocks a bound cuts (at most two per
// token) are decoded, doc ids only.
__global__ void __launch_bounds__(DEC_WARPS * 32)
k_count_shard_blocks(uint64_t n_blocks, const uint2 *__restrict__ first_last, const uint32_t *__restrict__ blk_min,
                     const uint32_t *__restrict__ blk_n, const uint8_t *__restrict__ meta_doc,
                     const uint64_t *__restrict__ doc_off, const uint8_t *__restrict__ bytes, uint64_t n_bytes, uint32_t lo,
                     uint32_t hi, uint2 *__restrict__ count_skip, uint32_t *__restrict__ err) {
    __shared__ __align__(16) uint8_t stage[DEC_WARPS][512];
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
    const uint64_t j = (uint64_t)blockIdx.x * DEC_WARPS + warp;
    if (j >= n_blocks) return;
    const uint32_t n = blk_n[j];
    const uint2 fl = first_last[j];
    if (fl.x >= lo && fl.y < hi) {
        if (lane == 0) count_skip[j] = make_uint2(n, 0u);
        return;
    }
    const uint8_t md = meta_doc[j];
    if (!stage_stream(stage[warp], lane, bytes, n_bytes, md, n, doc_off[j])) {
        if (lane == 0) {
            count_skip[j] = make_uint2(0u, 0u);
            atomicOr(err, BM25X_BLKERR_DIR);
        }
        return;
    }
    __syncwarp();
    uint32_t doc[4];
    decode_stream(stage[warp], md, n, lane, true, blk_min[j], doc);
    uint32_t in = 0, below = 0;
#pragma unroll
    for (uint32_t l = 0; l < 4; l++) {
        const uint32_t i = 4u * lane + l;
        if (i >= n) continue;
        below += doc[l] < lo;
        in += doc[l] >= lo && doc[l] < hi;
    }
    in = __reduce_add_sync(0xFFFFFFFFu, in);
    below = __reduce_add_sync(0xFFFFFFFFu, below);
    if (lane == 0) count_skip[j] = make_uint2(in, below);
}

// Per-shard decode: one warp per selected block; its postings in [lo, lo + n_local) written as {doc - lo, tf << 8 |
// fieldnorm(local)} at the token's padded offset + rank[j] (the in-range postings of the token's earlier selected blocks) +
// the posting's rank among the block's in-range ones.  The posting checks run again (n_docs: the segment's); a position
// outside the token's shard df (a payload that decodes otherwise than it did in the count) is reported, never written.
__global__ void __launch_bounds__(DEC_WARPS * 32)
k_decode_shard_blocks(uint64_t n_blocks, const uint64_t *__restrict__ sel_off, uint32_t n_terms,
                      const uint32_t *__restrict__ blk_min, const uint32_t *__restrict__ blk_n,
                      const uint8_t *__restrict__ meta_doc, const uint8_t *__restrict__ meta_tf,
                      const uint64_t *__restrict__ doc_off, const uint64_t *__restrict__ tf_off,
                      const uint8_t *__restrict__ bytes, uint64_t n_bytes, const uint2 *__restrict__ count_skip,
                      const uint32_t *__restrict__ rank, uint32_t n_docs, uint32_t lo, uint32_t n_local,
                      const uint64_t *__restrict__ off_pad, const uint32_t *__restrict__ df,
                      const uint8_t *__restrict__ fieldnorm, Posting *__restrict__ post, uint32_t *__restrict__ err) {
    __shared__ __align__(16) uint8_t stage[DEC_WARPS][2][512];
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
    const uint64_t j = (uint64_t)blockIdx.x * DEC_WARPS + warp;
    if (j >= n_blocks) return;
    const uint32_t n = blk_n[j];
    const uint8_t md = meta_doc[j], mt = meta_tf[j];
    if (!stage_stream(stage[warp][0], lane, bytes, n_bytes, md, n, doc_off[j]) ||
        !stage_stream(stage[warp][1], lane, bytes, n_bytes, mt, n, tf_off[j])) {
        if (lane == 0) atomicOr(err, BM25X_BLKERR_DIR);
        return;
    }
    __syncwarp();
    const uint32_t t = owner_of(sel_off, n_terms, j);  // token of this block
    uint32_t doc[4], tf[4];
    const uint32_t min_doc = blk_min[j];
    const bool summed = decode_stream(stage[warp][0], md, n, lane, true, min_doc, doc);
    decode_stream(stage[warp][1], mt, n, lane, false, 0u, tf);
    const uint32_t prev_last = __shfl_up_sync(0xFFFFFFFFu, doc[3], 1);
    const uint32_t skip = count_skip[j].y, r0 = rank[j], n_t = df[t];
    Posting *dst = post + off_pad[t];
    uint32_t bad = 0;
#pragma unroll
    for (uint32_t l = 0; l < 4; l++) {
        const uint32_t i = 4u * lane + l;
        if (i >= n) continue;
        bad |= posting_errors(doc[l], tf[l], i, l ? doc[l - 1] : prev_last, summed, min_doc, n_docs);
        const uint32_t local = doc[l] - lo;
        if (doc[l] < lo || local >= n_local) continue;
        const uint64_t pos = (uint64_t)r0 + i - skip;
        if (i < skip || pos >= n_t || tf[l] >= (1u << 24)) {
            bad |= BM25X_BLKERR_RANGE;
            continue;
        }
        Posting p;
        p.doc = local;
        p.w = (tf[l] << 8) | fieldnorm[local];
        dst[pos] = p;
    }
    if (bad) atomicOr(err, bad);
}

// ---- export (bm25x_index_export_blocks, DESIGN §4.4): the encoder of the same codec, compress_document_ids /
// compress_term_frequencies (compression.rs:36-110), over an index's own blocks.  One warp per block with the decoder's
// lane mapping: lane `it` holds postings 4*it .. 4*it+3 ----

// Metadata byte of a stream of n values whose OR has `bits` significant bits: the bit width of a full block, else the
// byte width div_ceil(bits, 8).max(1) with the flag (compression.rs:43-62, bytepacking_u32_ordered.rs:29).
__host__ __device__ __forceinline__ uint8_t stream_meta(uint32_t bits, uint32_t n) {
    if (n == BM25X_BLOCK) return (uint8_t)bits;
    const uint32_t by = (bits + 7u) / 8u;
    return (uint8_t)(0x80u | (by ? by : 1u));
}

// Block g of an index (blocks of 128 postings per term, the last shorter) in the lane's registers: returns n, fills
// doc / w (tf << 8 | fieldnorm) of postings 4*lane .. 4*lane+3, zero past n.
__device__ __forceinline__ uint32_t load_block(uint64_t g, uint32_t lane, const uint64_t *__restrict__ blk_off,
                                               uint32_t n_terms, const uint64_t *__restrict__ post_off,
                                               const uint32_t *__restrict__ df, const Posting *__restrict__ post,
                                               uint32_t doc[4], uint32_t w[4]) {
    const uint32_t t = owner_of(blk_off, n_terms, g);
    const uint64_t k = g - blk_off[t];
    const uint64_t rest = df[t] - k * BM25X_BLOCK;
    const uint32_t n = rest < BM25X_BLOCK ? (uint32_t)rest : BM25X_BLOCK;
    const Posting *src = post + post_off[t] + k * BM25X_BLOCK;
#pragma unroll
    for (uint32_t l = 0; l < 4; l++) {
        const uint32_t i = 4u * lane + l;
        const Posting p = i < n ? src[i] : Posting{0u, 0u};
        doc[l] = p.doc;
        w[l] = p.w;
    }
    return n;
}

// The doc-id stream's values as compress_document_ids stores them: deltas from min_doc, or the ids themselves at bit width
// 32 / byte width 4 (bitpacking_u32_ordered.rs:119-121, bytepacking_u32_ordered.rs:195).  Returns the OR of the deltas.
__device__ __forceinline__ uint32_t doc_deltas(const uint32_t doc[4], uint32_t n, uint32_t lane, uint32_t min_doc,
                                               uint32_t v[4]) {
    const uint32_t before = __shfl_up_sync(0xFFFFFFFFu, doc[3], 1);
    uint32_t acc = 0;
#pragma unroll
    for (uint32_t l = 0; l < 4; l++) {
        const uint32_t prev = l ? doc[l - 1] : (lane ? before : min_doc);
        v[l] = 4u * lane + l < n ? doc[l] - prev : 0u;
        acc |= v[l];
    }
    return __reduce_or_sync(0xFFFFFFFFu, acc);
}

// Directory pass: per block its SummaryTuple (min / max from blk, n, the Wand pair) and the two metadata bytes.  wand_v =
// the pair's tf() (bm25.rs:291-295: (tf·(k1+1)) / (tf + s1[fn]), k1p1 = k1 + 1), which the token pass folds.
__global__ void __launch_bounds__(DEC_WARPS * 32)
k_export_dir(uint64_t n_blocks, const uint64_t *__restrict__ blk_off, uint32_t n_terms,
             const uint64_t *__restrict__ post_off, const uint32_t *__restrict__ df, const Posting *__restrict__ post,
             const uint2 *__restrict__ blk, const double *__restrict__ s1d, double k1p1, uint32_t *__restrict__ min_doc,
             uint32_t *__restrict__ max_doc, uint32_t *__restrict__ blk_n, uint8_t *__restrict__ meta_doc,
             uint8_t *__restrict__ meta_tf, uint8_t *__restrict__ wand_fn, uint32_t *__restrict__ wand_tf,
             double *__restrict__ wand_v) {
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
    const uint64_t g = (uint64_t)blockIdx.x * DEC_WARPS + warp;
    if (g >= n_blocks) return;  // whole warps leave
    uint32_t doc[4], w[4], v[4];
    const uint32_t n = load_block(g, lane, blk_off, n_terms, post_off, df, post, doc, w);
    const uint2 mm = blk[g];
    const uint32_t or_doc = doc_deltas(doc, n, lane, mm.x, v);
    // Wand::push (bm25.rs:297-318): a posting replaces the pair only when its tf() is strictly greater, so the first
    // posting of the largest tf() wins; the start pair (0.0, 255, 0) is never replaced by NaN
    uint32_t or_tf = 0, pos = 0xFFFFFFFFu;
    double best = 0.0;
#pragma unroll
    for (uint32_t l = 0; l < 4; l++) {
        const uint32_t i = 4u * lane + l, tf = w[l] >> 8;
        or_tf |= tf;
        if (i >= n) continue;
        const double tfd = (double)tf;
        const double x = __ddiv_rn(__dmul_rn(tfd, k1p1), __dadd_rn(tfd, s1d[w[l] & 0xFFu]));
        if (x > best) {
            best = x;
            pos = i;
        }
    }
    or_tf = __reduce_or_sync(0xFFFFFFFFu, or_tf);
    for (int o = 16; o > 0; o >>= 1) {  // arg-max; equal tf(): the earlier posting
        const double ob = __shfl_xor_sync(0xFFFFFFFFu, best, o);
        const uint32_t op = __shfl_xor_sync(0xFFFFFFFFu, pos, o);
        if (ob > best || (ob == best && op < pos)) {
            best = ob;
            pos = op;
        }
    }
    uint32_t mine = w[0];
#pragma unroll
    for (uint32_t l = 1; l < 4; l++)
        if ((pos & 3u) == l) mine = w[l];
    const uint32_t win = __shfl_sync(0xFFFFFFFFu, mine, (pos >> 2) & 31u);
    if (lane == 0) {
        min_doc[g] = mm.x;
        max_doc[g] = mm.y;
        blk_n[g] = n;
        meta_doc[g] = stream_meta(32u - __clz(or_doc), n);
        meta_tf[g] = stream_meta(32u - __clz(or_tf), n);
        wand_fn[g] = pos == 0xFFFFFFFFu ? 255u : (uint8_t)(win & 0xFFu);
        wand_tf[g] = pos == 0xFFFFFFFFu ? 0u : win >> 8;
        wand_v[g] = best;
    }
}

// Token pass: one warp per token folds its blocks' pairs with Wand::extend (bm25.rs:319-325) in block order: strictly
// greater tf() replaces, so the earliest block wins; a token without blocks keeps (255, 0).
__global__ void k_export_tokens(uint32_t n_terms, const uint64_t *__restrict__ blk_off, const double *__restrict__ wand_v,
                                const uint8_t *__restrict__ wand_fn, const uint32_t *__restrict__ wand_tf,
                                uint8_t *__restrict__ tok_fn, uint32_t *__restrict__ tok_tf) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t t = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (t >= n_terms) return;  // whole warps leave
    double best = 0.0;
    uint64_t pos = ~0ull;
    for (uint64_t g = blk_off[t] + lane; g < blk_off[t + 1]; g += 32)
        if (wand_v[g] > best) {
            best = wand_v[g];
            pos = g;
        }
    for (int o = 16; o > 0; o >>= 1) {
        const double ob = __shfl_xor_sync(0xFFFFFFFFu, best, o);
        const uint64_t op = __shfl_xor_sync(0xFFFFFFFFu, pos, o);
        if (ob > best || (ob == best && op < pos)) {
            best = ob;
            pos = op;
        }
    }
    if (lane == 0) {
        tok_fn[t] = pos == ~0ull ? 255u : wand_fn[pos];
        tok_tf[t] = pos == ~0ull ? 0u : wand_tf[pos];
    }
}

// One stream of a block, values v (4 per lane) under metadata `meta`, written to dst (byte-aligned).  Full block, width
// 1..31: the compress! macro (bitpacking.rs:14-52) — value `it` of lane stream l at bit it*bw of that stream, output word
// 4j + l holds its bits 32j .. 32j+31 — OR-ed together in the warp's shared stage (a value spans at most two words), then
// copied out; width 32: the values as they are.  Shorter block: `width` little-endian bytes per value.
__device__ __forceinline__ void encode_stream(uint32_t *stage, uint8_t meta, uint32_t n, uint32_t lane,
                                              const uint32_t v[4], uint8_t *__restrict__ dst) {
    const uint32_t width = meta & 0x7Fu;
    if (meta >> 7) {
#pragma unroll
        for (uint32_t l = 0; l < 4; l++) {
            const uint32_t i = 4u * lane + l;
            if (i < n)
                for (uint32_t k = 0; k < width; k++) dst[i * width + k] = (uint8_t)(v[l] >> (8u * k));
        }
        return;
    }
    if (width == 0) return;
    if (width == 32) {
#pragma unroll
        for (uint32_t l = 0; l < 4; l++) stage[4u * lane + l] = v[l];
    } else {
        for (uint32_t i = lane; i < 4u * width; i += 32) stage[i] = 0u;
        __syncwarp();
        const uint32_t bit = lane * width, j = bit >> 5, cur = bit & 31u;
#pragma unroll
        for (uint32_t l = 0; l < 4; l++) {
            atomicOr(stage + 4u * j + l, v[l] << cur);
            if (cur + width > 32u) atomicOr(stage + 4u * (j + 1u) + l, v[l] >> (32u - cur));
        }
    }
    __syncwarp();
    const uint8_t *bytes = reinterpret_cast<const uint8_t *>(stage);  // little-endian words: the payload's byte order
    for (uint32_t i = lane; i < 16u * width; i += 32) dst[i] = bytes[i];
    __syncwarp();  // the stage is reused by the next stream
}

// Encode pass over the blocks [g0, g0 + n_blocks): block g's doc payload at out + doc_off[g] - base, its tf payload right
// after it.  The metadata bytes are the directory pass's.
__global__ void __launch_bounds__(DEC_WARPS * 32)
k_export_encode(uint64_t g0, uint64_t n_blocks, const uint64_t *__restrict__ blk_off, uint32_t n_terms,
                const uint64_t *__restrict__ post_off, const uint32_t *__restrict__ df, const Posting *__restrict__ post,
                const uint2 *__restrict__ blk, const uint8_t *__restrict__ meta_doc, const uint8_t *__restrict__ meta_tf,
                const uint64_t *__restrict__ doc_off, uint64_t base, uint8_t *__restrict__ out) {
    __shared__ __align__(16) uint32_t stage[DEC_WARPS][BM25X_BLOCK];
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
    const uint64_t g = g0 + (uint64_t)blockIdx.x * DEC_WARPS + warp;
    if (g >= g0 + n_blocks) return;  // whole warps leave; no block-wide barrier below
    uint32_t doc[4], w[4], v[4];
    const uint32_t n = load_block(g, lane, blk_off, n_terms, post_off, df, post, doc, w);
    const uint8_t md = meta_doc[g], mt = meta_tf[g];
    doc_deltas(doc, n, lane, blk[g].x, v);
    if (md == 32u || md == (0x80u | 4u))  // stored as they are
#pragma unroll
        for (uint32_t l = 0; l < 4; l++) v[l] = doc[l];
    uint8_t *dst = out + (doc_off[g] - base);
    encode_stream(stage[warp], md, n, lane, v, dst);
#pragma unroll
    for (uint32_t l = 0; l < 4; l++) v[l] = w[l] >> 8;
    encode_stream(stage[warp], mt, n, lane, v, dst + stream_bytes(md, n));
}

// Ingest check: the stored SummaryTuple.(wand_fieldnorm, wand_term_frequency) of a block must evaluate to the block's
// real maximum (it is the arg-max of the block's own postings, flush.rs:101-110); anything else is a corrupt index.
__global__ void k_check_block_wand(uint64_t n_blocks, const uint64_t *__restrict__ blk_off, uint32_t n_terms,
                                   const uint8_t *__restrict__ wand_fn, const uint32_t *__restrict__ wand_tf,
                                   const double *__restrict__ s0d, const double *__restrict__ s1d,
                                   const float *__restrict__ blk_ub, uint32_t *__restrict__ err) {
    uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= n_blocks) return;
    const uint32_t t = owner_of(blk_off, n_terms, g);
    if (!wand_pair_ok(wand_tf[g], wand_fn[g], s0d[t], s1d, blk_ub[g])) atomicOr(err, BM25X_BLKERR_WAND);
}

}  // namespace
