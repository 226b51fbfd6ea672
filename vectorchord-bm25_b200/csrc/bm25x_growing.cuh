// bm25x_growing.cuh — the refresh of a mutable growing segment (bm25x_growing_segment, DESIGN §4.5): the term-major
// postings of the next handle from those of the current one and the postings inserted since, on the device.
//
// Both kernels take one warp per term and read the same inputs: the current handle's lists (old_post at old_off[t],
// old_df[t] postings; old_df == NULL when there is no current handle), the pending lists (pend_doc / pend_tf at
// pend_off[t] .. pend_off[t + 1], ordinals ascending, every one above every indexed ordinal) and the deleted bitmap (bit o
// of del[o >> 5] set = ordinal o deleted).  A posting survives when its document is not deleted.
#pragma once

#include "bm25x_common.h"

__device__ __forceinline__ bool growing_deleted(const uint32_t *__restrict__ del, uint32_t o) {
    return (del[o >> 5] >> (o & 31u)) & 1u;
}

// df[t] = surviving postings of term t's current list and of its pending list.
__global__ void k_growing_count(uint32_t n_terms, const Posting *__restrict__ old_post, const uint64_t *__restrict__ old_off,
                                const uint32_t *__restrict__ old_df, const uint64_t *__restrict__ pend_off,
                                const uint32_t *__restrict__ pend_doc, const uint32_t *__restrict__ del,
                                uint32_t *__restrict__ df) {
    const uint32_t lane = threadIdx.x & 31u, warps = gridDim.x * (blockDim.x >> 5);
    for (uint32_t t = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); t < n_terms; t += warps) {
        uint32_t n = 0;
        if (old_df) {
            const Posting *p = old_post + old_off[t];
            for (uint32_t i = lane; i < old_df[t]; i += 32) n += !growing_deleted(del, p[i].doc);
        }
        for (uint64_t i = pend_off[t] + lane; i < pend_off[t + 1]; i += 32) n += !growing_deleted(del, pend_doc[i]);
        n = __reduce_add_sync(0xFFFFFFFFu, n);
        if (lane == 0) df[t] = n;
    }
}

// Term t's survivors at new_off[t] of the new handle: those of the current list (their words as they are), then those of
// the pending list (w = tf << 8 | fieldnorm[ordinal], as k_build_postings writes it).  Each 32-posting step is an
// order-preserving ballot / popc compaction, so doc ids stay ascending inside the term.
__global__ void k_growing_splice(uint32_t n_terms, const Posting *__restrict__ old_post,
                                 const uint64_t *__restrict__ old_off, const uint32_t *__restrict__ old_df,
                                 const uint64_t *__restrict__ pend_off, const uint32_t *__restrict__ pend_doc,
                                 const uint32_t *__restrict__ pend_tf, const uint32_t *__restrict__ del,
                                 const uint8_t *__restrict__ fieldnorm, const uint64_t *__restrict__ new_off,
                                 Posting *__restrict__ new_post) {
    const uint32_t lane = threadIdx.x & 31u, warps = gridDim.x * (blockDim.x >> 5), lt = (1u << lane) - 1u;
    for (uint32_t t = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); t < n_terms; t += warps) {
        Posting *out = new_post + new_off[t];
        uint32_t pos = 0;
        if (old_df) {
            const Posting *p = old_post + old_off[t];
            const uint32_t n = old_df[t];
            for (uint32_t base = 0; base < n; base += 32) {
                const uint32_t i = base + lane;
                Posting v;
                v.doc = 0;
                v.w = 0;
                bool keep = false;
                if (i < n) {
                    v = p[i];
                    keep = !growing_deleted(del, v.doc);
                }
                const uint32_t m = __ballot_sync(0xFFFFFFFFu, keep);
                if (keep) out[pos + __popc(m & lt)] = v;
                pos += __popc(m);
            }
        }
        const uint64_t p0 = pend_off[t], p1 = pend_off[t + 1];
        for (uint64_t base = p0; base < p1; base += 32) {
            const uint64_t i = base + lane;
            Posting v;
            v.doc = 0;
            v.w = 0;
            bool keep = false;
            if (i < p1) {
                v.doc = pend_doc[i];
                keep = !growing_deleted(del, v.doc);
                if (keep) v.w = (pend_tf[i] << 8) | fieldnorm[v.doc];
            }
            const uint32_t m = __ballot_sync(0xFFFFFFFFu, keep);
            if (keep) out[pos + __popc(m & lt)] = v;
            pos += __popc(m);
        }
    }
}
