// bm25x_splice.cuh — the term-major postings of a new index handle spliced from lists already on the device
// (DESIGN §4.5): the refresh of a mutable growing segment (bm25x_growing_refresh), its seal (bm25x_growing_seal) and its
// rebind (bm25x_growing_rebind).  The refresh is the seal's splice with identity maps and no sealed source; the rebind's
// splice takes the carried postings of the current handle and those coming up from the host.
//
// A term's postings come from up to three disjoint sources, each read in doc order; a later source's doc ids (after its
// map) are above every earlier source's, so a term's survivors stay ascending when written source by source:
//   - refresh: the current growing handle's list, then the pending list;
//   - seal: the sealed handle's list, then the growing handle's, then the dormant list (the postings the growing handle
//     leaves out: terms >= the sealed n_terms, terms without sealed postings).  Over a document-sharded index each old
//     shard is one such splice on its own device, with local ids; only the last one has the growing sources.
// A posting survives when its document is not deleted.  Every kernel takes one warp per term.
#pragma once

#include "bm25x_common.h"

// One posting source over terms t < n_terms (n_terms == 0: no source), in one of two forms:
//   - handle form (df != NULL): an index handle's lists, post / doc = its pdoc at off[t], df[t] postings (tf = w >> 8);
//   - grouped-list form (df == NULL): doc / tf at off[t] .. off[t + 1], grouped by term on the host.
// del is the deleted bitmap over the source's doc ids (bit d of del[d >> 5] set = doc d deleted); map[d] is the new doc
// id of doc d (map == NULL: d).
struct SpliceSrc {
    const uint64_t *off;
    const uint32_t *df;
    const uint32_t *doc;
    const uint32_t *tf;
    const Posting *post;
    const uint32_t *del;
    const uint32_t *map;
    uint32_t n_terms;
};

// The sources of one splice, in the order their survivors are written (unused entries zeroed).
struct SpliceSources {
    SpliceSrc s[3];
};

__device__ __forceinline__ bool splice_deleted(const uint32_t *__restrict__ del, uint32_t d) {
    return (del[d >> 5] >> (d & 31u)) & 1u;
}

// [b, e): term t's list in source q (empty when q holds none).
__device__ __forceinline__ void splice_range(const SpliceSrc &q, uint32_t t, uint64_t &b, uint64_t &e) {
    b = e = 0;
    if (t < q.n_terms) {
        b = q.off[t];
        e = q.df ? b + q.df[t] : q.off[t + 1];
    }
}

// cnt[d] += 1 per posting of a surviving sealed document d: the length maintain.rs gives it (add_element adds 1 per
// posting, maintain.rs:356-360).  cnt starts zeroed.
__global__ void k_seal_doc_postings(uint32_t s_terms, const uint32_t *__restrict__ s_pdoc, const uint64_t *__restrict__ s_off,
                                    const uint32_t *__restrict__ s_df, const uint32_t *__restrict__ sdel,
                                    uint32_t *__restrict__ cnt) {
    const uint32_t lane = threadIdx.x & 31u, warps = gridDim.x * (blockDim.x >> 5);
    for (uint32_t t = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); t < s_terms; t += warps) {
        const uint32_t *p = s_pdoc + s_off[t];
        for (uint32_t i = lane; i < s_df[t]; i += 32) {
            const uint32_t d = p[i];
            if (!splice_deleted(sdel, d)) atomicAdd(&cnt[d], 1u);
        }
    }
}

// df[t] = surviving postings of term t over the sources, t < n.
__global__ void k_splice_count(uint32_t n, const SpliceSources src, uint32_t *__restrict__ df) {
    const uint32_t lane = threadIdx.x & 31u, warps = gridDim.x * (blockDim.x >> 5);
    for (uint32_t t = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); t < n; t += warps) {
        uint32_t c = 0;
#pragma unroll
        for (int k = 0; k < 3; k++) {
            const SpliceSrc &q = src.s[k];
            uint64_t b, e;
            splice_range(q, t, b, e);
            for (uint64_t i = b + lane; i < e; i += 32) c += !splice_deleted(q.del, q.doc[i]);
        }
        c = __reduce_add_sync(0xFFFFFFFFu, c);
        if (lane == 0) df[t] = c;
    }
}

// The reverse direction, for a rebind (bm25x_growing_rebind): the survivors of the handle-form source q for the terms
// t < n that out_off selects (out_off[t + 1] > out_off[t]; out_off is the exclusive scan of k_splice_count's df over the
// selected terms, 0 for the others), written at out_off[t] as (map[doc], tf) in doc order, so that one download brings
// them to the host, which reads each posting's term off out_off.  The same order-preserving ballot / popc compaction as
// k_splice.
__global__ void k_splice_emit(uint32_t n, const SpliceSrc q, const uint64_t *__restrict__ out_off,
                              uint32_t *__restrict__ out_doc, uint32_t *__restrict__ out_tf) {
    const uint32_t lane = threadIdx.x & 31u, warps = gridDim.x * (blockDim.x >> 5), lt = (1u << lane) - 1u;
    for (uint32_t t = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); t < n; t += warps) {
        uint64_t pos = out_off[t];
        if (out_off[t + 1] == pos) continue;
        const uint64_t b = q.off[t], e = b + q.df[t];
        for (uint64_t base = b; base < e; base += 32) {
            const uint64_t i = base + lane;
            Posting p;
            p.doc = 0;
            p.w = 0;
            bool keep = false;
            if (i < e) {
                p = q.post[i];
                keep = !splice_deleted(q.del, p.doc);
            }
            const uint32_t m = __ballot_sync(0xFFFFFFFFu, keep);
            if (keep) {
                const uint64_t at = pos + __popc(m & lt);
                out_doc[at] = q.map ? q.map[p.doc] : p.doc;
                out_tf[at] = p.w >> 8;
            }
            pos += __popc(m);
        }
    }
}

// New term j (source term src_of[j]; src_of == NULL: j) at new_off[j]: the survivors of each source in order, each
// written as {map[doc], tf << 8 | fieldnorm[map[doc]]}.  Every word is recomposed: the seal changes the sealed
// survivors' norms, and for a refresh the recomposed word is the stored one (a growing ordinal's fieldnorm byte never
// changes).  Each 32-posting step is an order-preserving ballot / popc compaction, so doc ids stay ascending.
__global__ void k_splice(uint32_t n_new, const uint32_t *__restrict__ src_of, const SpliceSources src,
                         const uint8_t *__restrict__ fieldnorm, const uint64_t *__restrict__ new_off,
                         Posting *__restrict__ new_post) {
    const uint32_t lane = threadIdx.x & 31u, warps = gridDim.x * (blockDim.x >> 5), lt = (1u << lane) - 1u;
    for (uint32_t j = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); j < n_new; j += warps) {
        const uint32_t t = src_of ? src_of[j] : j;
        Posting *out = new_post + new_off[j];
        uint32_t pos = 0;
#pragma unroll
        for (int k = 0; k < 3; k++) {
            const SpliceSrc &q = src.s[k];
            uint64_t b, e;
            splice_range(q, t, b, e);
            for (uint64_t base = b; base < e; base += 32) {
                const uint64_t i = base + lane;
                Posting v;
                v.doc = 0;
                v.w = 0;
                bool keep = false;
                if (i < e) {
                    uint32_t tf = 0;
                    if (q.df) {
                        const Posting p = q.post[i];
                        v.doc = p.doc;
                        tf = p.w >> 8;
                    } else {
                        v.doc = q.doc[i];
                    }
                    keep = !splice_deleted(q.del, v.doc);
                    if (keep) {
                        if (!q.df) tf = q.tf[i];
                        if (q.map) v.doc = q.map[v.doc];
                        v.w = (tf << 8) | fieldnorm[v.doc];
                    }
                }
                const uint32_t m = __ballot_sync(0xFFFFFFFFu, keep);
                if (keep) out[pos + __popc(m & lt)] = v;
                pos += __popc(m);
            }
        }
    }
}
