// bm25x_seal.cuh — the seal of a growing segment (bm25x_growing_seal, DESIGN §4.5): the postings of a new sealed index
// from the sealed index's, the growing handle's and the dormant ones (postings the handle does not hold), on the device.
//
// Every kernel takes one warp per term and reads its three disjoint sources in doc order:
//   - sealed: term t < s_terms of the sealed handle (s_post / s_pdoc at s_off[t], s_df[t] postings), doc ids old sealed
//     ids, sdel the sealed deleted bitmap (bit d of sdel[d >> 5]);
//   - growing: term t < s_terms of the segment's refreshed handle (g_post at g_off[t], g_df[t] postings; g_df == NULL
//     when there is none), doc ids growing ordinals, gdel the growing deleted bitmap;
//   - dormant: dorm_doc / dorm_tf at dorm_off[t] .. dorm_off[t + 1] (ordinals ascending) for every source term, the
//     postings the growing handle leaves out (terms >= s_terms, terms without sealed postings): disjoint from its terms.
// A posting survives when its document is not deleted.  Every ordinal of the growing side is above every sealed id in
// the new numbering, so a term's survivors stay ascending when written sealed first, then growing, then dormant.
#pragma once

#include "bm25x_common.h"
#include "bm25x_growing.cuh"

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
            if (!growing_deleted(sdel, d)) atomicAdd(&cnt[d], 1u);
        }
    }
}

// df[t] = surviving postings of source term t over the three sources.
__global__ void k_seal_df(uint32_t n_src, uint32_t s_terms, const uint32_t *__restrict__ s_pdoc,
                          const uint64_t *__restrict__ s_off, const uint32_t *__restrict__ s_df,
                          const uint32_t *__restrict__ sdel, const Posting *__restrict__ g_post,
                          const uint64_t *__restrict__ g_off, const uint32_t *__restrict__ g_df,
                          const uint32_t *__restrict__ gdel, const uint64_t *__restrict__ dorm_off,
                          const uint32_t *__restrict__ dorm_doc, uint32_t *__restrict__ df) {
    const uint32_t lane = threadIdx.x & 31u, warps = gridDim.x * (blockDim.x >> 5);
    for (uint32_t t = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); t < n_src; t += warps) {
        uint32_t n = 0;
        if (t < s_terms) {
            const uint32_t *p = s_pdoc + s_off[t];
            for (uint32_t i = lane; i < s_df[t]; i += 32) n += !growing_deleted(sdel, p[i]);
            if (g_df) {
                const Posting *q = g_post + g_off[t];
                for (uint32_t i = lane; i < g_df[t]; i += 32) n += !growing_deleted(gdel, q[i].doc);
            }
        }
        for (uint64_t i = dorm_off[t] + lane; i < dorm_off[t + 1]; i += 32) n += !growing_deleted(gdel, dorm_doc[i]);
        n = __reduce_add_sync(0xFFFFFFFFu, n);
        if (lane == 0) df[t] = n;
    }
}

// New term j (source term src_of[j]) at new_off[j]: its sealed survivors {smap[doc], tf << 8 | fieldnorm[new]}, then its
// growing ones {gmap[ordinal], tf << 8 | fieldnorm[new]} from the handle or the dormant list.  Every word is recomposed:
// the sealed survivors' norms change with their lengths.  Each 32-posting step is an order-preserving ballot / popc
// compaction, as in k_growing_splice.
__global__ void k_seal_splice(uint32_t n_new, const uint32_t *__restrict__ src_of, uint32_t s_terms,
                              const Posting *__restrict__ s_post, const uint64_t *__restrict__ s_off,
                              const uint32_t *__restrict__ s_df, const uint32_t *__restrict__ sdel,
                              const uint32_t *__restrict__ smap, const Posting *__restrict__ g_post,
                              const uint64_t *__restrict__ g_off, const uint32_t *__restrict__ g_df,
                              const uint32_t *__restrict__ gdel, const uint32_t *__restrict__ gmap,
                              const uint64_t *__restrict__ dorm_off, const uint32_t *__restrict__ dorm_doc,
                              const uint32_t *__restrict__ dorm_tf, const uint8_t *__restrict__ fieldnorm,
                              const uint64_t *__restrict__ new_off, Posting *__restrict__ new_post) {
    const uint32_t lane = threadIdx.x & 31u, warps = gridDim.x * (blockDim.x >> 5), lt = (1u << lane) - 1u;
    for (uint32_t j = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); j < n_new; j += warps) {
        const uint32_t t = src_of[j];
        Posting *out = new_post + new_off[j];
        uint32_t pos = 0;
        // one 32-posting step: lane's posting (doc, tf) is written when keep, in lane order
        auto emit = [&](bool keep, uint32_t doc, uint32_t tf) {
            const uint32_t m = __ballot_sync(0xFFFFFFFFu, keep);
            if (keep) {
                Posting v;
                v.doc = doc;
                v.w = (tf << 8) | fieldnorm[doc];
                out[pos + __popc(m & lt)] = v;
            }
            pos += __popc(m);
        };
        if (t < s_terms) {
            const Posting *p = s_post + s_off[t];
            const uint32_t n = s_df[t];
            for (uint32_t base = 0; base < n; base += 32) {
                const uint32_t i = base + lane;
                bool keep = false;
                uint32_t doc = 0, tf = 0;
                if (i < n) {
                    const Posting v = p[i];
                    keep = !growing_deleted(sdel, v.doc);
                    if (keep) {
                        doc = smap[v.doc];
                        tf = v.w >> 8;
                    }
                }
                emit(keep, doc, tf);
            }
            if (g_df) {
                const Posting *q = g_post + g_off[t];
                const uint32_t ng = g_df[t];
                for (uint32_t base = 0; base < ng; base += 32) {
                    const uint32_t i = base + lane;
                    bool keep = false;
                    uint32_t doc = 0, tf = 0;
                    if (i < ng) {
                        const Posting v = q[i];
                        keep = !growing_deleted(gdel, v.doc);
                        if (keep) {
                            doc = gmap[v.doc];
                            tf = v.w >> 8;
                        }
                    }
                    emit(keep, doc, tf);
                }
            }
        }
        const uint64_t d0 = dorm_off[t], d1 = dorm_off[t + 1];
        for (uint64_t base = d0; base < d1; base += 32) {
            const uint64_t i = base + lane;
            bool keep = false;
            uint32_t doc = 0, tf = 0;
            if (i < d1) {
                const uint32_t o = dorm_doc[i];
                keep = !growing_deleted(gdel, o);
                if (keep) {
                    doc = gmap[o];
                    tf = dorm_tf[i];
                }
            }
            emit(keep, doc, tf);
        }
    }
}
