// bm25x_export.cu — a finalized index written out as the reference's stored segment (bm25x_index_export_blocks, DESIGN
// §4.4): the inverse of bm25x_index_create_from_blocks.  The encoder kernels are in bm25x_blocks.cuh, beside the decoder.
#include <string.h>

#include "bm25x_blocks.cuh"

namespace {

// A stream created for one call and destroyed with it: the export never queues behind the handle's searches.
struct OwnStream {
    cudaStream_t s = nullptr;
    ~OwnStream() {
        if (s) cudaStreamDestroy(s);
    }
};

// Payload bytes per chunk of the encode pass: whole blocks, a block holding at most 1 KiB, so every chunk makes progress.
constexpr uint64_t EXPORT_CHUNK = 256ull << 20;

template <typename T>
cudaError_t d2h(T *dst, const T *src, size_t n, cudaStream_t st) {
    return dst && n ? cudaMemcpyAsync(dst, src, sizeof(T) * n, cudaMemcpyDeviceToHost, st) : cudaSuccess;
}

}  // namespace

extern "C" int bm25x_index_export_blocks(const bm25x_index *ix, bm25x_export *out) {
    const char *who = "bm25x_index_export_blocks";
    if (!ix || !out) {
        bm25x_set_error("%s: null argument", who);
        return BM25X_ERR_INVALID;
    }
    const DeviceIndex &d = ix->d;
    const uint32_t N = d.n_docs, T = d.n_terms;
    const uint64_t NB = d.n_blocks;
    if (ix->h_df.size() != T) {
        bm25x_set_error("%s: replica not finalized", who);
        return BM25X_ERR_INVALID;
    }
    // the Wand pairs flush writes use the segment's own avgdl; a handle that scores with another segment's statistics
    // has other s1 tables
    if (!own_statistics(ix)) {
        bm25x_set_error("%s: the index scores with another segment's statistics (a growing handle); its Wand pairs would "
                        "not be the ones flush writes", who);
        return BM25X_ERR_INVALID;
    }
    if (out->term_key && ix->h_keys.empty() && T) {
        bm25x_set_error("%s: term_key given, but the index was created without term keys", who);
        return BM25X_ERR_INVALID;
    }

    // ---- directory pass: every block's summary and metadata bytes (about 35 bytes per block on the device) ----
    Scratch sc(ix->device);
    OwnStream own;
    sc.e = cudaSetDevice(ix->device);
    if (sc.e == cudaSuccess) sc.e = cudaStreamCreateWithFlags(&own.s, cudaStreamNonBlocking);
    const cudaStream_t st = own.s;
    uint32_t *d_min = sc.alloc<uint32_t>(NB), *d_max = sc.alloc<uint32_t>(NB), *d_n = sc.alloc<uint32_t>(NB);
    uint8_t *d_md = sc.alloc<uint8_t>(NB), *d_mt = sc.alloc<uint8_t>(NB), *d_wfn = sc.alloc<uint8_t>(NB);
    uint32_t *d_wtf = sc.alloc<uint32_t>(NB);
    double *d_wv = sc.alloc<double>(NB);
    uint64_t *d_doff = sc.alloc<uint64_t>(NB);
    const double k1p1 = ix->k1 + 1.0;
    if (sc.e == cudaSuccess && NB) {
        k_export_dir<<<(unsigned)((NB + DEC_WARPS - 1) / DEC_WARPS), DEC_WARPS * 32, 0, st>>>(
            NB, d.blk_off, T, d.post_off, d.df, d.post, d.blk, d.s1d, k1p1, d_min, d_max, d_n, d_md, d_mt, d_wfn, d_wtf,
            d_wv);
        sc.e = cudaGetLastError();
    }
    std::vector<uint32_t> h_n(NB);
    std::vector<uint8_t> h_md(NB), h_mt(NB);
    if (sc.e == cudaSuccess) sc.e = d2h(h_n.data(), d_n, NB, st);
    if (sc.e == cudaSuccess) sc.e = d2h(h_md.data(), d_md, NB, st);
    if (sc.e == cudaSuccess) sc.e = d2h(h_mt.data(), d_mt, NB, st);
    if (sc.e == cudaSuccess) sc.e = cudaStreamSynchronize(st);
    if (sc.e != cudaSuccess) return cuda_refusal(who, "directory pass", sc.e);

    // ---- payload offsets: per block the doc payload, then the tf payload, blocks in token order ----
    std::vector<uint64_t> h_doff(NB), h_toff(NB);
    uint64_t total = 0;
    for (uint64_t g = 0; g < NB; g++) {
        h_doff[g] = total;
        total += stream_bytes(h_md[g], h_n[g]);
        h_toff[g] = total;
        total += stream_bytes(h_mt[g], h_n[g]);
    }
    out->n_bytes = total;
    if (!out->bytes) return BM25X_OK;  // sizing call
    if (out->bytes_cap < total) {
        bm25x_set_error("%s: bytes_cap %llu is below the payload size %llu", who, (unsigned long long)out->bytes_cap,
                        (unsigned long long)total);
        return BM25X_ERR_INVALID;
    }

    // ---- every device allocation before the first output byte ----
    const uint64_t chunk_cap = std::min(total, EXPORT_CHUNK);
    uint8_t *d_stage = sc.alloc<uint8_t>(chunk_cap);
    uint8_t *d_tfn = sc.alloc<uint8_t>(T);
    uint32_t *d_ttf = sc.alloc<uint32_t>(T);
    if (sc.e == cudaSuccess && NB) sc.e = cudaMemcpyAsync(d_doff, h_doff.data(), sizeof(uint64_t) * NB, cudaMemcpyHostToDevice, st);
    if (sc.e == cudaSuccess && T) {
        k_export_tokens<<<(unsigned)(((uint64_t)T * 32 + 255) / 256), 256, 0, st>>>(T, d.blk_off, d_wv, d_wfn, d_wtf, d_tfn,
                                                                                    d_ttf);
        sc.e = cudaGetLastError();
    }
    if (sc.e == cudaSuccess) sc.e = cudaStreamSynchronize(st);
    if (sc.e != cudaSuccess) return cuda_refusal(who, "token pass", sc.e);

    // ---- the outputs: per document, per token, per block ----
    out->sum_doc_len = ix->sum_len;
    if (out->term_key && T) memcpy(out->term_key, ix->h_keys.data(), (size_t)T * 16);
    if (out->tok_df && T) memcpy(out->tok_df, ix->h_df.data(), sizeof(uint32_t) * T);
    if (out->blk_n && NB) memcpy(out->blk_n, h_n.data(), sizeof(uint32_t) * NB);
    if (out->blk_meta_doc && NB) memcpy(out->blk_meta_doc, h_md.data(), NB);
    if (out->blk_meta_tf && NB) memcpy(out->blk_meta_tf, h_mt.data(), NB);
    if (out->blk_doc_off && NB) memcpy(out->blk_doc_off, h_doff.data(), sizeof(uint64_t) * NB);
    if (out->blk_tf_off && NB) memcpy(out->blk_tf_off, h_toff.data(), sizeof(uint64_t) * NB);
    const cudaError_t copies[] = {
        d2h(out->doc_fieldnorm, d.fieldnorm, N, st),
        d2h(out->payload, d.payload, (size_t)N * 3, st),
        d2h(out->tok_wand_fieldnorm, d_tfn, T, st),
        d2h(out->tok_wand_tf, d_ttf, T, st),
        d2h(out->term_blk_off, (const uint64_t *)d.blk_off, (size_t)T + 1, st),
        d2h(out->blk_min_doc, d_min, NB, st),
        d2h(out->blk_max_doc, d_max, NB, st),
        d2h(out->blk_wand_fieldnorm, d_wfn, NB, st),
        d2h(out->blk_wand_tf, d_wtf, NB, st),
    };
    for (cudaError_t e : copies)
        if (sc.e == cudaSuccess) sc.e = e;

    // ---- encode pass: runs of whole blocks of at most EXPORT_CHUNK payload bytes, each encoded into the staging buffer
    // at (offset - chunk base) and copied out ----
    for (uint64_t g0 = 0; g0 < NB && sc.e == cudaSuccess;) {
        const uint64_t base = h_doff[g0];
        uint64_t g1 = g0;
        while (g1 < NB && (g1 + 1 < NB ? h_doff[g1 + 1] : total) - base <= chunk_cap) g1++;
        const uint64_t end = g1 < NB ? h_doff[g1] : total;
        k_export_encode<<<(unsigned)((g1 - g0 + DEC_WARPS - 1) / DEC_WARPS), DEC_WARPS * 32, 0, st>>>(
            g0, g1 - g0, d.blk_off, T, d.post_off, d.df, d.post, d.blk, d_md, d_mt, d_doff, base, d_stage);
        sc.e = cudaGetLastError();
        if (sc.e == cudaSuccess && end > base)
            sc.e = cudaMemcpyAsync(out->bytes + base, d_stage, end - base, cudaMemcpyDeviceToHost, st);
        g0 = g1;
    }
    if (sc.e == cudaSuccess) sc.e = cudaStreamSynchronize(st);
    if (sc.e != cudaSuccess) return cuda_refusal(who, "block encode/download", sc.e);
    return BM25X_OK;
}
