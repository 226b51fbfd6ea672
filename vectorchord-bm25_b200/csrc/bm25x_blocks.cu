// bm25x_blocks.cu — ingest of the reference's stored posting blocks (SURVEY §8 f1): one index, or a document-sharded
// index whose shards each decode only the blocks that hold their documents.  Every handle is built by the contract of
// bm25x_build.h; the decode and check kernels are in bm25x_blocks.cuh.
#include <string.h>

#include <algorithm>

#include "bm25x_blocks.cuh"

// ---- f1: the sealed segment as the reference stores it (blocks in the codec of compression.rs), decoded on the GPU ----

// Host validation of the stored blocks, shared by bm25x_index_create_from_blocks and
// bm25x_index_create_sharded_from_blocks: same codes, same messages.  Gives each token's postings (df) and their total P.
// check_device == false leaves the device check to the caller (the sharded build checks its shard arguments first, so
// that they are refused without a GPU).
static int validate_blocks(const bm25x_blocks *c, int device, bool check_device, std::vector<uint32_t> &df,
                           uint64_t &n_post) {
    const char *who = "bm25x_index_create_from_blocks";
    const uint32_t N = c->n_docs, T = c->n_terms;
    const uint64_t NB = c->n_blocks;
    if (!c->term_blk_off || (NB && (!c->blk_min_doc || !c->blk_n || !c->blk_meta_doc || !c->blk_meta_tf ||
                                    !c->blk_doc_off || !c->blk_tf_off || (c->n_bytes && !c->bytes)))) {
        bm25x_set_error("%s: empty or malformed corpus", who);
        return BM25X_ERR_INVALID;
    }
    int rc = check_common(who, N, c->doc_len ? (const void *)c->doc_len : (const void *)c->doc_fieldnorm, c->k1, c->b, device);
    if (rc != BM25X_OK && (check_device || rc != BM25X_ERR_CUDA)) return rc;
    if (c->term_blk_off[0] != 0 || c->term_blk_off[T] != NB) {
        bm25x_set_error("%s: term_blk_off must run from 0 to n_blocks", who);
        return BM25X_ERR_INVALID;
    }
    // ---- host-side validation of the block directory (payloads are validated by the decoder on the device) ----
    df.assign(T, 0);
    uint64_t P = 0;
    int bad = 0;
#pragma omp parallel for schedule(dynamic, 256) reduction(| : bad) reduction(+ : P) num_threads(bm25x_host_threads(0))
    for (uint32_t t = 0; t < T; t++) {
        const uint64_t b0 = c->term_blk_off[t], b1 = c->term_blk_off[t + 1];
        if (b1 < b0 || b1 > NB) {
            bad |= 1;
            df[t] = 0;
            continue;
        }
        uint64_t n_t = 0;
        for (uint64_t g = b0; g < b1; g++) {
            const uint32_t n = c->blk_n[g];
            // flush.rs:80-90: every block of a token holds 128 postings except the last one
            if (n == 0 || n > BM25X_BLOCK || (n < BM25X_BLOCK && g + 1 != b1)) bad |= 1;
            const uint8_t metas[2] = {c->blk_meta_doc[g], c->blk_meta_tf[g]};
            const uint64_t offs[2] = {c->blk_doc_off[g], c->blk_tf_off[g]};
            for (int s = 0; s < 2; s++) {
                const uint32_t w = metas[s] & 0x7Fu;
                uint64_t nbytes;
                if ((metas[s] >> 7) == 0) {  // compression.rs:43-52: bit packing only for full blocks, width <= 32
                    if (w > 32 || n != BM25X_BLOCK) bad |= 2;
                    nbytes = (uint64_t)w * 16;
                } else {                      // compression.rs:53-62: 1..4 bytes per value
                    if (w < 1 || w > 4) bad |= 2;
                    nbytes = (uint64_t)w * n;
                }
                if (offs[s] > c->n_bytes || nbytes > c->n_bytes - offs[s]) bad |= 1;
            }
            n_t += n;
        }
        if (n_t > N) bad |= 1;
        df[t] = (uint32_t)std::min<uint64_t>(n_t, N);
        P += n_t;
    }
    if (bad & 1) {
        bm25x_set_error("%s: corrupt block directory (block sizes, token ranges or payload offsets)", who);
        return BM25X_ERR_INVALID;
    }
    if (bad & 2) {
        bm25x_set_error("%s: corrupt block metadata (bitwidth out of bound / unexpected input len)", who);
        return BM25X_ERR_INVALID;
    }
    n_post = P;
    return check_keys(who, c->term_key, T);
}

// The refusal for the error bits of the decode and check kernels (bm25x_blocks.cuh), with the messages of
// bm25x_index_create_from_blocks whichever entry point decoded the blocks.
static int blocks_refusal(uint32_t h_err) {
    const char *who = "bm25x_index_create_from_blocks";
    if (h_err & BM25X_BLKERR_RANGE) {
        bm25x_set_error("%s: corrupt blocks (doc ids must be < n_docs and strictly ascending per token, tf != 0)", who);
        return BM25X_ERR_INVALID;
    }
    if (h_err & BM25X_BLKERR_TF) {
        bm25x_set_error("%s: term frequency >= 2^24 is not supported by the packed posting layout", who);
        return BM25X_ERR_UNSUPPORTED;
    }
    if (h_err & BM25X_BLKERR_WAND) {
        bm25x_set_error("%s: corrupt blocks (SummaryTuple wand_fieldnorm/wand_term_frequency is not the block's maximum)", who);
        return BM25X_ERR_INVALID;
    }
    if (h_err & BM25X_BLKERR_DIR) {  // only blocks staged by the sharded build: the caller's directory changed under it
        bm25x_set_error("%s: corrupt block directory (block sizes, token ranges or payload offsets)", who);
        return BM25X_ERR_INVALID;
    }
    return BM25X_OK;
}

extern "C" int bm25x_index_create_from_blocks(const bm25x_blocks *c, int device, bm25x_index **out) {
    const char *who = "bm25x_index_create_from_blocks";
    if (!c || !out) {
        bm25x_set_error("%s: null argument", who);
        return BM25X_ERR_INVALID;
    }
    *out = nullptr;
    std::vector<uint32_t> df;
    uint64_t P = 0;
    int rc = validate_blocks(c, device, true, df, P);
    if (rc != BM25X_OK) return rc;
    const uint32_t N = c->n_docs, T = c->n_terms;
    const uint64_t NB = c->n_blocks;

    BuildMeta m{N, T, c->doc_len, c->payload, c->term_key, c->k1, c->b, df.data(), P};
    m.fieldnorm = c->doc_fieldnorm;
    m.sum_len = c->sum_doc_len;
    IndexGuard ix;
    rc = index_begin(m, nullptr, device, ix);
    if (rc != BM25X_OK) return rc;
    DeviceIndex &d = ix->d;

    // ---- upload the directory + payloads, decode on the device ----
    uint32_t h_err = 0;
    Scratch sc(device);
    const uint64_t *d_tbo = sc.up(c->term_blk_off, (size_t)T + 1);
    const uint32_t *d_min = sc.up(c->blk_min_doc, NB), *d_n = sc.up(c->blk_n, NB);
    const uint8_t *d_md = sc.up(c->blk_meta_doc, NB), *d_mt = sc.up(c->blk_meta_tf, NB);
    const uint64_t *d_doff = sc.up(c->blk_doc_off, NB), *d_toff = sc.up(c->blk_tf_off, NB);
    const uint8_t *d_bytes = sc.up(c->bytes, c->n_bytes);
    uint32_t *d_err = sc.up(&h_err, 1);
    if (sc.e == cudaSuccess && NB) {
        k_decode_blocks<<<(unsigned)((NB + DEC_WARPS - 1) / DEC_WARPS), DEC_WARPS * 32>>>(
            NB, d_tbo, T, d_min, d_n, d_md, d_mt, d_doff, d_toff, d_bytes, d.post_off, d.fieldnorm, N, d.post, d_err);
        sc.e = cudaGetLastError();
    }
    if (sc.e == cudaSuccess) sc.e = index_finish_device(ix.get());
    if (c->blk_wand_fieldnorm && c->blk_wand_tf) {  // the stored per-block bounds must be those of the decoded postings
        const uint8_t *d_wfn = sc.up(c->blk_wand_fieldnorm, NB);
        const uint32_t *d_wtf = sc.up(c->blk_wand_tf, NB);
        if (sc.e == cudaSuccess && NB) {
            k_check_block_wand<<<(unsigned)((NB + 255) / 256), 256>>>(NB, d.blk_off, T, d_wfn, d_wtf, d.s0d, d.s1d, d.blk_ub,
                                                                     d_err);
            sc.e = cudaGetLastError();
        }
    }
    if (sc.e == cudaSuccess && NB > 1) {
        k_check_block_order<<<(unsigned)((NB + 255) / 256), 256>>>(d.blk_off, T, NB, d.blk, d_err);
        sc.e = cudaGetLastError();
    }
    if (sc.e == cudaSuccess) sc.e = cudaMemcpy(&h_err, d_err, sizeof(h_err), cudaMemcpyDeviceToHost);
    if (sc.e != cudaSuccess) return cuda_refusal(who, "block upload/decode", sc.e);
    rc = blocks_refusal(h_err);
    if (rc == BM25X_OK) *out = ix.release();
    return rc;
}

// ---- a document-sharded index from the stored blocks (DESIGN §4.7): one check pass over the whole segment on shard 0's
// device, then per shard a decode of just the stored blocks that hold its documents, on its own device ----

// Directory entries and payloads of some stored blocks, gathered back to back with the offsets rebased to `bytes`: what a
// kernel of bm25x_blocks.cuh reads for just these blocks.  The directory has passed validate_blocks.
struct StagedBlocks {
    std::vector<uint32_t> min, n;
    std::vector<uint8_t> md, mt;
    std::vector<uint64_t> doff, toff;
    std::vector<uint8_t> bytes;

    void gather(const bm25x_blocks *c, const uint64_t *ids, size_t nb) {
        min.resize(nb);
        n.resize(nb);
        md.resize(nb);
        mt.resize(nb);
        doff.resize(nb);
        toff.resize(nb);
        uint64_t pos = 0;
        for (size_t j = 0; j < nb; j++) {
            const uint64_t g = ids[j];
            min[j] = c->blk_min_doc[g];
            n[j] = c->blk_n[g];
            md[j] = c->blk_meta_doc[g];
            mt[j] = c->blk_meta_tf[g];
            doff[j] = pos;
            pos += stream_bytes(md[j], n[j]);
            toff[j] = pos;
            pos += stream_bytes(mt[j], n[j]);
        }
        bytes.resize(pos ? pos : 1);
        n_bytes = pos;
#pragma omp parallel for schedule(static) num_threads(bm25x_host_threads(0))
        for (size_t j = 0; j < nb; j++) {
            const uint64_t g = ids[j];
            memcpy(bytes.data() + doff[j], c->bytes + c->blk_doc_off[g], toff[j] - doff[j]);
            memcpy(bytes.data() + toff[j], c->bytes + c->blk_tf_off[g], stream_bytes(mt[j], n[j]));
        }
    }
    uint64_t n_bytes = 0;
};

// The check pass: every stored block decoded once on `device`, in chunks of at most 256 MiB of payload (so the compressed
// segment never has to fit on one GPU), with every check bm25x_index_create_from_blocks makes on the device.  Gives the
// error bits, each block's decoded (first, last) doc id, and with cum != NULL the postings of the documents < d (cum[d]).
// fieldnorm and the s0 / s1 tables of stats are the segment's; they are read only to check the stored wand pairs.
static int check_stored_blocks(const char *who, const bm25x_blocks *c, const uint8_t *fieldnorm, const Stats &stats,
                               int device, std::vector<uint2> &first_last, std::vector<uint64_t> *cum, uint32_t &h_err) {
    const uint32_t N = c->n_docs, T = c->n_terms;
    const uint64_t NB = c->n_blocks;
    const bool wand = c->blk_wand_fieldnorm && c->blk_wand_tf;
    first_last.assign(NB, make_uint2(0, 0));
    h_err = 0;
    Scratch sc(device);
    sc.e = cudaSetDevice(device);
    const uint64_t *d_tbo = sc.up(c->term_blk_off, (size_t)T + 1);
    const uint8_t *d_fn = wand ? sc.up(fieldnorm, N) : nullptr;  // the whole segment's norms: a block may straddle a bound
    const double *d_s0d = wand ? sc.up(stats.s0d.data(), T) : nullptr;
    const double *d_s1d = wand ? sc.up(stats.s1d, 256) : nullptr;
    uint32_t *d_cnt = cum ? sc.alloc<uint32_t>(N) : nullptr;
    if (d_cnt && sc.e == cudaSuccess) sc.e = cudaMemset(d_cnt, 0, sizeof(uint32_t) * (size_t)N);
    uint32_t *d_err = sc.up(&h_err, 1);
    const uint64_t CH_BYTES = 256ull << 20, CH_BLOCKS = 1ull << 21;
    std::vector<uint64_t> ids;
    StagedBlocks st;
    for (uint64_t g0 = 0; g0 < NB && sc.e == cudaSuccess;) {
        uint64_t g1 = g0, nbytes = 0;
        while (g1 < NB && g1 - g0 < CH_BLOCKS) {
            const uint64_t b = (uint64_t)stream_bytes(c->blk_meta_doc[g1], c->blk_n[g1]) +
                               stream_bytes(c->blk_meta_tf[g1], c->blk_n[g1]);
            if (g1 > g0 && nbytes + b > CH_BYTES) break;
            nbytes += b;
            g1++;
        }
        const uint64_t nb = g1 - g0;
        ids.resize(nb);
        for (uint64_t j = 0; j < nb; j++) ids[j] = g0 + j;
        st.gather(c, ids.data(), nb);
        Scratch ch(device);
        const uint32_t *d_min = ch.up(st.min.data(), nb), *d_n = ch.up(st.n.data(), nb);
        const uint8_t *d_md = ch.up(st.md.data(), nb), *d_mt = ch.up(st.mt.data(), nb);
        const uint64_t *d_doff = ch.up(st.doff.data(), nb), *d_toff = ch.up(st.toff.data(), nb);
        const uint8_t *d_bytes = ch.up(st.bytes.data(), st.bytes.size());
        const uint8_t *d_wfn = wand ? ch.up(c->blk_wand_fieldnorm + g0, nb) : nullptr;
        const uint32_t *d_wtf = wand ? ch.up(c->blk_wand_tf + g0, nb) : nullptr;
        uint2 *d_fl = ch.alloc<uint2>(nb);
        if (ch.e == cudaSuccess) {
            k_check_blocks<<<(unsigned)((nb + DEC_WARPS - 1) / DEC_WARPS), DEC_WARPS * 32>>>(
                g0, nb, d_tbo, T, d_min, d_n, d_md, d_mt, d_doff, d_toff, d_bytes, st.n_bytes, d_fn, N, d_wfn, d_wtf, d_s0d,
                d_s1d, d_fl, d_cnt, d_err);
            ch.e = cudaGetLastError();
        }
        if (ch.e == cudaSuccess) ch.e = cudaMemcpy(first_last.data() + g0, d_fl, sizeof(uint2) * nb, cudaMemcpyDeviceToHost);
        sc.e = ch.e;
        g0 = g1;
    }
    if (sc.e == cudaSuccess) sc.e = cudaMemcpy(&h_err, d_err, sizeof(h_err), cudaMemcpyDeviceToHost);
    if (sc.e == cudaSuccess && cum) {
        std::vector<uint32_t> cnt(N);
        sc.e = cudaMemcpy(cnt.data(), d_cnt, sizeof(uint32_t) * (size_t)N, cudaMemcpyDeviceToHost);
        cum->assign((size_t)N + 1, 0);
        for (uint32_t d = 0; d < N; d++) (*cum)[(size_t)d + 1] = (*cum)[d] + cnt[d];
    }
    if (sc.e != cudaSuccess) return cuda_refusal(who, "block upload/decode", sc.e);
    // k_check_block_order's rule on the decoded (first, last): ids ascend across the blocks of a token
    uint32_t order = 0;
#pragma omp parallel for schedule(dynamic, 256) reduction(| : order) num_threads(bm25x_host_threads(0))
    for (uint32_t t = 0; t < T; t++)
        for (uint64_t g = c->term_blk_off[t] + 1; g < c->term_blk_off[t + 1]; g++)
            if (first_last[g].x <= first_last[g - 1].y) order |= BM25X_BLKERR_RANGE;
    h_err |= order;
    return BM25X_OK;
}

// Shard s, documents [lo, hi), from the stored blocks, on `device`: the blocks whose decoded [first, last] meets [lo, hi)
// gathered with rebased offsets (host memory beyond the caller's: this payload), counted (k_count_shard_blocks), then the
// shard index allocated with the whole segment's statistics, decoded into place (k_decode_shard_blocks) and finished as
// every index is.
static int build_shard_from_blocks(const char *who, const bm25x_blocks *c, const std::vector<uint2> &first_last,
                                   const Stats &stats, uint32_t s, uint32_t lo, uint32_t hi, int device, IndexGuard &ix) {
    const uint32_t T = c->n_terms;
    // ---- select: per token the run of its blocks with last >= lo and first < hi (both ascend along the chain) ----
    std::vector<uint64_t> sel_b0(T), sel_off((size_t)T + 1, 0);
#pragma omp parallel for schedule(dynamic, 256) num_threads(bm25x_host_threads(0))
    for (uint32_t t = 0; t < T; t++) {
        const uint2 *a = first_last.data() + c->term_blk_off[t], *e = first_last.data() + c->term_blk_off[t + 1];
        const uint2 *b0 = std::partition_point(a, e, [&](const uint2 &f) { return f.y < lo; });
        const uint2 *b1 = std::partition_point(b0, e, [&](const uint2 &f) { return f.x < hi; });
        sel_b0[t] = (uint64_t)(b0 - first_last.data());
        sel_off[(size_t)t + 1] = (uint64_t)(b1 - b0);
    }
    for (uint32_t t = 0; t < T; t++) sel_off[(size_t)t + 1] += sel_off[t];
    const uint64_t nsel = sel_off[T];
    std::vector<uint64_t> ids(nsel);
    std::vector<uint2> sel_fl(nsel);
#pragma omp parallel for schedule(dynamic, 256) num_threads(bm25x_host_threads(0))
    for (uint32_t t = 0; t < T; t++)
        for (uint64_t j = sel_off[t]; j < sel_off[(size_t)t + 1]; j++) {
            ids[j] = sel_b0[t] + (j - sel_off[t]);
            sel_fl[j] = first_last[ids[j]];
        }
    StagedBlocks st;
    st.gather(c, ids.data(), nsel);
    std::vector<uint64_t>().swap(ids);
    // ---- count: the shard's df, and each selected block's rank inside its token's shard list ----
    Scratch sc(device);
    sc.e = cudaSetDevice(device);
    const uint32_t *d_min = sc.up(st.min.data(), nsel), *d_n = sc.up(st.n.data(), nsel);
    const uint8_t *d_md = sc.up(st.md.data(), nsel), *d_mt = sc.up(st.mt.data(), nsel);
    const uint64_t *d_doff = sc.up(st.doff.data(), nsel), *d_toff = sc.up(st.toff.data(), nsel);
    const uint8_t *d_bytes = sc.up(st.bytes.data(), st.bytes.size());
    const uint2 *d_fl = sc.up(sel_fl.data(), nsel);
    const uint64_t *d_sel_off = sc.up(sel_off.data(), (size_t)T + 1);
    uint2 *d_cs = sc.alloc<uint2>(nsel);
    uint32_t h_err = 0, *d_err = sc.up(&h_err, 1);
    const unsigned grid = (unsigned)((nsel + DEC_WARPS - 1) / DEC_WARPS);
    if (sc.e == cudaSuccess && nsel) {
        k_count_shard_blocks<<<grid, DEC_WARPS * 32>>>(nsel, d_fl, d_min, d_n, d_md, d_doff, d_bytes, st.n_bytes, lo, hi,
                                                        d_cs, d_err);
        sc.e = cudaGetLastError();
    }
    std::vector<uint2> cs(nsel);
    if (sc.e == cudaSuccess && nsel) sc.e = cudaMemcpy(cs.data(), d_cs, sizeof(uint2) * nsel, cudaMemcpyDeviceToHost);
    if (sc.e != cudaSuccess) return cuda_refusal(who, "block upload/decode", sc.e);
    std::vector<uint32_t> df(T), rank(nsel);
    uint64_t Ps = 0;
    for (uint32_t t = 0; t < T; t++) {
        uint64_t run = 0;
        for (uint64_t j = sel_off[t]; j < sel_off[(size_t)t + 1]; j++) {
            rank[j] = (uint32_t)std::min<uint64_t>(run, 0xFFFFFFFFu);
            run += cs[j].x;
        }
        df[t] = (uint32_t)std::min<uint64_t>(run, hi - lo);  // more than the shard's documents: refused by the decode
        Ps += df[t];
    }
    // ---- allocate the shard as bm25x_sharded_create does (the term keys once, with shard 0) ----
    BuildMeta m{hi - lo, T, c->doc_len ? c->doc_len + lo : nullptr, c->payload ? c->payload + (size_t)lo * 3 : nullptr,
                s ? nullptr : c->term_key, c->k1, c->b, df.data(), Ps};
    m.fieldnorm = c->doc_len ? nullptr : c->doc_fieldnorm + lo;
    m.sum_len = c->sum_doc_len;  // stored norms: the pages hold the segment's sum only
    m.doc_base = lo;
    const int rc = index_begin(m, &stats, device, ix);
    if (rc != BM25X_OK) return rc;
    // ---- write the postings, then what every index derives from them ----
    const uint32_t *d_rank = sc.up(rank.data(), nsel);
    if (sc.e == cudaSuccess && nsel) {
        k_decode_shard_blocks<<<grid, DEC_WARPS * 32>>>(nsel, d_sel_off, T, d_min, d_n, d_md, d_mt, d_doff, d_toff, d_bytes,
                                                         st.n_bytes, d_cs, d_rank, c->n_docs, lo, hi - lo,
                                                         ix->d.post_off, ix->d.df, ix->d.fieldnorm, ix->d.post, d_err);
        sc.e = cudaGetLastError();
    }
    if (sc.e == cudaSuccess) sc.e = cudaMemcpy(&h_err, d_err, sizeof(h_err), cudaMemcpyDeviceToHost);
    if (sc.e == cudaSuccess && !h_err) sc.e = index_finish_device(ix.get());
    return sc.e != cudaSuccess ? cuda_refusal(who, "block upload/decode", sc.e) : blocks_refusal(h_err);
}

extern "C" int bm25x_index_create_sharded_from_blocks(const bm25x_blocks *c, uint32_t S, const uint32_t *doc_bounds,
                                                      const int *devices, bm25x_sharded_index **out) {
    const char *who = "bm25x_index_create_sharded_from_blocks";
    if (!c || !out) {
        bm25x_set_error("%s: null argument", who);
        return BM25X_ERR_INVALID;
    }
    *out = nullptr;
    // every host check before any device is used: the blocks exactly as bm25x_index_create_from_blocks checks them, then
    // the shard arguments exactly as bm25x_sharded_create checks them
    std::vector<uint32_t> df;
    uint64_t P = 0;
    int rc = validate_blocks(c, 0, false, df, P);
    if (rc != BM25X_OK) return rc;
    const uint32_t N = c->n_docs, T = c->n_terms;
    rc = check_shard_args(N, S, doc_bounds);
    if (rc != BM25X_OK) return rc;
    // the segment's norms (the stored ones, or quantised for the check pass) and statistics
    std::vector<uint8_t> h_fn(c->doc_len ? N : 0);
    const uint8_t *fn = c->doc_len ? h_fn.data() : c->doc_fieldnorm;
    const Stats st(N, doc_norms(N, c->doc_len, c->doc_fieldnorm, c->sum_doc_len, c->doc_len ? h_fn.data() : nullptr),
                   df.data(), T, c->k1, c->b);
    std::vector<uint2> first_last;
    // ---- check pass on shard 0's device: the refusals of the unsharded ingest, before any shard exists ----
    auto check = [&](int device, std::vector<uint64_t> *cum) {
        uint32_t h_err = 0;
        const int rc = check_stored_blocks(who, c, fn, st, device, first_last, cum, h_err);
        std::vector<uint8_t>().swap(h_fn);
        return rc != BM25X_OK ? rc : blocks_refusal(h_err);
    };
    // one shard at a time: host memory beyond the blocks stays within one shard's selected payload
    auto build = [&](uint32_t s, int device, uint32_t lo, uint32_t hi, IndexGuard &ix) {
        return build_shard_from_blocks(who, c, first_last, st, s, lo, hi, device, ix);
    };
    return sharded_build(who, c, P, df, st, S, doc_bounds, devices, check, build, out);
}
