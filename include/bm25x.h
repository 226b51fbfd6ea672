/*
 * bm25x.h — C ABI of the H100-native BM25 top-k engine (libbm25x.so).
 *
 * This is the drop-in boundary for ONE path of tensorchord/VectorChord-bm25: the
 * ranked top-k query `bm25::search` (and, next, `bm25::evaluate`).  Each entry
 * point cites the reference interface it replaces (paths relative to the
 * reference tree).  Plain pointers and sizes only: no C++/torch types, no
 * exceptions or unwinding across the boundary (the reference denies
 * ffi_unwind_calls, src/lib.rs:16): every call returns an int status and
 * bm25x_last_error() holds a thread-local message.
 *
 * There is NO CPU fallback: every search entry point fails with
 * BM25X_ERR_CUDA when no sm_90 device / kernel image is available.
 */
#ifndef BM25X_H
#define BM25X_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BM25X_OK 0
#define BM25X_ERR_INVALID 1     /* bad argument / corrupt corpus ("data corruption" panics in the reference) */
#define BM25X_ERR_CUDA 2        /* CUDA runtime / launch failure, or no usable device */
#define BM25X_ERR_OOM 3
#define BM25X_ERR_UNSUPPORTED 4 /* k > BM25X_MAX_K, > BM25X_MAX_QUERY_TERMS live terms, tf >= 2^24 */
#define BM25X_ERR_LIMIT_ZERO 5  /* k == 0: "number of needed rows is set to 0" (scanners/default.rs:114-116) */

#define BM25X_MAX_K 65535 /* the reference's bm25.limit maximum (src/index/gucs.rs:37-46) */
#define BM25X_MAX_QUERY_TERMS 64 /* live (known, distinct) tokens per query; more than 32 run as two passes over term groups */
#define BM25X_TERM_MISSING 0xFFFFFFFFu
#define BM25X_KEY_WIDTH 16 /* crates/bm25/src/lib.rs:37 WIDTH */

typedef struct bm25x_index bm25x_index;
typedef struct bm25x_batch bm25x_batch;

/* The sealed segment as the reference hands it to flush():
 * `Segment{records: Record(len, payload), mappings: Mapping(key, doc, tf)}` sorted by (key, doc)
 * (crates/bm25/src/segment.rs:19-45, flush.rs:40-67).  Term-major CSR on the host. */
typedef struct {
    uint32_t n_docs;          /* number_of_documents; doc id = record order (io.rs:52-60) */
    const uint32_t *doc_len;  /* [n_docs] exact document length = Σ tf (vector.rs:77-83) */
    const uint16_t *payload;  /* [n_docs*3] heap ctid of each record, or NULL (payload = doc id split) */
    uint32_t n_terms;         /* distinct tokens */
    const uint8_t *term_key;  /* [n_terms*16] interned keys, strictly ascending (vector.rs:19-35), or NULL when
                                 callers address terms by dense ordinal (the bm25vector u32-token-id surface) */
    const uint64_t *post_off; /* [n_terms+1] */
    const uint32_t *post_doc; /* [P] doc ids, strictly ascending inside a term */
    const uint32_t *post_tf;  /* [P] term frequencies, != 0 */
    double k1, b;             /* Bm25IndexOptions (crates/bm25/src/types.rs:18-45): defaults 1.2 / 0.75 */
} bm25x_corpus;

typedef struct {
    uint32_t n_docs, n_terms;
    uint64_t n_postings;
    uint64_t sum_doc_len;  /* JumpTuple.sum_of_document_lengths (tuples.rs:141-160) */
    double avgdl, k1, b;
    uint64_t device_bytes; /* HBM held by the index */
    uint64_t n_blocks;     /* 128-posting blocks (flush.rs:78-125) */
    int device;
} bm25x_index_info;

typedef struct {
    double kernel_ms;        /* device time of the search kernels, CUDA events on the launch stream */
    double h2d_ms, d2h_ms;   /* bm25x_search_batch only (host clock): canonicalise + upload, download of the results */
    uint64_t postings;       /* Σ df over live query terms (algorithmic postings touched, exhaustive) */
    uint64_t bytes_algo;     /* 8 B/posting + 8 B/result slot + 16 B/query term (SURVEY §8d) */
    uint32_t launches;       /* kernels launched */
    uint32_t queries;        /* live queries (>= 1 known term) */
    /* postings streamed into shared memory (pad slots excluded), plus the block-table entries and postings read by the
     * probes of pruned terms and of a two-pass query's other group, plus what is read again: the ring contents a
     * two-phase query re-reads when it resumes, and the rings re-split when terms are pruned.  With pruning and two-phase
     * off, it equals `postings` for queries of <= 32 live terms; with pruning on it can land on either side. */
    uint64_t postings_fetched;
} bm25x_search_stats;

/* ---- index lifetime: replaces bm25::build → flush (crates/bm25/src/build.rs:22-71, flush.rs:40-158) for the
 * read path: lays the postings out in HBM and precomputes per-term s0 and per-fieldnorm s1 (bm25.rs:334-354). */
int bm25x_index_create(const bm25x_corpus *corpus, int device, bm25x_index **out);
void bm25x_index_destroy(bm25x_index *idx);
int bm25x_index_get_info(const bm25x_index *idx, bm25x_index_info *out);

/* ---- the sealed segment AS STORED by the reference (SURVEY §8 f1: ingest of the on-page format).  While walking the
 * index pages the caller flattens, per token, the chain of SummaryTuples (crates/bm25/src/tuples.rs:900-910) and the
 * BlockTuples they point to (tuples.rs:973-983) that flush() wrote (flush.rs:78-120); the block payloads are taken
 * exactly as compression.rs:36-136 left them (4-lane vertical bit packing with delta-coded doc ids for full blocks,
 * byte packing for a token's last block) and are decoded on the GPU — replacing fill_block (search.rs:498-518) +
 * crates/simd/src/bitpacking*.rs / bytepacking*.rs on the CPU.  Searches on the resulting index are identical to those
 * on an index created from the same postings with bm25x_index_create. */
typedef struct {
    uint32_t n_docs;
    const uint32_t *doc_len;       /* [n_docs] exact lengths, or NULL: then the two fields below (what the pages hold) */
    const uint8_t *doc_fieldnorm;  /* [n_docs] DocumentTuple.fieldnorm (tuples.rs:756-762); used when doc_len == NULL */
    uint64_t sum_doc_len;          /* JumpTuple.sum_of_document_lengths (tuples.rs:141-160); used when doc_len == NULL */
    const uint16_t *payload;       /* [n_docs*3] DocumentTuple.payload (ctid), or NULL */
    uint32_t n_terms;
    const uint8_t *term_key;       /* [n_terms*16] TokenTuple.id, strictly ascending, or NULL */
    const uint64_t *term_blk_off;  /* [n_terms+1] first block of each token; term_blk_off[n_terms] == n_blocks */
    uint64_t n_blocks;
    const uint32_t *blk_min_doc;   /* [n_blocks] SummaryTuple.min_document_id: the delta seed of the block */
    const uint32_t *blk_n;         /* [n_blocks] SummaryTuple.number_of_documents: 128 except a token's last block */
    const uint8_t *blk_meta_doc;   /* [n_blocks] BlockTuple.metadata_document_ids: flag << 7 | width */
    const uint8_t *blk_meta_tf;    /* [n_blocks] BlockTuple.metadata_term_frequencies */
    const uint64_t *blk_doc_off;   /* [n_blocks] byte offset of compressed_document_ids inside `bytes` */
    const uint64_t *blk_tf_off;    /* [n_blocks] byte offset of compressed_term_frequencies inside `bytes` */
    const uint8_t *bytes;          /* concatenated block payloads */
    uint64_t n_bytes;
    double k1, b;
    /* SummaryTuple.wand_fieldnorm / wand_term_frequency (tuples.rs:900-910; written by flush.rs:101-120): the arg-max
     * posting of each block, whose score is the block's upper bound (search.rs:381,426-429).  Optional (both or
     * neither): when given they are checked against the decoded postings ("corrupt blocks" on mismatch); the bounds
     * the kernels use are always computed from the decoded postings themselves. */
    const uint8_t *blk_wand_fieldnorm; /* [n_blocks] or NULL */
    const uint32_t *blk_wand_tf;       /* [n_blocks] or NULL */
} bm25x_blocks;
int bm25x_index_create_from_blocks(const bm25x_blocks *blocks, int device, bm25x_index **out);

/* ---- the sealed segment from its DOCUMENTS: CREATE INDEX below the heap scan (ambuild → io::write → readers → build,
 * src/index/bm25/am/am_build.rs:312-313, crates/bm25/src/io.rs:187-244), the inversion run on the GPU.  Documents are
 * doc-major, in heap-scan order (doc id = position); each is a bm25vector Document: elements strictly ascending by key,
 * tf != 0 (vector.rs:38-83).  Exactly one of elem_key / elem_term is given.
 * The handle equals, array for array, the one bm25x_index_create builds from the reference's Segment of the same
 * documents: records in input order, doc_len[d] = the saturating Σ tf of document d (Document::length), postings sorted
 * by (key, doc); keyed: term_key = the distinct keys ascending bytewise (bm25x_lookup_terms, the export's term_key and the
 * seal's new_keys work on it); keyless: n_terms as given (ordinals without postings keep df 0) and no keys.
 * Refusals, every host one before any device is used (*out = NULL, no device memory left behind), named
 * bm25x_index_create_from_documents: BM25X_ERR_INVALID for a null argument, both or neither of elem_key / elem_term,
 * n_terms != 0 with keys, n_docs 0 or 0xFFFFFFFF, k1 / b out of range, elem_off[0] != 0, and naming the first offending
 * document: elem_off going backwards, keys or ordinals not strictly ascending inside a document, an ordinal >= n_terms
 * (BM25X_TERM_MISSING included), tf == 0; BM25X_ERR_UNSUPPORTED for tf >= 2^24.  Then the device check, and on the device,
 * before the index is allocated, more than 0xFFFFFFFE distinct keys (BM25X_ERR_UNSUPPORTED); BM25X_ERR_OOM /
 * BM25X_ERR_CUDA from the build steps.
 * The device works in chunks of 2^22 elements (DESIGN §4.9).  Device memory beyond the index: 12 B per term (per-term
 * cursors), per chunk 128 MiB keyless or 192 MiB keyed, CUB's temporary storage for one chunk's sort, and for a keyed
 * build the vocabulary: 16 B per distinct key while the postings are written; the
 * vocabulary pass before it holds up to 80 B per distinct key plus 80 B per element of one chunk (a list of (key, count)
 * with room to double, and the sort's second buffer). */
typedef struct {
    uint32_t n_docs;            /* records, in heap-scan order: doc id = position (io.rs:193, readers) */
    const uint64_t *elem_off;   /* [n_docs+1], elem_off[0] == 0, non-decreasing; E = elem_off[n_docs] may exceed 2^32 */
    const uint8_t *elem_key;    /* [E*16] Element.key, strictly ascending (bytewise) inside a document: keyed build; or NULL */
    const uint32_t *elem_term;  /* [E] term ordinal < n_terms, strictly ascending inside a document: keyless build; or NULL */
    const uint32_t *elem_tf;    /* [E] Element.value, != 0 */
    const uint16_t *payload;    /* [n_docs*3] Record payload (ctid), or NULL: the synthetic ctid, as bm25x_index_create */
    uint32_t n_terms;           /* keyless: the vocabulary size (ordinals without postings keep df 0); keyed: must be 0 */
    double k1, b;
} bm25x_documents;
int bm25x_index_create_from_documents(const bm25x_documents *docs, int device, bm25x_index **out);

/* ---- documents and queries as PostgreSQL tsvectors, the type every way into the reference takes (bm25_ops is FOR TYPE
 * tsvector, src/sql/finalize.sql:34-35): CREATE INDEX and aminsert cast each row with cast_tsvector_to_document, the
 * index scan casts its query with cast_tsvector_to_query (src/datatype/tsvector.rs:84-105).  A batch of n tsvectors as
 * the reference borrows them (TsVectorBorrowed, tsvector.rs:43-71; memory_tsvector.rs:30-51): vector i = its WordEntry
 * words entries[ent_off[i] .. ent_off[i+1]) and its lexeme area bytes[byte_off[i] .. byte_off[i+1]), exactly what follows
 * the datum's header.  Entry: bit 0 haspos, bits 1..11 len, bits 12..31 pos; the lexeme is area[pos .. pos+len), and with
 * haspos its count is the native-endian u16 at area[pos+len rounded up to even] (the number of positions).
 * Host refusals, all before any device is touched, BM25X_ERR_INVALID, the message naming the vector and the entry where
 * there is one (the reference panics in each): null arguments (entries / bytes may be NULL when there are none), ent_off[0]
 * or byte_off[0] != 0, offsets going backwards, a lexeme or a count running past its area, and in document mode an entry
 * without positions ("tsvector must have positions", tsvector.rs:88). */
typedef struct {
    uint32_t n;
    const uint64_t *ent_off;   /* [n+1], ent_off[0] == 0 */
    const uint32_t *entries;   /* WordEntry: bit 0 haspos, bits 1..11 len, bits 12..31 pos */
    const uint64_t *byte_off;  /* [n+1], byte_off[0] == 0 */
    const uint8_t *bytes;
} bm25x_tsvectors;
/* The cast alone, on `device`: cast_tsvector_to_document (as_query == 0) or cast_tsvector_to_query of every vector.  Row i
 * is out_off[i] .. out_off[i+1] of out_key ([.., 16] keys, ascending bytewise and distinct, vector::intern under seed) and,
 * in document mode, out_tf (the saturating sum of the merged counts; not written in query mode, may be NULL there).  A cast
 * never grows: size out_key and out_tf for ent_off[n] elements.  The output is bit for bit the restated casts over
 * bm25x_intern.  Refusals: the host ones above; then, after the device work and before any output is written, a document
 * element whose merged count is 0 (Document::new, vector.rs:51-64; BM25X_ERR_INVALID naming the vector).  The device works
 * on chunks of whole vectors (at most 2^22 entries, 64 MiB of lexeme area and 2^22 vectors, or one larger vector; a vector
 * of more than 2^31 - 1 entries is BM25X_ERR_UNSUPPORTED) and holds the cast until the end: 16 B (query) or 20 B
 * (document) per entry, 4 B per vector (8 more in document mode), and per chunk about 60 B per entry plus its area and
 * CUB's temporary storage. */
int bm25x_cast_tsvectors(const bm25x_tsvectors *tsv, const uint8_t seed[32], int as_query, int device,
                         uint64_t *out_off, uint8_t *out_key, uint32_t *out_tf);
/* CREATE INDEX from the tsvectors (am_build.rs:722): the index bm25x_index_create_from_documents builds from the keyed
 * documents the document cast gives, array for array; doc id = position (NULL rows are the caller's to leave out, as
 * ambuild does), payload as there.  The keys never travel to the host: the cast leaves a device-resident keyed CSR that
 * the build from documents reads chunk by chunk; only the row offsets and the document lengths come down (12 B per
 * document).  Refusals (*out = NULL, no device memory left behind): the cast's; check_common's on n_docs (0 or 0xFFFFFFFF),
 * k1 and b, on the host; on the device BM25X_ERR_UNSUPPORTED for a merged tf >= 2^24 (naming the first such document)
 * and for more than 0xFFFFFFFE distinct keys, as the build from documents refuses them; BM25X_ERR_OOM / BM25X_ERR_CUDA.
 * Device memory beyond the index: 20 B per tsvector entry (the cast, held through the build), one upload chunk of the cast
 * (freed before the build starts), and the build from documents' own figures. */
int bm25x_index_create_from_tsvectors(const bm25x_tsvectors *tsv, const uint8_t seed[32], const uint16_t *payload,
                                      double k1, double b, int device, bm25x_index **out);
/* Queries from tsvectors, ready for bm25x_search_batch, bm25x_search_candidates, bm25x_batch_prepare and the growing
 * segment's searches as they are: for each vector the query cast (cast_tsvector_to_query) and then address_tokens::read
 * (address_tokens.rs:61-98) on the index's device.  Row i = q_terms[q_off[i] .. q_off[i+1]) holds its distinct keys in
 * key order as term ordinals, BM25X_TERM_MISSING for a key the vocabulary lacks (the searches drop those,
 * search.rs:60-62).  Size q_terms for ent_off[n] terms.  The vocabulary goes to the device once per handle (16 B per term,
 * kept until bm25x_index_destroy).  Refusals: the host ones above (query mode), then an index without term keys (a
 * replica, a keyless build) with bm25x_lookup_terms' message, both before any device work; more than 2^32 - 1 output terms
 * (BM25X_ERR_UNSUPPORTED), before any output is written.  Thread-safe alongside the searches on the same handle.  Device
 * memory: 4 B per entry and 4 B per vector, held until the call returns, plus one upload chunk of the cast. */
int bm25x_tsvector_queries(bm25x_index *idx, const uint8_t seed[32], const bm25x_tsvectors *tsv, uint32_t *q_off,
                           uint32_t *q_terms);

/* ---- the inverse: a finalized index written out as the reference's stored segment, i.e. everything flush() writes for
 * it (flush.rs:40-158) but the pages, tapes and address trees, which stay the caller's.  Encoded on the index's device:
 * per token, blocks of 128 postings in doc order, the last one shorter (flush.rs:78-90; the index's own blocks); payloads
 * in the codec of compression.rs:36-110 (full blocks bit-packed in the 4-lane vertical layout, doc ids delta-coded from
 * the block's first id, width 32 raw; shorter blocks byte-packed, byte width 4 raw), per block the doc payload then the
 * tf payload, blocks in token order.  The directory and `bytes` feed bm25x_index_create_from_blocks as they are (the
 * doc_fieldnorm + sum_doc_len form: the handle keeps quantised norms, never exact lengths).
 * n_docs, n_terms, n_blocks: those bm25x_index_get_info reports.  Every output array is optional (NULL: not written).
 * bytes == NULL is a sizing call: it sets n_bytes and writes nothing else.  Refused with BM25X_ERR_INVALID: a null idx or
 * out; term_key on an index without term keys (a finalized replica, a seal of one); a replica not finalized yet; a
 * handle that scores with another segment's statistics, i.e. whose avgdl is not its Σlen / n_docs (bm25x_growing_create's
 * handles score with the sealed segment's: flush would write other Wand pairs for their documents); bytes_cap < n_bytes (n_bytes is set, nothing else is written).  Every refusal, and every device allocation
 * (BM25X_ERR_OOM), comes before the first output byte; after a later CUDA failure (BM25X_ERR_CUDA) the outputs are
 * unspecified.  The handle is not changed, and the export runs on a stream of its own: searches on the same handle may
 * run meanwhile.  Device memory beyond the index: about 35 bytes per block plus one payload chunk of at most 256 MiB. */
typedef struct {
    /* per document: DocumentTuple (tuples.rs:756-762) and JumpTuple (tuples.rs:141-160) */
    uint8_t *doc_fieldnorm;        /* [n_docs] DocumentTuple.fieldnorm, or NULL */
    uint16_t *payload;             /* [n_docs*3] DocumentTuple.payload: the stored ctid, the synthetic one when none was
                                      given; or NULL */
    uint64_t sum_doc_len;          /* out: JumpTuple.sum_of_document_lengths, the handle's Σlen */
    /* per token: TokenTuple (flush.rs:126-135) */
    uint8_t *term_key;             /* [n_terms*16] TokenTuple.id, or NULL; refused on an index without term keys */
    uint32_t *tok_df;              /* [n_terms] TokenTuple.number_of_documents, or NULL */
    uint8_t *tok_wand_fieldnorm;   /* [n_terms] TokenTuple.wand_fieldnorm: Wand::extend over the token's blocks in order
                                      (flush.rs:111-112, bm25.rs:319-325); 255 for a token without postings; or NULL */
    uint32_t *tok_wand_tf;         /* [n_terms] TokenTuple.wand_term_frequency; 0 for a token without postings; or NULL */
    uint64_t *term_blk_off;        /* [n_terms+1] first block of each token, or NULL */
    /* per block: SummaryTuple (flush.rs:113-120) + BlockTuple (flush.rs:91-100) */
    uint32_t *blk_min_doc;         /* [n_blocks] SummaryTuple.min_document_id: the block's first doc id, or NULL */
    uint32_t *blk_max_doc;         /* [n_blocks] SummaryTuple.max_document_id: its last, or NULL */
    uint32_t *blk_n;               /* [n_blocks] SummaryTuple.number_of_documents, or NULL */
    uint8_t *blk_meta_doc;         /* [n_blocks] BlockTuple.metadata_document_ids: flag << 7 | width, or NULL */
    uint8_t *blk_meta_tf;          /* [n_blocks] BlockTuple.metadata_term_frequencies, or NULL */
    uint64_t *blk_doc_off;         /* [n_blocks] byte offset of compressed_document_ids inside `bytes`, or NULL */
    uint64_t *blk_tf_off;          /* [n_blocks] byte offset of compressed_term_frequencies inside `bytes`, or NULL */
    uint8_t *blk_wand_fieldnorm;   /* [n_blocks] SummaryTuple.wand_fieldnorm: Wand over the block's postings in doc order
                                      (bm25.rs:297-318), the first posting of the largest tf() (bm25.rs:291-295); or NULL */
    uint32_t *blk_wand_tf;         /* [n_blocks] SummaryTuple.wand_term_frequency, or NULL */
    uint8_t *bytes;                /* [bytes_cap] the concatenated block payloads, or NULL: a sizing call */
    uint64_t bytes_cap;
    uint64_t n_bytes;              /* out: the payload size, set by every call that gets past the argument checks */
} bm25x_export;
int bm25x_index_export_blocks(const bm25x_index *idx, bm25x_export *out);

/* ---- replication across the GPUs of one box (queries shard, the index is replicated; NCCL broadcast at load
 * only).  The library stays NCCL-free: it exposes the device arrays, the caller moves the bytes (bench.py uses
 * torch.distributed.broadcast over NVLink).  Sender: bm25x_index_get_layout.  Receiver: bm25x_index_alloc_replica
 * with the sender's layout (scalars only are read), fill the arrays named by its own layout, then
 * bm25x_index_finalize_replica. */
#define BM25X_N_ARRAYS 13
typedef struct {
    uint32_t n_docs, n_terms;
    uint64_t n_postings, n_postings_padded, n_blocks, sum_doc_len;
    double k1, b, avgdl;
    void *dev_ptr[BM25X_N_ARRAYS];     /* device addresses of the index arrays (valid on `device` only) */
    uint64_t bytes[BM25X_N_ARRAYS];
    int device;
} bm25x_index_layout;
int bm25x_index_get_layout(const bm25x_index *idx, bm25x_index_layout *out);
int bm25x_index_alloc_replica(const bm25x_index_layout *like, int device, bm25x_index **out);
/* Rebuilds the derived structures below from the arrays as they are now; may be called again after a refill. */
int bm25x_index_finalize_replica(bm25x_index *idx);
/* Test hook: the derived structures every index builds on its own device and never replicates (finalize_replica rebuilds
 * them), so that tests can read them back and compare them with a CPU restatement.  Device addresses, valid on `device`
 * until the handle is destroyed or finalized again; a replica that is not finalized yet has no champion lists (NULL, 0). */
typedef struct {
    void *pdoc;                /* [n_postings_padded + 4] u32: post[i].doc; pad and slack slots read 0xFFFFFFFF */
    uint64_t pdoc_bytes;
    void *champ;               /* [n_champ] {u32 doc, u32 tf << 8 | fieldnorm}: per term its best min(df, 128) postings,
                                  exact single-term score descending, then doc id ascending */
    uint64_t champ_bytes;
    void *champ_off;           /* [n_terms + 1] u64: term t's list is champ[champ_off[t] .. champ_off[t + 1]) */
    uint64_t champ_off_bytes;
    uint64_t n_champ;
    float s1f_min;             /* min over the documents d of (float) s1[fieldnorm(d)] */
    int device;
} bm25x_index_derived;
int bm25x_index_get_derived(const bm25x_index *idx, bm25x_index_derived *out);
/* Options.  "prune" (default 1): MaxScore-style pruning in the warp-per-query kernel — terms whose summed score upper
 * bounds (the token-level WAND bound of the reference: TokenTuple.wand_fieldnorm/wand_term_frequency,
 * flush.rs:101-120, search.rs:363) stay at or below half the current k-th score are no longer streamed; their postings
 * are looked up in HBM only for the candidates.  Results are identical with it on or off.
 * "seed" (default 1): queries of 2..8 terms with limit <= 128 and no prefilter bitmap run through the SEEDED kernel —
 * the documents that hold a single query term come from per-term champion lists (the term's best 128 postings in
 * result order, built with the index), so the stream reads doc ids only (half the bytes) and never tests a posting on
 * its own; "seed_max_terms" (4 | 8), "seed_dense_div" (default 64: queries with a list of >= n_docs / 64 postings go
 * back to the plain kernel; 0: never), "seed_prune_min" (default 32768: so do queries with a list this long and 8x
 * their shortest one — pruning pays).  "twophase" (default 0): queries of 2..4 terms with limit <= 224 that the seeded
 * kernel does not take run as two launches — 8-byte postings while single postings can still enter the top-k, then
 * doc ids only.  "slice_min" (default 32768): bm25x_search_batch pipelines batches of >= 2 x this many queries as slices
 * (upload / kernels / download overlap; 0: one piece).  None of these changes a result bit. */
int bm25x_index_set_option(bm25x_index *idx, const char *name, int64_t value);
/* df of every term (TokenTuple.number_of_documents), host copy. */
int bm25x_index_get_df(const bm25x_index *idx, uint32_t *df_out);

/* address_tokens::read (crates/bm25/src/address_tokens.rs:61-98): key → dense term ordinal,
 * BM25X_TERM_MISSING when absent (search.rs:60-62 then skips it).  Needs term_key at create time. */
int bm25x_lookup_terms(const bm25x_index *idx, const uint8_t *keys, uint32_t n, uint32_t *ordinals_out);

/* vector::intern (crates/bm25/src/vector.rs:19-35): the 16-byte key of a token under the index's 32-byte seed.  Tokens
 * shorter than 16 bytes without a NUL byte are their own zero-padded key; all others are the first 16 bytes of
 * blake3::keyed_hash(seed, token) with a zero last byte replaced by 1.  Host-only (no device involved); the tsvector
 * casts below intern whole batches on the device, bit for bit the same. */
int bm25x_intern(const uint8_t seed[32], const uint8_t *token, size_t len, uint8_t key_out[BM25X_KEY_WIDTH]);
/* Test hook: first 16 bytes of BLAKE3 keyed_hash(key, data) without the interning rules (known-answer tests). */
int bm25x_blake3_keyed16(const uint8_t key[32], const uint8_t *data, size_t len, uint8_t out[16]);

/* ---- bm25::search (crates/bm25/src/search.rs:28-282) for a whole batch of queries, called where
 * DefaultBuilder::build calls it (src/index/bm25/scanners/default.rs:117-129).
 *   q_off[nq+1], q_terms[]: query i = term ordinals q_terms[q_off[i]..q_off[i+1]) — any order, duplicates and
 *     BM25X_TERM_MISSING / df==0 terms allowed (they are dropped exactly as search.rs:55-62 drops them).
 *   k: `limit` (NonZero<usize>, 1..=BM25X_MAX_K).
 *   allow: optional prefilter bitmap [ceil(n_docs/8)], bit d set ⇒ filter(payload(d)) is true
 *     (search.rs:230; the per-candidate callback of the reference cannot cross a batch ABI); NULL ⇒ all pass.
 *   outputs, row i at offset i*k, best first (score desc, then doc id asc — the canonical tie rule):
 *     out_doc u32, out_score f32 (positive; the SQL binding negates, operators.rs:54),
 *     out_score64 f64 or NULL (bit-identical to Cache::evaluate summed in ascending term order),
 *     out_payload u16[3] or NULL, out_n[i] = rows returned (<= k).
 * Host pointers; the call copies H2D, runs the sm_90a kernels, copies D2H. */
int bm25x_search_batch(bm25x_index *idx, uint32_t nq, const uint32_t *q_off, const uint32_t *q_terms, uint32_t k,
                       const uint8_t *allow, uint32_t *out_doc, float *out_score, double *out_score64,
                       uint16_t *out_payload, uint32_t *out_n, bm25x_search_stats *stats);

/* ---- Per-query candidate lists: each query's top-k over its own doc ids.  The reference's bm25::search
 * (crates/bm25/src/search.rs:28-36) takes one filter per index scan, and every scan has its own WHERE clause and
 * bm25.prefilter (src/index/fetcher.rs:181-215); here every query of the batch carries its own candidate list (a filter's
 * qualifying rows, or the ids an ANN search returned for hybrid retrieval).
 *   q_off, q_terms, k: as bm25x_search_batch (up to BM25X_MAX_QUERY_TERMS live terms).
 *   c_off[nq+1], c_docs[]: query i's candidates are c_docs[c_off[i]..c_off[i+1]): doc ids in any order, duplicates
 *     allowed (counted once), possibly none.
 *   outputs: row i is bit for bit the row bm25x_search_batch returns for query i alone with `allow` = the bitmap of its
 *     candidates: the candidates that hold a live query term, score desc then doc id asc, out_n[i] <= k, empty slots doc
 *     0xFFFFFFFF with zeros elsewhere.  With k >= |C_i| the row holds every matching candidate with its score.
 * Refusals, all before any device work (a refused call writes no output): those of bm25x_search_batch with its codes and
 * messages (null arguments, k == 0, k > BM25X_MAX_K, q_off not monotone, > 64 live terms, replica not finalized); c_off
 * not monotone and a candidate >= n_docs (BM25X_ERR_INVALID, the message names the query, the entry and the id); more
 * than 2^31 - 1 candidates of live queries, or more than 2^31 - 1 queries, in one call (BM25X_ERR_UNSUPPORTED).
 * Thread-safe on one handle, alongside the other searches.  The device sorts every query's candidates by doc id (CUB
 * segmented sort), looks every (candidate, live term) pair up in the term's block table and then inside its 128-posting
 * block, and sorts the scores per query (DESIGN §4.8).  Device memory beyond the rows: 24 B per candidate of a live query
 * (4 B uploaded, 4 B for the sort's second doc-id buffer, 2 x 8 B of sort keys), 8 B per query and 4 B per live query
 * term uploaded, plus CUB's temporary storage for the two segmented sorts.  Host memory: the upload goes through the
 * handle's page-locked staging buffer, which bm25x_search_batch shares; it grows to 1.25x the largest upload the handle
 * has made (about 4 B per candidate plus 8 B per query) and is kept until bm25x_index_destroy, so that repeated calls
 * of that size do not pay a page-locked allocation each time.
 * stats: queries = live queries; kernel_ms = device events around the sorts and kernels; launches = 4 when any live
 * query has a candidate (two segmented sorts counted once each, the lookups, the rows), else 0; h2d_ms, d2h_ms as for
 * bm25x_search_batch; postings = Σ df of the live terms, as elsewhere (no list is streamed here); postings_fetched =
 * block-table entries plus postings the lookups read; bytes_algo = 8 B per (candidate, live term) lookup + 8 B per
 * result slot + 16 B per query term. */
int bm25x_search_candidates(bm25x_index *idx, uint32_t nq, const uint32_t *q_off, const uint32_t *q_terms,
                            const uint32_t *c_off, const uint32_t *c_docs, uint32_t k, uint32_t *out_doc, float *out_score,
                            double *out_score64, uint16_t *out_payload, uint32_t *out_n, bm25x_search_stats *stats);

/* Split form of the same call, for pipelining and for timing the device part alone:
 * prepare = canonicalise + upload queries; run = kernels only, everything resident in HBM
 * (stream = cudaStream_t as void*, NULL = the library's stream; asynchronous unless stats != NULL);
 * fetch = D2H of the results, on the stream of the last run.
 * A batch may be run any number of times: every run rewrites every result row of its live queries.  Runs of different
 * batches may overlap on different streams.  The only wait run adds is for the batch's upload by prepare; ordering the
 * runs of ONE batch on different streams (and reads of bm25x_batch_device_results after a run) is the caller's job,
 * e.g. an event recorded on the earlier run's stream and waited on by the later one. */
int bm25x_batch_prepare(bm25x_index *idx, uint32_t nq, const uint32_t *q_off, const uint32_t *q_terms, uint32_t k,
                        const uint8_t *allow, bm25x_batch **out);
int bm25x_batch_run(bm25x_batch *batch, void *stream, bm25x_search_stats *stats);
int bm25x_batch_fetch(bm25x_batch *batch, uint32_t *out_doc, float *out_score, double *out_score64,
                      uint16_t *out_payload, uint32_t *out_n);
/* Device addresses of the batch's result rows ([nq*k] u32 / f32 / f64 / u16[3], [nq] u32; any pointer may be NULL),
 * written by bm25x_batch_run on its stream and valid until bm25x_batch_destroy — for callers that move results
 * GPU → GPU (the NCCL gather of sharded results to one rank, vectorchord-bm25_b200/shard.py) instead of fetching. */
int bm25x_batch_device_results(bm25x_batch *batch, void **doc, void **score, void **score64, void **payload, void **n);
void bm25x_batch_destroy(bm25x_batch *batch);

/* ---- the growing segment (SURVEY §8 f3): documents inserted since the last seal.  bm25::search scans them one by one
 * before it walks the sealed postings (crates/bm25/src/search.rs:83-135): every non-deleted growing document is scored
 * over the query tokens that exist in the SEALED segment with the sealed statistics — Cache::new(sealed N, sealed df,
 * k1, b, sealed avgdl) (search.rs:49-51,66-77; `insert` does not update them) — and shares the Results heap with the
 * sealed documents.  Here the growing documents are inverted once into a second, small index handle that carries
 * the sealed statistics, so the same kernels unite their postings; a query then is two top-k searches + a merge.
 * Doc ids of the growing handle are growing ordinals (insertion order).  The handle is immutable: a segment that takes
 * inserts and deletes in place is bm25x_growing_segment below; `maintain`/seal = bm25x_growing_seal on that segment. */
typedef struct {
    uint32_t n_docs;               /* growing documents, in VectorTuple-chain order */
    const uint32_t *doc_len;       /* [n_docs] exact lengths, or NULL: then doc_fieldnorm */
    const uint8_t *doc_fieldnorm;  /* [n_docs] VectorTuple fieldnorm (search.rs:96-98); used when doc_len == NULL */
    const uint16_t *payload;       /* [n_docs*3] VectorTuple.payload (ctid), or NULL */
    const uint8_t *deleted;        /* [n_docs] VectorTuple.deleted (search.rs:110): non-zero = skipped; or NULL */
    const uint64_t *elem_off;      /* [n_docs+1] */
    const uint32_t *elem_term;     /* Element.key as term ordinal of the SEALED index (bm25x_lookup_terms), strictly
                                      ascending inside a document; BM25X_TERM_MISSING = token unknown to the sealed
                                      segment: it can never match a query token (search.rs:60-62) */
    const uint32_t *elem_tf;       /* Element.value, != 0 */
} bm25x_growing_docs;
int bm25x_growing_create(const bm25x_index *sealed, const bm25x_growing_docs *docs, bm25x_index **out);
/* bm25::search over sealed + growing: bm25x_search_batch on both handles and the merge below.  `growing` may be NULL
 * (sealed only).  Doc ids >= n_docs(sealed) denote growing ordinal (id - n_docs(sealed)); on equal scores sealed
 * documents come first, then ascending id (the reference's order of equal scores is not pinned, see bm25x_search_batch).
 * allow_growing: optional prefilter bitmap over growing ordinals.  Both lists are merged on the device
 * (k_merge_shards): stats are those of bm25x_sharded_search_batch (sums over both handles plus the merge launch, so
 * `launches` and `kernel_ms` include the merge), except `queries` = the sealed search's live queries. */
int bm25x_search_batch_growing(bm25x_index *sealed, bm25x_index *growing, uint32_t nq, const uint32_t *q_off,
                               const uint32_t *q_terms, uint32_t k, const uint8_t *allow_sealed,
                               const uint8_t *allow_growing, uint32_t *out_doc, float *out_score, double *out_score64,
                               uint16_t *out_payload, uint32_t *out_n, bm25x_search_stats *stats);
/* Host-only: row-wise merge of two top-k result sets (score desc; equal scores: list a first, then ascending id);
 * ids of list b are shifted by doc_base_b.  f64 scores of both lists are required; f32 scores / payloads optional. */
int bm25x_merge_topk(uint32_t nq, uint32_t k, const uint32_t *doc_a, const float *score_a, const double *score64_a,
                     const uint16_t *payload_a, const uint32_t *n_a, const uint32_t *doc_b, const float *score_b,
                     const double *score64_b, const uint16_t *payload_b, const uint32_t *n_b, uint32_t doc_base_b,
                     uint32_t *out_doc, float *out_score, double *out_score64, uint16_t *out_payload, uint32_t *out_n);

/* ---- the mutable growing segment: the documents inserted since the last seal, owned by the library and indexed on the
 * sealed index's device.  bm25x_growing_insert appends documents (`insert`, crates/bm25/src/insert.rs) and
 * bm25x_growing_delete sets their deleted flag (`bulkdelete`, bulkdelete.rs); both cost host work in proportion to what
 * they change.  A refresh brings the segment's index handle up to date on the device: the surviving postings of the
 * current handle and the inserted ones are spliced into a new handle built beside it, which then replaces it.  A search
 * over sealed + growing is one call (both handles' kernels, one device merge, one download) and refreshes first when
 * anything is pending.  Every call may come from any thread: a search sees one state of the segment, with every insert
 * and delete that returned before it started and never part of one; a handle a running search still holds is destroyed
 * when that search ends.  The sealed index must outlive the segment, or the rebind to its successor
 * (bm25x_growing_rebind). */
typedef struct bm25x_growing_segment bm25x_growing_segment;
typedef struct {
    uint32_t n_docs;        /* ordinals handed out (deleted ones included) */
    uint32_t n_deleted;
    uint64_t n_postings;    /* postings in the segment's handle (as of the last refresh) */
    uint64_t device_bytes;  /* HBM held by the segment's handle */
    uint32_t pending;       /* 1: inserts or deletes since the last refresh */
    int device;             /* the sealed index's */
} bm25x_growing_info;
/* An empty segment on the sealed index's device, scoring with its statistics.  Any finalized handle serves; a finalized
 * replica holds no term keys (they do not travel with the 13 arrays), so a keyed index's replica seals as a keyless one:
 * stable ordinals, new_keys refused. */
int bm25x_growing_open(bm25x_index *sealed, bm25x_growing_segment **out);
/* Appends docs as ordinals n_docs .. n_docs + docs->n_docs - 1 (deleted flags included).  Refuses what
 * bm25x_growing_create refuses, with its codes and messages (terms not ascending, tf = 0, tf >= 2^24, sealed n_docs +
 * growing n_docs above 2^32 - 2), and documents in the other norm form than the segment's first insert (doc_len vs
 * doc_fieldnorm, BM25X_ERR_INVALID).  A refused insert changes nothing.  Without a payload a document gets the synthetic
 * ctid of its ordinal, as bm25x_growing_create gives it. */
int bm25x_growing_insert(bm25x_growing_segment *g, const bm25x_growing_docs *docs);
/* Marks ordinals deleted (bulkdelete).  An ordinal >= n_docs is refused (BM25X_ERR_INVALID, naming the first one) and
 * nothing is applied; deleting a deleted ordinal is a no-op.  Sealed documents are filtered with allow_sealed. */
int bm25x_growing_delete(bm25x_growing_segment *g, uint32_t n, const uint32_t *ordinals);
/* Brings the handle up to date (a no-op when nothing is pending).  Optional: the search refreshes too.  Its arrays are
 * those bm25x_growing_create builds over all documents inserted so far with their deleted flags. */
int bm25x_growing_refresh(bm25x_growing_segment *g);
int bm25x_growing_get_info(const bm25x_growing_segment *g, bm25x_growing_info *out);
/* The contract, refusals and rows of bm25x_search_batch_growing on a handle bm25x_growing_create builds from the
 * segment's documents: sealed ids as they are, growing ordinal o as n_docs(sealed) + o; score desc, on equal scores
 * sealed first, then ascending id.  allow_growing covers ordinals [0, allow_growing_docs): ordinals at or past it are
 * filtered out (NULL = all pass).  A pending refresh runs first and counts in h2d_ms.  stats: sums over both
 * searches plus the merge launch (queries included); before the first insert, the call is bm25x_search_batch on the
 * sealed index, stats included. */
int bm25x_growing_search_batch(bm25x_growing_segment *g, uint32_t nq, const uint32_t *q_off, const uint32_t *q_terms,
                               uint32_t k, const uint8_t *allow_sealed, const uint8_t *allow_growing,
                               uint32_t allow_growing_docs, uint32_t *out_doc, float *out_score, double *out_score64,
                               uint16_t *out_payload, uint32_t *out_n, bm25x_search_stats *stats);
/* bm25x_search_candidates over the segment: candidate ids in the result id space (sealed ids below n_docs(sealed),
 * growing ordinal o as n_docs(sealed) + o); a candidate at or past n_docs(sealed) + n_docs(segment) is refused
 * (BM25X_ERR_INVALID).  A pending refresh runs first; deleted ordinals are never returned.  Every list (the sealed side's
 * and the growing handle's) runs the candidate search at k over the candidates in its id range, and the lists are merged
 * on the device as in bm25x_growing_search_batch, whose refusals, stats and behaviour before the first insert apply
 * (with bm25x_search_candidates in place of bm25x_search_batch). */
int bm25x_growing_search_candidates(bm25x_growing_segment *g, uint32_t nq, const uint32_t *q_off,
                                    const uint32_t *q_terms, const uint32_t *c_off, const uint32_t *c_docs, uint32_t k,
                                    uint32_t *out_doc, float *out_score, double *out_score64, uint16_t *out_payload,
                                    uint32_t *out_n, bm25x_search_stats *stats);
/* Test hook: the arrays of the segment's current handle, as bm25x_sharded_get_shard reports a shard's (either output may
 * be NULL); valid until the next refresh or close.  Refused before the first refresh of a non-empty segment. */
int bm25x_growing_get_index(const bm25x_growing_segment *g, bm25x_index_layout *layout, bm25x_index_derived *derived);
void bm25x_growing_close(bm25x_growing_segment *g);
/* aminsert of tsvectors (src/index/bm25/am/mod.rs:261-287: cast_tsvector_to_document, then bm25::insert): vector i
 * becomes ordinal n_docs + i.  The call equals bm25x_growing_insert of the restated rows: the document cast of each vector
 * (bm25x_cast_tsvectors); each key as the ordinal of the sealed vocabulary (bm25x_lookup_terms, df 0 terms included), else
 * the ordinal an earlier insert numbered it with, else a fresh one: n_terms(sealed) + K + r, K = the keys the segment held
 * before the call, r = the key's rank among the call's fresh keys ascending bytewise; each row ascending by ordinal with
 * the merged counts as tf; the norm in the segment's form (doc_len = the saturating Σ tf, or in doc_fieldnorm form
 * length_to_fieldnorm of it); payload as given (NULL: the synthetic ctid of the ordinal); no deleted flags.
 * From its first successful call on the segment OWNS its keys: bm25x_growing_insert refuses an ordinal >= n_terms(sealed)
 * other than BM25X_TERM_MISSING (BM25X_ERR_INVALID, naming the document and the ordinal), and the seal takes the
 * segment's keys as new_keys (args->new_keys must be NULL and n_new_keys 0, else BM25X_ERR_INVALID; n_source_terms =
 * n_terms(sealed) + K).  Refusals, before any device work: null arguments; the tsvectors' host refusals (document mode);
 * a sealed side without term keys (bm25x_lookup_terms' message); a segment that took ordinals >= n_terms(sealed) from
 * bm25x_growing_insert (BM25X_ERR_INVALID: its numbering is the caller's).  After the cast: a merged count of 0; more
 * than 2^31 - 1 elements or tsvectors in one call (BM25X_ERR_UNSUPPORTED); then everything bm25x_growing_insert refuses
 * for the restated rows, with its codes and messages.  A refused call changes nothing and leaves no device memory behind.
 * Concurrency: tsvector inserts are serialised with each other (fresh keys are numbered in commit order), and hold the
 * segment's lock only for the host insert and the key commit, so searches do not wait on their device work.  Device
 * memory on the segment's device, held until the call returns: the document cast's figures (bm25x_cast_tsvectors),
 * 32 B per element whose key the sealed vocabulary lacks (compacted, sort buffer), 4 B per distinct such key, 16 B per
 * element for the re-sort by ordinal, and CUB's temporary storage; the sealed vocabulary, 16 B per sealed term, once per
 * index (bm25x_tsvector_queries' copy) or, over a document-sharded index, once per segment until bm25x_growing_close.
 * Host: 16 B per owned key plus a hash table entry, until close. */
int bm25x_growing_insert_tsvectors(bm25x_growing_segment *g, const uint8_t seed[32], const bm25x_tsvectors *tsv,
                                   const uint16_t *payload);
/* The keys the segment numbered: *n_out = K and key i (of ordinal n_terms(sealed) + i) at keys_out + 16 i.  cap < K is
 * refused (BM25X_ERR_INVALID) with *n_out set and nothing written.  K = 0 for a segment without tsvector inserts. */
int bm25x_growing_get_new_keys(const bm25x_growing_segment *g, uint32_t cap, uint8_t *keys_out, uint32_t *n_out);
/* Queries from tsvectors for the segment's searches: bm25x_tsvector_queries over the sealed side (an index: equal to
 * that call on it; a document-sharded index: the query cast plus bm25x_sharded_lookup_terms), with its refusals, named by
 * this call.  Keys the segment numbered are BM25X_TERM_MISSING: before the seal they never match (search.rs:60-62).
 * Thread-safe alongside inserts and searches. */
int bm25x_growing_tsvector_queries(bm25x_growing_segment *g, const uint8_t seed[32], const bm25x_tsvectors *tsv,
                                   uint32_t *q_off, uint32_t *q_terms);

/* ---- the seal (`maintain`, crates/bm25/src/maintain.rs:27-311, called from amvacuumcleanup): a NEW sealed index on the
 * sealed index's device from the sealed documents not marked deleted (ascending old id, relabelled densely) followed by
 * the segment's surviving documents (ascending ordinal), with fresh statistics (N, Σlen, df, blocks, bounds).  Every
 * document keeps its stored payload (the synthetic ctid of its OLD id / ordinal when none was given).  Lengths: a
 * sealed survivor's is the number of postings it holds in the sealed segment (add_element adds 1 per posting,
 * maintain.rs:356-360), a growing survivor's its doc_len, or in doc_fieldnorm form the saturating Σ tf over all its
 * elements, BM25X_TERM_MISSING ones included (Document::length, vector.rs:77-83).  Vocabulary: an inserted ordinal >=
 * n_terms(sealed) becomes a term, BM25X_TERM_MISSING never does.  Keyless index: ordinals are stable, the new n_terms
 * = max(n_terms(sealed), 1 + the largest ordinal inserted), a term without surviving posting stays with df 0.  Keyed
 * index: ordinal n_terms(sealed) + i has key new_keys[i]; the new terms are the keys with df > 0, ascending.  The
 * segment takes its state (refreshing first) under its lock and builds outside it: inserts, deletes and searches go on
 * meanwhile and the seal covers exactly ordinals [0, n_growing).  The sealed index and the segment are not changed; the
 * new index has bm25x_index_create's option defaults.  Refusals (nothing changes, *out = NULL): null arguments; no
 * surviving document (BM25X_ERR_INVALID); new_keys on a keyless index; a new key equal to a sealed or another new key;
 * on a keyed index an inserted ordinal >= n_terms(sealed) + n_new_keys (the first one is named); a non-NULL map whose
 * cap is below what the seal writes (n_growing and n_source_terms are set for a retry); a surviving posting with
 * tf >= 2^24 (BM25X_ERR_UNSUPPORTED); BM25X_ERR_OOM when the new index does not fit. */
typedef struct {
    const uint8_t *sealed_deleted; /* in: [ceil(n_docs(sealed)/8)] bit d set = sealed document d is deleted
                                      (DocumentTuple.deleted, bulkdelete.rs), the bit layout of `allow`; NULL = none */
    const uint8_t *new_keys;       /* in, keyed sealed index only: [n_new_keys*16] key of token ordinal n_terms(sealed)+i */
    uint32_t n_new_keys;
    uint32_t *sealed_map;          /* out [n_docs(sealed)]: new doc id, or 0xFFFFFFFF if deleted; or NULL */
    uint32_t *growing_map;         /* out [growing_cap]: new doc id of growing ordinal o < n_growing, or 0xFFFFFFFF; or NULL */
    uint32_t growing_cap;
    uint32_t *term_map;            /* out [term_cap]: new ordinal of source term t < n_source_terms, or BM25X_TERM_MISSING;
                                      or NULL */
    uint32_t term_cap;
    uint32_t n_growing;            /* out: ordinals [0, n_growing) were folded in */
    uint32_t n_source_terms;       /* out: keyless: the new n_terms; keyed: n_terms(sealed) + n_new_keys */
} bm25x_seal_args;
int bm25x_growing_seal(bm25x_growing_segment *g, bm25x_seal_args *args, bm25x_index **out);

/* ---- document-sharded index: one sealed segment split by document range over one or more GPUs, so that its postings
 * need not fit in one GPU's HBM.  Every shard scores with the WHOLE segment's statistics (N, avgdl, df), so its top-k is
 * the whole index's ranking restricted to its documents; the shards' lists are merged on shard 0's device
 * (k_merge_shards).  Results are bit-identical to bm25x_search_batch on an index created from the same corpus.  The
 * shard handles stay internal: their df and N are not the segment's. */
#define BM25X_MAX_SHARDS 16
typedef struct bm25x_sharded_index bm25x_sharded_index;
/* `whole` exactly as for bm25x_index_create.  doc_bounds[n_shards+1]: shard s holds the documents
 * [doc_bounds[s], doc_bounds[s+1]), strictly ascending, doc_bounds[0] = 0, doc_bounds[n_shards] = n_docs; NULL = balanced
 * by postings: b_s (0 < s < S) is the smallest d > b_{s-1} with Σ_{d' < d} c_{d'} >= ceil(s·P/S), c_d = distinct terms of
 * document d, clamped so that every shard keeps at least one document.  devices[n_shards], or NULL = all on device 0; one
 * device may hold several shards.  The shards are built one after the other (host memory beyond `whole`: one shard's
 * CSR). */
int bm25x_sharded_create(const bm25x_corpus *whole, uint32_t n_shards, const uint32_t *doc_bounds, const int *devices,
                         bm25x_sharded_index **out);
/* The same document-sharded index, built from the sealed segment AS STORED (`blocks` exactly as for
 * bm25x_index_create_from_blocks: SummaryTuple chains and BlockTuple payloads, tuples.rs:900-910,973-983, in the codec of
 * compression.rs:36-136).  No CSR of the segment is ever built on the host: a check pass on devices[0] decodes every stored
 * block once, in bounded chunks, with every check bm25x_index_create_from_blocks makes (the same codes and messages, the
 * wand pair included), then each shard's device receives and decodes only the stored blocks that hold its documents.
 * n_shards, doc_bounds and devices mean what they mean for bm25x_sharded_create (its refusals, its messages); with
 * doc_bounds == NULL the bounds are its balanced ones, c_d counted from the decoded postings.  With doc_len the shards'
 * arrays equal those bm25x_sharded_create builds from the decoded corpus; with doc_fieldnorm + sum_doc_len they hold the
 * stored norms, and each shard's own sum_doc_len is the segment's.  Every host check runs before any device is used; on
 * a refusal no handle is returned and every device allocation is freed.  The handle is an ordinary
 * bm25x_sharded_index. */
int bm25x_index_create_sharded_from_blocks(const bm25x_blocks *blocks, uint32_t n_shards, const uint32_t *doc_bounds,
                                           const int *devices, bm25x_sharded_index **out);
/* The same document-sharded index, built from the documents (`docs` exactly as for bm25x_index_create_from_documents):
 * equal to bm25x_sharded_create on that call's CSR with the same n_shards / doc_bounds / devices.  With doc_bounds == NULL
 * the bounds are its balanced ones with c_d = the elements of document d (cum[d] = elem_off[d]).  Keyed: the vocabulary
 * pass runs on devices[0] over every element, and the keys go with shard 0.  Then every shard's device counts its own df
 * over its element range (the host sums them into the segment's df and statistics), and each shard inverts only
 * [elem_off[lo], elem_off[hi]) with local doc ids.  Refusals: those of bm25x_index_create_from_documents (its codes and
 * messages), then the shard arguments and devices with bm25x_sharded_create's messages, all before any device is used.
 * Device memory per device beyond its shards: as bm25x_index_create_from_documents, for its own shards' documents. */
int bm25x_index_create_sharded_from_documents(const bm25x_documents *docs, uint32_t n_shards, const uint32_t *doc_bounds,
                                              const int *devices, bm25x_sharded_index **out);
/* The same document-sharded index, built from tsvectors (CREATE INDEX, am_build.rs:722, over a segment too large for one
 * GPU): equal, shard for shard and array for array, to bm25x_index_create_sharded_from_documents on the keyed documents
 * the document cast gives (doc id = position; bm25x_index_create_from_tsvectors), with the same payload, k1, b, n_shards,
 * devices and the bounds this call reports (bm25x_sharded_get_info): n_terms = the distinct keys of the whole batch
 * ascending bytewise, df / N / Σlen / avgdl the whole segment's, the keys with shard 0.  With doc_bounds == NULL the
 * bounds are bm25x_sharded_create's balanced ones with c_d = the ENTRIES of tsvector d (cum[d] = ent_off[d]), known
 * before any cast; for tsvectors with distinct lexemes (as PostgreSQL keeps them) that is the documents build's rule.
 * Two passes, and no shard's keys leave its device but its distinct ones: each shard's slice is cast on its own device
 * (the cast of bm25x_cast_tsvectors) and its distinct keys counted there; the host merges the shards' key lists into the
 * vocabulary and sums their counts into df; each shard's device turns its keys into the vocabulary's ordinals and frees
 * them; then the shards are built one after the other from (ordinal, tf).
 * Refusals (*out = NULL; every shard built so far destroyed and every cast freed, no device memory left behind), in
 * this order: null arguments; the tsvectors' host refusals (document mode); n of 0 or 0xFFFFFFFF, k1 and b
 * (bm25x_index_create_from_tsvectors' messages); the shard arguments with bm25x_sharded_create's messages; every
 * device (BM25X_ERR_CUDA).  Then, once EVERY shard is cast: the first vector (global numbering) with a merged count of 0
 * (BM25X_ERR_INVALID), then the first document with a merged tf >= 2^24 (BM25X_ERR_UNSUPPORTED), then more than
 * 0xFFFFFFFE distinct keys (BM25X_ERR_UNSUPPORTED), each with the unsharded call's message; BM25X_ERR_OOM /
 * BM25X_ERR_CUDA.  Device memory per device, for each of its shards: 20 B per entry of its own slice and 12 B per
 * tsvector (the cast), held until the vocabulary is known, plus the cast's chunk scratch while it runs and then the
 * vocabulary pass's scratch (the shards' passes run one after the other, once every shard is cast); then 16 B per term
 * of the vocabulary and 24 B per element while the ordinals are written; then 8 B per element (ordinal, tf) until that
 * shard is built; plus its index and the build from documents' inversion figures.  Host: each shard's distinct keys
 * (16 B each) and counts, the vocabulary (16 B per key), each shard's df (4 B per term), 12 B per tsvector. */
int bm25x_index_create_sharded_from_tsvectors(const bm25x_tsvectors *tsv, const uint8_t seed[32],
                                              const uint16_t *payload, double k1, double b, uint32_t n_shards,
                                              const uint32_t *doc_bounds, const int *devices,
                                              bm25x_sharded_index **out);
/* bm25x_tsvector_queries on a document-sharded index: equal to that call on the unsharded index of the same corpus.  The
 * query cast runs on shard 0's device against the segment's keys, which shard 0 holds; their device copy is made once
 * per sharded index (16 B per term) and freed with it.  Refusals: bm25x_tsvector_queries', named by this call (a keyless
 * sharded index: bm25x_lookup_terms' message).  Thread-safe alongside the searches on the same handle. */
int bm25x_tsvector_queries_sharded(bm25x_sharded_index *sx, const uint8_t seed[32], const bm25x_tsvectors *tsv,
                                   uint32_t *q_off, uint32_t *q_terms);
void bm25x_sharded_destroy(bm25x_sharded_index *sx);
/* info as the unsharded index would report it (n_docs, n_terms, n_postings, sum_doc_len, avgdl, k1, b); device_bytes
 * and n_blocks summed over the shards; device = shard 0's.  doc_bounds_out[n_shards+1] or NULL. */
int bm25x_sharded_get_info(const bm25x_sharded_index *sx, bm25x_index_info *out, uint32_t *n_shards_out,
                           uint32_t *doc_bounds_out);
int bm25x_sharded_set_option(bm25x_sharded_index *sx, const char *name, int64_t value); /* every shard */
int bm25x_sharded_lookup_terms(const bm25x_sharded_index *sx, const uint8_t *keys, uint32_t n, uint32_t *ordinals_out);
/* Same contract, arguments and outputs as bm25x_search_batch on an index created from `whole`: global doc ids, `allow`
 * over global ids, the same status codes and messages.  The shards run concurrently (one device each, or side by side
 * on a shared one).  stats: queries = live queries of the whole index; postings, postings_fetched, launches, bytes_algo
 * and kernel_ms are SUMS over the shards plus the merge launch — kernel_ms is summed device time, not wall time;
 * h2d_ms = canonicalise + upload of all shards, d2h_ms = merge wait + download. */
int bm25x_sharded_search_batch(bm25x_sharded_index *sx, uint32_t nq, const uint32_t *q_off, const uint32_t *q_terms,
                               uint32_t k, const uint8_t *allow, uint32_t *out_doc, float *out_score, double *out_score64,
                               uint16_t *out_payload, uint32_t *out_n, bm25x_search_stats *stats);
/* bm25x_search_candidates on a document-sharded index.  Named after bm25x_search_batch_growing rather than in the
 * bm25x_sharded_* family: that family's prototypes are a fixed set, pinned by the binding's declaration test
 * (tests/test_sharded.py), and this call takes the same sharded handle.  Candidates are global ids, routed by doc_bounds to their shard as
 * local ids; every shard runs the candidate search at k and the lists are merged on shard 0's device.  Rows equal those
 * of bm25x_search_candidates on an unsharded index of the same corpus.  Refusals are bm25x_sharded_search_batch's (the
 * whole segment's canonicalisation first), then those of the candidate lists; stats as bm25x_sharded_search_batch. */
int bm25x_search_candidates_sharded(bm25x_sharded_index *sx, uint32_t nq, const uint32_t *q_off, const uint32_t *q_terms,
                                    const uint32_t *c_off, const uint32_t *c_docs, uint32_t k, uint32_t *out_doc,
                                    float *out_score, double *out_score64, uint16_t *out_payload, uint32_t *out_n,
                                    bm25x_search_stats *stats);
/* A growing segment over a document-sharded index.  It scores with the whole segment's statistics (as every shard
 * does).  Its handle lives on the LAST shard's device.  After this call the segment is an ordinary
 * bm25x_growing_segment: insert, delete, refresh, get_info, get_index, search_batch and close take it unchanged, with
 * "the sealed index" meaning the whole segment (n_docs, n_terms, df, keys, Σlen / avgdl) and
 * bm25x_growing_info.device the last shard's.  bm25x_growing_search_batch then has the refusals of
 * bm25x_sharded_search_batch (the whole segment's canonicalisation first) and merges the shards' lists and the growing
 * handle's, growing ordinal o as n_docs(whole) + o, allow_sealed over global ids; stats: queries = live queries of the
 * whole segment plus the growing handle's, the rest sums over the shards, the growing handle and the merge launch.
 * Before the first insert it is bm25x_sharded_search_batch, stats included.  The sharded index must outlive the segment,
 * or the rebind to its successor (bm25x_growing_rebind_sharded);
 * bm25x_growing_seal refuses the segment (BM25X_ERR_INVALID). */
int bm25x_growing_open_sharded(bm25x_sharded_index *sealed, bm25x_growing_segment **out);
/* The seal of a segment opened with bm25x_growing_open_sharded.  The result is a new document-sharded index.  args,
 * refusals and concurrency are bm25x_growing_seal's (sealed_deleted over global ids, the maps give new global ids, equal
 * to those of bm25x_growing_seal on an unsharded index over the same corpus).  New shard j comes from an old shard and
 * holds its surviving documents in ascending old id; the old LAST shard also takes the growing survivors after its own.
 * An old shard left with no document is dropped; the rest keep their order and devices, the new bounds are the prefix
 * sums of the survivors.  Every shard scores with the new segment's statistics; the keys, when keyed, are with shard 0;
 * options are bm25x_sharded_create's defaults.  Each shard is rebuilt on its own device from its own arrays: at the peak a
 * device holds its old and new shards, the last one also the growing handle.  BM25X_ERR_OOM when a new shard does not
 * fit (bounds are not rebalanced).  The old sharded index and the segment are not changed; an unsharded segment is
 * refused (BM25X_ERR_INVALID). */
int bm25x_growing_seal_sharded(bm25x_growing_segment *g, bm25x_seal_args *args, bm25x_sharded_index **out);
/* ---- the rebind: the segment goes on over the index its latest seal built, as the reference's segment goes on after
 * `maintain` rewrote the sealed segment in place.  The ordinals the seal folded in ([0, n_folded)) leave the segment;
 * old ordinal n_folded + i becomes ordinal i.  Afterwards the segment equals, array for array, field for field and row
 * for row, bm25x_growing_open (or _open_sharded) on the new index followed by ONE insert of the carried documents
 * restated: each keeps its stored payload (the synthetic ctid of its OLD ordinal when none was given), its norm in the
 * segment's form and its deleted flag; each element is translated and the rows re-sorted by the new ordinal:
 *   - keyless index: the ordinal is unchanged (the seal keeps keyless ordinals stable);
 *   - a segment that owns its keys (bm25x_growing_insert_tsvectors): the element's key becomes its ordinal in the new
 *     vocabulary when the new index has it, else an owned key again, n_terms(new) + r, r its rank ascending bytewise
 *     among the carried keys the new vocabulary lacks (the numbering of one tsvector insert into a fresh segment);
 *   - keyed index, ordinals numbered by the caller: the seal's term map.  A carried ordinal >= n_source_terms (no key
 *     is known for it) or whose key vanished in the seal is refused (BM25X_ERR_INVALID, naming the first carried
 *     document and the ordinal): the caller inserts those documents again;
 *   - BM25X_TERM_MISSING stays missing.
 * A carried document deleted before the rebind keeps no element: its postings are gone, so its keys are not carried.
 * The carried documents then score with the new index's N, df and avgdl, as the reference's do after `maintain`.
 * late_deleted is the seal's growing map applied to the folded ordinals deleted since its snapshot: the caller ORs it
 * into allow_sealed and the next seal's sealed_deleted.
 * The call accepts only the handle the segment's latest successful seal returned, named by a serial number every index
 * and sharded handle gets when it is created (an address may be reused).  Until the rebind the segment keeps the record
 * of that seal: 4 B per folded ordinal and 4 B per source term on the host; a later seal replaces it, a rebind clears
 * it.  Refusals change nothing but this: the call refreshes the segment first, as a search does, so a refusal that
 * comes after the refresh (the keyed refusals, the tf one, BM25X_ERR_OOM / BM25X_ERR_CUDA) leaves it refreshed (get_info's pending
 * 0, the handle of the same documents rebuilt); the documents, the seal's record and every row stay as they were.
 * Refusals: null arguments; no seal to rebind to, or a handle that is not the latest seal's
 * result; an unsharded segment given to _sharded or the reverse; the keyed refusals above; a carried posting with
 * tf >= 2^24 on a term the new index holds (BM25X_ERR_UNSUPPORTED, as the insert of the restated documents refuses it);
 * BM25X_ERR_OOM / BM25X_ERR_CUDA.  Concurrency: the call is ordered with tsvector inserts and holds the segment's lock while it
 * refreshes and builds the carried documents' handle, then swaps sealed side, statistics and handle in one step.  Every
 * search, candidate search and tsvector query takes that binding as one, so it sees the old one or the new one, never a
 * mix; ordinal arguments (delete, allow_growing, candidate ids) are read against the binding the call locks.  The call
 * returns once every call that took the old binding has released it (a seal in flight included): the old index may then
 * be destroyed.  A seal that began before the rebind and would take its snapshot after it is refused (BM25X_ERR_INVALID,
 * "seal it again"); a seal whose snapshot came before the rebind returns its index but leaves no record, so a rebind to
 * that index is refused ("no seal to rebind to").  Device memory at the peak, on the new home device (the index, or its
 * last shard): the old handle and the new one, plus scratch: 4.125 B per old ordinal (the bitmap of the folded and
 * deleted ordinals, the map of the carried ones), 12 B per term of the old handle (the count and its scan), 8 B per old
 * source term (the offsets of the postings going up), 4 B per new term, n_carried / 8 B, and 8 B per carried posting
 * that moves between the handle and the host (down through the host or up from it).  When the seal dropped the old last
 * shard and the new last shard is on another device, every carried posting goes through the host: the scratch of the
 * old ordinals and old terms is then on the old device. */
typedef struct {
    uint8_t *late_deleted;    /* out, [ceil(n_docs(new)/8)] or NULL: bit d set = new sealed document d is a growing
                                 ordinal the seal folded in and the segment deleted after the seal's snapshot; every
                                 other bit written 0 (the layout of `allow` / sealed_deleted) */
    uint32_t n_late_deleted;  /* out */
    uint32_t n_folded;        /* out: the seal's n_growing */
    uint32_t n_carried;       /* out: ordinals carried over: old ordinal n_folded + i becomes ordinal i */
} bm25x_rebind_args;
int bm25x_growing_rebind(bm25x_growing_segment *g, bm25x_index *sealed, bm25x_rebind_args *a);
int bm25x_growing_rebind_sharded(bm25x_growing_segment *g, bm25x_sharded_index *sealed, bm25x_rebind_args *a);
/* Test hook: the arrays of shard s (0 <= s < n_shards) as bm25x_index_get_layout / bm25x_index_get_derived report them
 * for an index: local doc ids, local n_docs / n_postings / df, the whole segment's avgdl and score tables.  The shard
 * handle itself stays internal.  Either output may be NULL. */
int bm25x_sharded_get_shard(const bm25x_sharded_index *sx, uint32_t s, bm25x_index_layout *layout,
                            bm25x_index_derived *derived);
/* Test / measurement hook: k_merge_shards on host rows.  Shard s's rows are doc/score/score64/payload + s·nq·k
 * (payload: ·3) and n + s·nq, local doc ids, each row in canonical order; global id = local + doc_base[s], doc_base
 * ascending with s.  Outputs as bm25x_search_batch; merge_ms (or NULL) = the kernel's device time. */
int bm25x_merge_shards(int device, uint32_t n_shards, uint32_t nq, uint32_t k, const uint32_t *doc_base,
                       const uint32_t *doc, const float *score, const double *score64, const uint16_t *payload,
                       const uint32_t *n, uint32_t *out_doc, float *out_score, double *out_score64,
                       uint16_t *out_payload, uint32_t *out_n, float *merge_ms);

/* Invariants of the reference's vector types (crates/bm25/src/vector.rs:46-134): n vectors in CSR form, keys strictly
 * ascending inside a vector, term frequencies (tfs, NULL for Query-like vectors) non-zero — what Document::new / Query::new
 * enforce with expect("invalid data").  BM25X_ERR_INVALID names the first offending vector.  Host only. */
int bm25x_check_vectors(uint32_t n, const uint32_t *off, const uint32_t *terms, const uint32_t *tfs);

/* ---- bm25::evaluate (crates/bm25/src/evaluate.rs:22-74) behind `<&>` without an index scan
 * (src/index/operators.rs:22-55): pair p scores document [d_off[p], d_off[p+1]) (sorted distinct term ordinals
 * with tfs) against query [q_off[p], q_off[p+1]) (sorted distinct ordinals).  out[p] = the f64 score, >= 0.
 * It scores with the handle's own statistics: its N, df, avgdl, k1 and b.  The document's length is the saturating
 * Σ tf (up to 2^32 - 1 per element and in sum), not a stored norm.  Query terms the document lacks, ordinals >= n_terms
 * (BM25X_TERM_MISSING included) and terms of df 0 add nothing; a query has no term limit.  A replica's tables follow
 * its latest bm25x_index_finalize_replica.
 * BM25X_ERR_INVALID, writing nothing to out: a null argument, vectors that break bm25x_check_vectors, a replica not
 * finalized, and a handle that scores with another segment's statistics (bm25x_growing_create's, or a replica of one;
 * evaluate on the sealed index instead). */
int bm25x_evaluate_batch(bm25x_index *idx, uint32_t n_pairs, const uint32_t *d_off, const uint32_t *d_terms,
                         const uint32_t *d_tfs, const uint32_t *q_off, const uint32_t *q_terms, double *out);
/* `<&>` from tsvectors in one call, what _bm25_evaluate(tsvector, bm25query) does (src/index/operators.rs:22-55): there
 * are docs->n pairs, and out[p] = bm25::evaluate of cast_tsvector_to_document(docs[p]) against
 * cast_tsvector_to_query(queries[pair_query ? pair_query[p] : p]), with the handle's N, df, avgdl, k1 and b.  Many rows
 * against one query: queries->n == 1 and every pair_query entry 0.  Both casts run on the index's device against the
 * copy of its vocabulary that bm25x_tsvector_queries keeps; the rows stay there in key order, known lexemes as their
 * ordinals and unknown ones as BM25X_TERM_MISSING, which score nothing but count in the document's length
 * (Document::length, vector.rs:77-83).  No key is numbered or re-sorted, and only out comes down.  A merged tf >= 2^24 is
 * scored (evaluate has no packed posting layout).
 * Refusals, BM25X_ERR_INVALID with out untouched, in this order and before any device work: a null argument (out may be
 * NULL when docs->n == 0, pair_query may be NULL); the document tsvectors' host refusals (document mode, "tsvector must
 * have positions" included), then the queries' (query mode); pair_query NULL with queries->n != docs->n, or an entry >=
 * queries->n (naming the pair); a replica not finalized; a handle that scores with another segment's statistics (as
 * bm25x_evaluate_batch); an index without term keys (bm25x_lookup_terms' message).  Then, after the casts and before out
 * is written, the first document with a merged count of 0 (the cast's message).  BM25X_ERR_OOM / BM25X_ERR_CUDA from the
 * device.  Thread-safe alongside the searches on the same handle; the idf table and the vocabulary copy are built once
 * per handle.  Device memory until the call returns: 8 B per document element and 28 B per document tsvector, 4 B per
 * query element and 16 B per query tsvector, 12 B per pair, plus one upload chunk of the cast (bm25x_cast_tsvectors);
 * kept with the handle after the first call: 8 B (idf) and 16 B (vocabulary) per term. */
int bm25x_evaluate_tsvectors(bm25x_index *idx, const uint8_t seed[32], const bm25x_tsvectors *docs,
                             const bm25x_tsvectors *queries, const uint32_t *pair_query, double *out);
/* bm25x_evaluate_batch and bm25x_evaluate_tsvectors on a document-sharded index: each returns exactly what its
 * unsharded form returns on an index of the same corpus (the whole segment's N, df, avgdl, k1 and b), with its refusals,
 * named by this call (there are no replicas or growing handles among sharded indexes).  Everything runs on shard 0's
 * device, which holds the segment's keys and, for the tsvector call, their device copy (bm25x_tsvector_queries_sharded's).
 * The whole segment's df and idf go to that device once per sharded index (12 B per term) and are freed by
 * bm25x_sharded_destroy.  A keyless sharded index is served by the ordinal call and refused by the tsvector call
 * (bm25x_lookup_terms' message).  Named in the bm25x_evaluate_* family rather than the bm25x_sharded_* one, whose
 * prototypes are a fixed set (see bm25x_search_candidates_sharded). */
int bm25x_evaluate_batch_sharded(bm25x_sharded_index *sx, uint32_t n_pairs, const uint32_t *d_off,
                                 const uint32_t *d_terms, const uint32_t *d_tfs, const uint32_t *q_off,
                                 const uint32_t *q_terms, double *out);
int bm25x_evaluate_tsvectors_sharded(bm25x_sharded_index *sx, const uint8_t seed[32], const bm25x_tsvectors *docs,
                                     const bm25x_tsvectors *queries, const uint32_t *pair_query, double *out);

/* ---- synthetic corpus generator (bench/test utility; spec in DESIGN.md, mirrors tests/fuzz:168-205).
 * Fills a host CSR the caller frees with bm25x_synth_free. zipf_s == 0 ⇒ uniform vocabulary. */
typedef struct {
    uint32_t n_docs, n_terms;
    uint64_t n_postings;
    uint32_t *doc_len;
    uint64_t *post_off;
    uint32_t *post_doc;
    uint32_t *post_tf;
} bm25x_synth_corpus;
int bm25x_synth_generate(uint64_t seed, uint32_t n_docs, uint32_t vocab, uint32_t len_min, uint32_t len_max,
                         double zipf_s, int nthreads, bm25x_synth_corpus *out);
void bm25x_synth_free(bm25x_synth_corpus *c);
/* Queries: n_min..n_max distinct terms with df > 0 drawn from the same distribution. q_off[nq+1], q_terms[nq*n_max]. */
int bm25x_synth_queries(uint64_t seed, uint32_t nq, uint32_t vocab, uint32_t n_min, uint32_t n_max, double zipf_s,
                        const uint64_t *post_off, uint32_t *q_off, uint32_t *q_terms);

const char *bm25x_last_error(void);
int bm25x_device_count(void);

#ifdef __cplusplus
}
#endif
#endif
