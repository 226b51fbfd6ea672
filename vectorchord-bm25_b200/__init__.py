"""vectorchord-bm25_b200 — H100-native (sm_90a) BM25 top-k engine (one hot path of tensorchord/VectorChord-bm25).

The product is the C-ABI shared library `libbm25x.so` (sources in csrc/, header in include/bm25x.h).
This package is the thin Python host binding used by tests and bench.py; it mirrors the reference's
host-side interface for the path (`bm25::search` / `bm25::evaluate`, Document / Query) and never
falls back to a CPU implementation: if the library or an H100 is missing, calls raise.
"""
from .bm25x import (Bm25xError, Index, Batch, SearchStats, IndexLayout, IndexDerived, synth_corpus, synth_queries, load_library, build_library,
                    device_count, Document, Query, MAX_K, MAX_QUERY_TERMS, TERM_MISSING, merge_topk, check_vectors, Broker,
                    ShardedIndex, MAX_SHARDS, merge_shards, GrowingSegment, GrowingInfo, SealArgs, RebindArgs, Export,
                    cast_tsvectors)

__all__ = ["Bm25xError", "Index", "Batch", "SearchStats", "IndexLayout", "IndexDerived", "synth_corpus", "synth_queries", "load_library",
           "build_library", "device_count", "Document", "Query", "MAX_K", "MAX_QUERY_TERMS", "TERM_MISSING", "merge_topk",
           "check_vectors", "Broker", "ShardedIndex", "MAX_SHARDS", "merge_shards",
           "GrowingSegment", "GrowingInfo", "SealArgs", "RebindArgs", "Export", "cast_tsvectors"]
