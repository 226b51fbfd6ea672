"""ctypes binding of include/bm25x.h (the drop-in C ABI).  No torch types cross this boundary."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
# BM25X_LIBRARY: load another build of the same library (tools/time_variants.py times tuning variants side by side)
_SO = os.environ.get("BM25X_LIBRARY") or os.path.join(_HERE, "libbm25x.so")

MAX_K = 65535
MAX_QUERY_TERMS = 64
TERM_MISSING = 0xFFFFFFFF


class Bm25xError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"bm25x error {code}: {msg}")
        self.code = code


class _Corpus(C.Structure):
    _fields_ = [("n_docs", C.c_uint32), ("doc_len", C.POINTER(C.c_uint32)), ("payload", C.POINTER(C.c_uint16)),
                ("n_terms", C.c_uint32), ("term_key", C.POINTER(C.c_uint8)), ("post_off", C.POINTER(C.c_uint64)),
                ("post_doc", C.POINTER(C.c_uint32)), ("post_tf", C.POINTER(C.c_uint32)), ("k1", C.c_double),
                ("b", C.c_double)]


class _Blocks(C.Structure):
    _fields_ = [("n_docs", C.c_uint32), ("doc_len", C.POINTER(C.c_uint32)), ("doc_fieldnorm", C.POINTER(C.c_uint8)),
                ("sum_doc_len", C.c_uint64), ("payload", C.POINTER(C.c_uint16)), ("n_terms", C.c_uint32),
                ("term_key", C.POINTER(C.c_uint8)), ("term_blk_off", C.POINTER(C.c_uint64)), ("n_blocks", C.c_uint64),
                ("blk_min_doc", C.POINTER(C.c_uint32)), ("blk_n", C.POINTER(C.c_uint32)),
                ("blk_meta_doc", C.POINTER(C.c_uint8)), ("blk_meta_tf", C.POINTER(C.c_uint8)),
                ("blk_doc_off", C.POINTER(C.c_uint64)), ("blk_tf_off", C.POINTER(C.c_uint64)),
                ("bytes", C.POINTER(C.c_uint8)), ("n_bytes", C.c_uint64), ("k1", C.c_double), ("b", C.c_double),
                ("blk_wand_fieldnorm", C.POINTER(C.c_uint8)), ("blk_wand_tf", C.POINTER(C.c_uint32))]


class _Documents(C.Structure):  # bm25x_documents
    _fields_ = [("n_docs", C.c_uint32), ("elem_off", C.POINTER(C.c_uint64)), ("elem_key", C.POINTER(C.c_uint8)),
                ("elem_term", C.POINTER(C.c_uint32)), ("elem_tf", C.POINTER(C.c_uint32)), ("payload", C.POINTER(C.c_uint16)),
                ("n_terms", C.c_uint32), ("k1", C.c_double), ("b", C.c_double)]


class _Tsvectors(C.Structure):  # bm25x_tsvectors
    _fields_ = [("n", C.c_uint32), ("ent_off", C.POINTER(C.c_uint64)), ("entries", C.POINTER(C.c_uint32)),
                ("byte_off", C.POINTER(C.c_uint64)), ("bytes", C.POINTER(C.c_uint8))]


class Export(C.Structure):  # bm25x_export
    _fields_ = [("doc_fieldnorm", C.POINTER(C.c_uint8)), ("payload", C.POINTER(C.c_uint16)), ("sum_doc_len", C.c_uint64),
                ("term_key", C.POINTER(C.c_uint8)), ("tok_df", C.POINTER(C.c_uint32)),
                ("tok_wand_fieldnorm", C.POINTER(C.c_uint8)), ("tok_wand_tf", C.POINTER(C.c_uint32)),
                ("term_blk_off", C.POINTER(C.c_uint64)), ("blk_min_doc", C.POINTER(C.c_uint32)),
                ("blk_max_doc", C.POINTER(C.c_uint32)), ("blk_n", C.POINTER(C.c_uint32)),
                ("blk_meta_doc", C.POINTER(C.c_uint8)), ("blk_meta_tf", C.POINTER(C.c_uint8)),
                ("blk_doc_off", C.POINTER(C.c_uint64)), ("blk_tf_off", C.POINTER(C.c_uint64)),
                ("blk_wand_fieldnorm", C.POINTER(C.c_uint8)), ("blk_wand_tf", C.POINTER(C.c_uint32)),
                ("bytes", C.POINTER(C.c_uint8)), ("bytes_cap", C.c_uint64), ("n_bytes", C.c_uint64)]


class _GrowingDocs(C.Structure):
    _fields_ = [("n_docs", C.c_uint32), ("doc_len", C.POINTER(C.c_uint32)), ("doc_fieldnorm", C.POINTER(C.c_uint8)),
                ("payload", C.POINTER(C.c_uint16)), ("deleted", C.POINTER(C.c_uint8)),
                ("elem_off", C.POINTER(C.c_uint64)), ("elem_term", C.POINTER(C.c_uint32)),
                ("elem_tf", C.POINTER(C.c_uint32))]


class GrowingInfo(C.Structure):  # bm25x_growing_info
    _fields_ = [("n_docs", C.c_uint32), ("n_deleted", C.c_uint32), ("n_postings", C.c_uint64),
                ("device_bytes", C.c_uint64), ("pending", C.c_uint32), ("device", C.c_int)]


class SealArgs(C.Structure):  # bm25x_seal_args
    _fields_ = [("sealed_deleted", C.POINTER(C.c_uint8)), ("new_keys", C.POINTER(C.c_uint8)), ("n_new_keys", C.c_uint32),
                ("sealed_map", C.POINTER(C.c_uint32)), ("growing_map", C.POINTER(C.c_uint32)), ("growing_cap", C.c_uint32),
                ("term_map", C.POINTER(C.c_uint32)), ("term_cap", C.c_uint32), ("n_growing", C.c_uint32),
                ("n_source_terms", C.c_uint32)]


class RebindArgs(C.Structure):  # bm25x_rebind_args
    _fields_ = [("late_deleted", C.POINTER(C.c_uint8)), ("n_late_deleted", C.c_uint32), ("n_folded", C.c_uint32),
                ("n_carried", C.c_uint32)]


class IndexInfo(C.Structure):
    _fields_ = [("n_docs", C.c_uint32), ("n_terms", C.c_uint32), ("n_postings", C.c_uint64),
                ("sum_doc_len", C.c_uint64), ("avgdl", C.c_double), ("k1", C.c_double), ("b", C.c_double),
                ("device_bytes", C.c_uint64), ("n_blocks", C.c_uint64), ("device", C.c_int)]


N_ARRAYS = 13


class IndexLayout(C.Structure):
    _fields_ = [("n_docs", C.c_uint32), ("n_terms", C.c_uint32), ("n_postings", C.c_uint64),
                ("n_postings_padded", C.c_uint64), ("n_blocks", C.c_uint64), ("sum_doc_len", C.c_uint64),
                ("k1", C.c_double), ("b", C.c_double), ("avgdl", C.c_double), ("dev_ptr", C.c_void_p * N_ARRAYS),
                ("bytes", C.c_uint64 * N_ARRAYS), ("device", C.c_int)]


class IndexDerived(C.Structure):  # bm25x_index_derived: test hook, the arrays an index builds and never replicates
    _fields_ = [("pdoc", C.c_void_p), ("pdoc_bytes", C.c_uint64), ("champ", C.c_void_p), ("champ_bytes", C.c_uint64),
                ("champ_off", C.c_void_p), ("champ_off_bytes", C.c_uint64), ("n_champ", C.c_uint64),
                ("s1f_min", C.c_float), ("device", C.c_int)]


class BrokerOptions(C.Structure):  # bm25x_broker_options (include/bm25x_broker.h)
    _fields_ = [("max_batch", C.c_uint32), ("max_wait_us", C.c_uint32), ("ring_slots", C.c_uint32), ("reserved", C.c_uint32)]


class BrokerStats(C.Structure):  # bm25x_broker_stats
    _fields_ = [("requests", C.c_uint64), ("batches", C.c_uint64), ("max_batch_seen", C.c_uint64),
                ("ring_full_waits", C.c_uint64), ("rejected", C.c_uint64)]


# bm25x_broker_backend: (ctx, nq, q_off, q_terms, k, out_doc, out_score, out_score64, out_payload, out_n) -> status
BROKER_BACKEND = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), C.c_uint32,
                             C.POINTER(C.c_uint32), C.POINTER(C.c_float), C.POINTER(C.c_double), C.POINTER(C.c_uint16),
                             C.POINTER(C.c_uint32))


class SearchStats(C.Structure):
    _fields_ = [("kernel_ms", C.c_double), ("h2d_ms", C.c_double), ("d2h_ms", C.c_double), ("postings", C.c_uint64),
                ("bytes_algo", C.c_uint64), ("launches", C.c_uint32), ("queries", C.c_uint32),
                ("postings_fetched", C.c_uint64)]


class _Synth(C.Structure):
    _fields_ = [("n_docs", C.c_uint32), ("n_terms", C.c_uint32), ("n_postings", C.c_uint64),
                ("doc_len", C.POINTER(C.c_uint32)), ("post_off", C.POINTER(C.c_uint64)),
                ("post_doc", C.POINTER(C.c_uint32)), ("post_tf", C.POINTER(C.c_uint32))]


def build_library(force: bool = False) -> str:
    """nvcc -gencode arch=compute_90a,code=sm_90a build of csrc/ → libbm25x.so (in-tree)."""
    srcdir = os.path.join(_HERE, "csrc")
    srcs = [os.path.join(srcdir, f) for f in os.listdir(srcdir)] + [os.path.join(_HERE, "..", "include", "bm25x.h")]
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < max(os.path.getmtime(s) for s in srcs):
        subprocess.check_call(["make", "-C", srcdir, "-s"], stdout=subprocess.DEVNULL)
    return _SO


_lib = None


def load_library():
    """Loads libbm25x.so; raises (never falls back) when it is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_SO):
        raise Bm25xError(-1, f"{_SO} not built: run `python -c 'import __graft_entry__ as g; g.build()'`")
    L = C.CDLL(_SO)
    vp, u8p, u16p, u32p, u64p, f32p, f64p = (C.c_void_p, C.POINTER(C.c_uint8), C.POINTER(C.c_uint16),
                                             C.POINTER(C.c_uint32), C.POINTER(C.c_uint64), C.POINTER(C.c_float),
                                             C.POINTER(C.c_double))
    L.bm25x_index_create.argtypes = [C.POINTER(_Corpus), C.c_int, C.POINTER(vp)]
    L.bm25x_index_create_from_blocks.argtypes = [C.POINTER(_Blocks), C.c_int, C.POINTER(vp)]
    L.bm25x_index_export_blocks.argtypes = [vp, C.POINTER(Export)]
    L.bm25x_index_create_from_documents.argtypes = [C.POINTER(_Documents), C.c_int, C.POINTER(vp)]
    L.bm25x_cast_tsvectors.argtypes = [C.POINTER(_Tsvectors), u8p, C.c_int, C.c_int, u64p, u8p, u32p]
    L.bm25x_index_create_from_tsvectors.argtypes = [C.POINTER(_Tsvectors), u8p, u16p, C.c_double, C.c_double, C.c_int,
                                                    C.POINTER(vp)]
    L.bm25x_tsvector_queries.argtypes = [vp, u8p, C.POINTER(_Tsvectors), u32p, u32p]
    L.bm25x_growing_create.argtypes = [vp, C.POINTER(_GrowingDocs), C.POINTER(vp)]
    L.bm25x_search_batch_growing.argtypes = [vp, vp, C.c_uint32, u32p, u32p, C.c_uint32, u8p, u8p, u32p, f32p, f64p,
                                             u16p, u32p, C.POINTER(SearchStats)]
    L.bm25x_growing_open.argtypes = [vp, C.POINTER(vp)]
    L.bm25x_growing_insert.argtypes = [vp, C.POINTER(_GrowingDocs)]
    L.bm25x_growing_delete.argtypes = [vp, C.c_uint32, u32p]
    L.bm25x_growing_refresh.argtypes = [vp]
    L.bm25x_growing_get_info.argtypes = [vp, C.POINTER(GrowingInfo)]
    L.bm25x_growing_search_batch.argtypes = [vp, C.c_uint32, u32p, u32p, C.c_uint32, u8p, u8p, C.c_uint32, u32p, f32p,
                                             f64p, u16p, u32p, C.POINTER(SearchStats)]
    L.bm25x_growing_get_index.argtypes = [vp, C.POINTER(IndexLayout), C.POINTER(IndexDerived)]
    L.bm25x_growing_close.argtypes = [vp]
    L.bm25x_growing_close.restype = None
    L.bm25x_growing_seal.argtypes = [vp, C.POINTER(SealArgs), C.POINTER(vp)]
    L.bm25x_growing_open_sharded.argtypes = [vp, C.POINTER(vp)]
    L.bm25x_growing_seal_sharded.argtypes = [vp, C.POINTER(SealArgs), C.POINTER(vp)]
    L.bm25x_growing_rebind.argtypes = [vp, vp, C.POINTER(RebindArgs)]
    L.bm25x_growing_rebind_sharded.argtypes = [vp, vp, C.POINTER(RebindArgs)]
    L.bm25x_growing_insert_tsvectors.argtypes = [vp, u8p, C.POINTER(_Tsvectors), u16p]
    L.bm25x_growing_get_new_keys.argtypes = [vp, C.c_uint32, u8p, u32p]
    L.bm25x_growing_tsvector_queries.argtypes = [vp, u8p, C.POINTER(_Tsvectors), u32p, u32p]
    L.bm25x_merge_topk.argtypes = [C.c_uint32, C.c_uint32, u32p, f32p, f64p, u16p, u32p, u32p, f32p, f64p, u16p, u32p,
                                   C.c_uint32, u32p, f32p, f64p, u16p, u32p]
    L.bm25x_index_destroy.argtypes = [vp]
    L.bm25x_index_destroy.restype = None
    L.bm25x_index_get_info.argtypes = [vp, C.POINTER(IndexInfo)]
    L.bm25x_lookup_terms.argtypes = [vp, u8p, C.c_uint32, u32p]
    L.bm25x_index_get_layout.argtypes = [vp, C.POINTER(IndexLayout)]
    L.bm25x_index_alloc_replica.argtypes = [C.POINTER(IndexLayout), C.c_int, C.POINTER(vp)]
    L.bm25x_index_finalize_replica.argtypes = [vp]
    L.bm25x_index_get_derived.argtypes = [vp, C.POINTER(IndexDerived)]
    L.bm25x_index_get_df.argtypes = [vp, u32p]
    L.bm25x_index_set_option.argtypes = [vp, C.c_char_p, C.c_int64]
    L.bm25x_search_batch.argtypes = [vp, C.c_uint32, u32p, u32p, C.c_uint32, u8p, u32p, f32p, f64p, u16p, u32p,
                                     C.POINTER(SearchStats)]
    L.bm25x_search_candidates.argtypes = [vp, C.c_uint32, u32p, u32p, u32p, u32p, C.c_uint32, u32p, f32p, f64p, u16p,
                                          u32p, C.POINTER(SearchStats)]
    L.bm25x_search_candidates_sharded.argtypes = L.bm25x_search_candidates.argtypes
    L.bm25x_growing_search_candidates.argtypes = L.bm25x_search_candidates.argtypes
    L.bm25x_batch_prepare.argtypes = [vp, C.c_uint32, u32p, u32p, C.c_uint32, u8p, C.POINTER(vp)]
    L.bm25x_batch_run.argtypes = [vp, vp, C.POINTER(SearchStats)]
    L.bm25x_batch_fetch.argtypes = [vp, u32p, f32p, f64p, u16p, u32p]
    L.bm25x_batch_device_results.argtypes = [vp, C.POINTER(vp), C.POINTER(vp), C.POINTER(vp), C.POINTER(vp), C.POINTER(vp)]
    L.bm25x_batch_destroy.argtypes = [vp]
    L.bm25x_batch_destroy.restype = None
    L.bm25x_evaluate_batch.argtypes = [vp, C.c_uint32, u32p, u32p, u32p, u32p, u32p, f64p]
    L.bm25x_evaluate_batch_sharded.argtypes = L.bm25x_evaluate_batch.argtypes
    L.bm25x_evaluate_tsvectors.argtypes = [vp, u8p, C.POINTER(_Tsvectors), C.POINTER(_Tsvectors), u32p, f64p]
    L.bm25x_evaluate_tsvectors_sharded.argtypes = L.bm25x_evaluate_tsvectors.argtypes
    L.bm25x_check_vectors.argtypes = [C.c_uint32, u32p, u32p, u32p]
    L.bm25x_synth_generate.argtypes = [C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_double,
                                       C.c_int, C.POINTER(_Synth)]
    L.bm25x_synth_free.argtypes = [C.POINTER(_Synth)]
    L.bm25x_synth_free.restype = None
    L.bm25x_synth_queries.argtypes = [C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_double, u64p,
                                      u32p, u32p]
    L.bm25x_intern.argtypes = [u8p, u8p, C.c_size_t, u8p]
    L.bm25x_blake3_keyed16.argtypes = [u8p, u8p, C.c_size_t, u8p]
    L.bm25x_broker_create.argtypes = [vp, C.POINTER(BrokerOptions), C.POINTER(vp)]
    L.bm25x_broker_create_with_backend.argtypes = [BROKER_BACKEND, vp, C.POINTER(BrokerOptions), C.POINTER(vp)]
    L.bm25x_broker_search.argtypes = [vp, u32p, C.c_uint32, C.c_uint32, u32p, f64p, u16p, u32p]
    L.bm25x_broker_get_stats.argtypes = [vp, C.POINTER(BrokerStats)]
    L.bm25x_broker_destroy.argtypes = [vp]
    L.bm25x_broker_destroy.restype = None
    L.bm25x_sharded_create.argtypes = [C.POINTER(_Corpus), C.c_uint32, u32p, C.POINTER(C.c_int), C.POINTER(vp)]
    L.bm25x_index_create_sharded_from_blocks.argtypes = [C.POINTER(_Blocks), C.c_uint32, u32p, C.POINTER(C.c_int),
                                                         C.POINTER(vp)]
    L.bm25x_index_create_sharded_from_documents.argtypes = [C.POINTER(_Documents), C.c_uint32, u32p, C.POINTER(C.c_int),
                                                            C.POINTER(vp)]
    L.bm25x_index_create_sharded_from_tsvectors.argtypes = [C.POINTER(_Tsvectors), u8p, u16p, C.c_double, C.c_double,
                                                             C.c_uint32, u32p, C.POINTER(C.c_int), C.POINTER(vp)]
    L.bm25x_tsvector_queries_sharded.argtypes = [vp, u8p, C.POINTER(_Tsvectors), u32p, u32p]
    L.bm25x_sharded_destroy.argtypes = [vp]
    L.bm25x_sharded_destroy.restype = None
    L.bm25x_sharded_get_info.argtypes = [vp, C.POINTER(IndexInfo), u32p, u32p]
    L.bm25x_sharded_set_option.argtypes = [vp, C.c_char_p, C.c_int64]
    L.bm25x_sharded_lookup_terms.argtypes = [vp, u8p, C.c_uint32, u32p]
    L.bm25x_sharded_get_shard.argtypes = [vp, C.c_uint32, C.POINTER(IndexLayout), C.POINTER(IndexDerived)]
    L.bm25x_sharded_search_batch.argtypes = [vp, C.c_uint32, u32p, u32p, C.c_uint32, u8p, u32p, f32p, f64p, u16p, u32p,
                                             C.POINTER(SearchStats)]
    L.bm25x_merge_shards.argtypes = [C.c_int, C.c_uint32, C.c_uint32, C.c_uint32, u32p, u32p, f32p, f64p, u16p, u32p,
                                     u32p, f32p, f64p, u16p, u32p, f32p]
    L.bm25x_last_error.restype = C.c_char_p
    L.bm25x_device_count.restype = C.c_int
    _lib = L
    return L


def intern(seed: bytes, token: bytes) -> bytes:
    """vector::intern (crates/bm25/src/vector.rs:19-35): 16-byte key of a token under the index seed."""
    assert len(seed) == 32
    out = (C.c_uint8 * 16)()
    sd = (C.c_uint8 * 32).from_buffer_copy(seed)
    tk = (C.c_uint8 * max(len(token), 1)).from_buffer_copy(token if token else b"\0")
    _check(load_library().bm25x_intern(sd, tk, len(token), out))
    return bytes(out)


def blake3_keyed16(key: bytes, data: bytes) -> bytes:
    out = (C.c_uint8 * 16)()
    kk = (C.c_uint8 * 32).from_buffer_copy(key)
    dd = (C.c_uint8 * max(len(data), 1)).from_buffer_copy(data if data else b"\0")
    _check(load_library().bm25x_blake3_keyed16(kk, dd, len(data), out))
    return bytes(out)


def _check(rc):
    if rc != 0:
        raise Bm25xError(rc, load_library().bm25x_last_error().decode())


def _p(a, ty):
    return a.ctypes.data_as(C.POINTER(ty)) if a is not None else None


def _kept(keep, a, dt, ct):
    """Pointer to `a` as a contiguous `dt` array, which `keep` holds alive until the library has copied it."""
    a = np.ascontiguousarray(a, dtype=dt)
    keep.append(a)
    return _p(a, ct)


def _corpus(keep, n_docs, doc_len, n_terms, post_off, post_doc, post_tf, k1, b, payload, term_keys):
    c = _Corpus()
    c.n_docs, c.n_terms, c.k1, c.b = int(n_docs), int(n_terms), float(k1), float(b)
    c.doc_len = _kept(keep, doc_len, np.uint32, C.c_uint32)
    c.post_off = _kept(keep, post_off, np.uint64, C.c_uint64)
    c.post_doc = _kept(keep, post_doc, np.uint32, C.c_uint32)
    c.post_tf = _kept(keep, post_tf, np.uint32, C.c_uint32)
    if payload is not None:
        c.payload = _kept(keep, payload, np.uint16, C.c_uint16)
    if term_keys is not None:
        c.term_key = _kept(keep, term_keys, np.uint8, C.c_uint8)
    return c


def _blocks(keep, n_docs, n_terms, term_blk_off, blk_min_doc, blk_n, blk_meta_doc, blk_meta_tf, blk_doc_off, blk_tf_off,
            data, doc_len, doc_fieldnorm, sum_doc_len, k1, b, payload, term_keys, blk_wand_fieldnorm, blk_wand_tf):
    c = _Blocks()
    c.n_docs, c.n_terms, c.k1, c.b = int(n_docs), int(n_terms), float(k1), float(b)
    if doc_len is not None:
        c.doc_len = _kept(keep, doc_len, np.uint32, C.c_uint32)
    if doc_fieldnorm is not None:
        c.doc_fieldnorm = _kept(keep, doc_fieldnorm, np.uint8, C.c_uint8)
    c.sum_doc_len = int(sum_doc_len)
    if payload is not None:
        c.payload = _kept(keep, payload, np.uint16, C.c_uint16)
    if term_keys is not None:
        c.term_key = _kept(keep, term_keys, np.uint8, C.c_uint8)
    c.term_blk_off = _kept(keep, term_blk_off, np.uint64, C.c_uint64)
    c.n_blocks = int(keep[-1][int(n_terms)]) if len(keep[-1]) > int(n_terms) else 0
    c.blk_min_doc = _kept(keep, blk_min_doc, np.uint32, C.c_uint32)
    c.blk_n = _kept(keep, blk_n, np.uint32, C.c_uint32)
    c.blk_meta_doc = _kept(keep, blk_meta_doc, np.uint8, C.c_uint8)
    c.blk_meta_tf = _kept(keep, blk_meta_tf, np.uint8, C.c_uint8)
    c.blk_doc_off = _kept(keep, blk_doc_off, np.uint64, C.c_uint64)
    c.blk_tf_off = _kept(keep, blk_tf_off, np.uint64, C.c_uint64)
    c.bytes = _kept(keep, data, np.uint8, C.c_uint8)
    c.n_bytes = len(keep[-1])
    if blk_wand_fieldnorm is not None and blk_wand_tf is not None:   # SummaryTuple.wand_* (checked against the blocks)
        c.blk_wand_fieldnorm = _kept(keep, blk_wand_fieldnorm, np.uint8, C.c_uint8)
        c.blk_wand_tf = _kept(keep, blk_wand_tf, np.uint32, C.c_uint32)
    return c


def _documents(keep, elem_off, elem_tf, elem_term, elem_key, n_terms, payload, k1, b):
    c = _Documents()
    c.elem_off = _kept(keep, elem_off, np.uint64, C.c_uint64)
    c.n_docs = len(keep[-1]) - 1
    c.elem_tf = _kept(keep, elem_tf, np.uint32, C.c_uint32)
    if elem_term is not None:
        c.elem_term = _kept(keep, elem_term, np.uint32, C.c_uint32)
    if elem_key is not None:
        c.elem_key = _kept(keep, elem_key, np.uint8, C.c_uint8)
    if payload is not None:
        c.payload = _kept(keep, payload, np.uint16, C.c_uint16)
    c.n_terms, c.k1, c.b = int(n_terms), float(k1), float(b)
    return c


def _tsvectors(keep, ent_off, entries, byte_off, data):
    """bm25x_tsvectors over host arrays: vector i = WordEntry words entries[ent_off[i]:ent_off[i+1]] and lexeme area
    data[byte_off[i]:byte_off[i+1]] (what follows each datum's header)."""
    t = _Tsvectors()
    t.ent_off = _kept(keep, ent_off, np.uint64, C.c_uint64)
    t.n = len(keep[-1]) - 1
    t.entries = _kept(keep, entries, np.uint32, C.c_uint32)
    t.byte_off = _kept(keep, byte_off, np.uint64, C.c_uint64)
    t.bytes = _kept(keep, np.frombuffer(data, np.uint8) if isinstance(data, (bytes, bytearray)) else data, np.uint8,
                    C.c_uint8)
    return t


def _seed(seed):
    assert len(seed) == 32
    return (C.c_uint8 * 32).from_buffer_copy(bytes(seed))


def cast_tsvectors(seed, ent_off, entries, byte_off, data, as_query=False, device=0):
    """cast_tsvector_to_document (or, as_query, cast_tsvector_to_query) of every tsvector on the GPU
    (bm25x_cast_tsvectors).  Returns (off u64 [n+1], keys u8 [E, 16], tf u32 [E] or None): row i = off[i]:off[i+1], its
    keys ascending bytewise and distinct, tf the saturating sum of the merged position counts."""
    keep = []
    t = _tsvectors(keep, ent_off, entries, byte_off, data)
    E = int(keep[0][-1]) if len(keep[0]) else 0
    off = np.zeros(t.n + 1, np.uint64)
    keys = np.zeros((max(E, 1), 16), np.uint8)
    tf = None if as_query else np.zeros(max(E, 1), np.uint32)
    _check(load_library().bm25x_cast_tsvectors(C.byref(t), _seed(seed), int(bool(as_query)), device, _p(off, C.c_uint64),
                                               _p(keys, C.c_uint8), _p(tf, C.c_uint32)))
    n = int(off[-1])
    return off, keys[:n].copy(), None if tf is None else tf[:n].copy()


def _result_arrays(nq, k, want_f64, want_payload):
    return {"doc": np.empty((nq, k), np.uint32), "score": np.empty((nq, k), np.float32),
            "score64": np.empty((nq, k), np.float64) if want_f64 else None,
            "payload": np.empty((nq, k, 3), np.uint16) if want_payload else None, "n": np.empty(nq, np.uint32)}


def _rows_args(out):
    """The five result arrays of a dict of _result_arrays as the out_doc .. out_n arguments of a search or merge."""
    return (_p(out["doc"], C.c_uint32), _p(out["score"], C.c_float), _p(out["score64"], C.c_double),
            _p(out["payload"], C.c_uint16), _p(out["n"], C.c_uint32))


def _search_batch(fn, h, q_off, q_terms, k, allow, want_f64, want_payload, out):
    """bm25x_search_batch or bm25x_sharded_search_batch (the same signature) on host buffers."""
    q_off = np.ascontiguousarray(q_off, dtype=np.uint32)
    q_terms = np.ascontiguousarray(q_terms, dtype=np.uint32)
    nq = len(q_off) - 1
    if out is None:
        out = _result_arrays(nq, max(int(k), 1), want_f64, want_payload)
    al = np.ascontiguousarray(allow, dtype=np.uint8) if allow is not None else None
    st = SearchStats()
    _check(fn(h, nq, _p(q_off, C.c_uint32), _p(q_terms, C.c_uint32), int(k), _p(al, C.c_uint8), *_rows_args(out),
              C.byref(st)))
    out["stats"] = st
    return out


def _search_candidates(fn, h, q_off, q_terms, c_off, c_docs, k, want_f64, want_payload):
    """bm25x_search_candidates or its sharded / growing form (the same signature) on host buffers."""
    q_off = np.ascontiguousarray(q_off, dtype=np.uint32)
    q_terms = np.ascontiguousarray(q_terms, dtype=np.uint32)
    c_off = np.ascontiguousarray(c_off, dtype=np.uint32)
    c_docs = np.ascontiguousarray(c_docs, dtype=np.uint32)
    nq = len(q_off) - 1
    out = _result_arrays(nq, max(int(k), 1), want_f64, want_payload)
    st = SearchStats()
    _check(fn(h, nq, _p(q_off, C.c_uint32), _p(q_terms, C.c_uint32), _p(c_off, C.c_uint32), _p(c_docs, C.c_uint32),
              int(k), *_rows_args(out), C.byref(st)))
    out["stats"] = st
    return out


def check_vectors(off, terms, tfs=None):
    """bm25x_check_vectors: the Document / Query invariants of crates/bm25/src/vector.rs:46-134 for n vectors in CSR form
    (keys strictly ascending, tfs non-zero); raises Bm25xError(1, "invalid data: ...")."""
    off = np.ascontiguousarray(off, dtype=np.uint32)
    terms = np.ascontiguousarray(terms, dtype=np.uint32)
    tfs = np.ascontiguousarray(tfs, dtype=np.uint32) if tfs is not None else None
    _check(load_library().bm25x_check_vectors(len(off) - 1, _p(off, C.c_uint32), _p(terms, C.c_uint32), _p(tfs, C.c_uint32)))


def device_count() -> int:
    return load_library().bm25x_device_count()


class Document:
    """crates/bm25/src/vector.rs:46-98 `Document`: strictly ascending term ordinals with tf != 0."""

    def __init__(self, terms, tfs):
        self.terms = np.ascontiguousarray(terms, dtype=np.uint32)
        self.tfs = np.ascontiguousarray(tfs, dtype=np.uint32)
        if len(self.terms) != len(self.tfs) or np.any(np.diff(self.terms.astype(np.int64)) <= 0) or np.any(self.tfs == 0):
            raise ValueError("invalid data")  # Document::new → expect("invalid data")

    def length(self) -> int:
        return int(min(int(self.tfs.astype(np.uint64).sum()), 0xFFFFFFFF))


class Query:
    """crates/bm25/src/vector.rs:100-134 `Query`: strictly ascending term ordinals."""

    def __init__(self, terms):
        self.terms = np.ascontiguousarray(terms, dtype=np.uint32)
        if np.any(np.diff(self.terms.astype(np.int64)) <= 0):
            raise ValueError("invalid data")


class SyntheticCorpus:
    """Host CSR owned by libbm25x (malloc); numpy views without copying (10 GB at the 10M-doc config)."""

    def __init__(self, raw: _Synth):
        self._raw = raw
        self.n_docs, self.n_terms, self.n_postings = raw.n_docs, raw.n_terms, raw.n_postings
        self.doc_len = np.ctypeslib.as_array(raw.doc_len, shape=(raw.n_docs,))
        self.post_off = np.ctypeslib.as_array(raw.post_off, shape=(raw.n_terms + 1,))
        n = max(int(raw.n_postings), 1)
        self.post_doc = np.ctypeslib.as_array(raw.post_doc, shape=(n,))[:raw.n_postings]
        self.post_tf = np.ctypeslib.as_array(raw.post_tf, shape=(n,))[:raw.n_postings]
        self.k1, self.b = 1.2, 0.75

    def free(self):
        if self._raw is not None:
            self.doc_len = self.post_off = self.post_doc = self.post_tf = None
            load_library().bm25x_synth_free(C.byref(self._raw))
            self._raw = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def synth_corpus(seed, n_docs, vocab, len_min, len_max=None, zipf_s=0.0, nthreads=0) -> SyntheticCorpus:
    raw = _Synth()
    _check(load_library().bm25x_synth_generate(seed, n_docs, vocab, len_min, len_min if len_max is None else len_max,
                                               float(zipf_s), nthreads, C.byref(raw)))
    return SyntheticCorpus(raw)


def synth_queries(seed, nq, vocab, n_min, n_max, post_off, zipf_s=0.0):
    post_off = np.ascontiguousarray(post_off, dtype=np.uint64)
    q_off = np.zeros(nq + 1, dtype=np.uint32)
    q_terms = np.zeros(nq * n_max, dtype=np.uint32)
    _check(load_library().bm25x_synth_queries(seed, nq, vocab, n_min, n_max, float(zipf_s), _p(post_off, C.c_uint64),
                                              _p(q_off, C.c_uint32), _p(q_terms, C.c_uint32)))
    return q_off, q_terms[:q_off[-1]].copy()


class Index:
    """Sealed-segment index resident in one GPU's HBM (bm25x_index_*)."""

    def __init__(self, n_docs, doc_len, n_terms, post_off, post_doc, post_tf, k1=1.2, b=0.75, payload=None,
                 term_keys=None, device=0):
        keep = []
        c = _corpus(keep, n_docs, doc_len, n_terms, post_off, post_doc, post_tf, k1, b, payload, term_keys)
        h = C.c_void_p()
        _check(load_library().bm25x_index_create(C.byref(c), device, C.byref(h)))
        self.h, self._keep = h, None  # the library copied everything to the device
        self.n_docs, self.n_terms = int(n_docs), int(n_terms)

    @classmethod
    def from_blocks(cls, n_docs, n_terms, term_blk_off, blk_min_doc, blk_n, blk_meta_doc, blk_meta_tf, blk_doc_off,
                    blk_tf_off, data, doc_len=None, doc_fieldnorm=None, sum_doc_len=0, k1=1.2, b=0.75, payload=None,
                    term_keys=None, device=0, blk_wand_fieldnorm=None, blk_wand_tf=None) -> "Index":
        """Index from the sealed segment as the reference stores it: per-token chains of 128-posting blocks in the
        codec of compression.rs, decoded on the GPU (bm25x_index_create_from_blocks).  Document norms come either from
        exact lengths (`doc_len`) or, as on the pages, from `doc_fieldnorm` + `sum_doc_len`."""
        keep = []
        c = _blocks(keep, n_docs, n_terms, term_blk_off, blk_min_doc, blk_n, blk_meta_doc, blk_meta_tf, blk_doc_off,
                    blk_tf_off, data, doc_len, doc_fieldnorm, sum_doc_len, k1, b, payload, term_keys, blk_wand_fieldnorm,
                    blk_wand_tf)
        h = C.c_void_p()
        _check(load_library().bm25x_index_create_from_blocks(C.byref(c), device, C.byref(h)))
        return cls._adopt(h, n_docs, n_terms)

    @classmethod
    def from_documents(cls, elem_off, elem_tf, *, elem_term=None, elem_key=None, n_terms=0, payload=None, k1=1.2, b=0.75,
                       device=0) -> "Index":
        """Index from documents in heap-scan order (doc id = position), inverted on the GPU
        (bm25x_index_create_from_documents): document d holds elements elem_off[d]..elem_off[d+1], each a term and its tf,
        strictly ascending by term.  Exactly one of elem_term (ordinals < n_terms: keyless) or elem_key ([E, 16] keys:
        keyed, the vocabulary is the distinct keys ascending).  The handle equals Index() on the reference's Segment of the
        same documents."""
        keep = []
        c = _documents(keep, elem_off, elem_tf, elem_term, elem_key, n_terms, payload, k1, b)
        h = C.c_void_p()
        _check(load_library().bm25x_index_create_from_documents(C.byref(c), device, C.byref(h)))
        info = IndexInfo()
        _check(load_library().bm25x_index_get_info(h, C.byref(info)))
        return cls._adopt(h, info.n_docs, info.n_terms)

    @classmethod
    def from_tsvectors(cls, seed, ent_off, entries, byte_off, data, *, payload=None, k1=1.2, b=0.75, device=0) -> "Index":
        """CREATE INDEX from tsvectors (bm25x_index_create_from_tsvectors): the index from_documents builds from the keyed
        documents of the document cast (doc id = position), the cast and the inversion on the GPU without the keys
        coming to the host.  The tsvectors as cast_tsvectors takes them."""
        keep = []
        t = _tsvectors(keep, ent_off, entries, byte_off, data)
        pay = _kept(keep, payload, np.uint16, C.c_uint16) if payload is not None else None
        h = C.c_void_p()
        _check(load_library().bm25x_index_create_from_tsvectors(C.byref(t), _seed(seed), pay, float(k1), float(b),
                                                                device, C.byref(h)))
        info = IndexInfo()
        _check(load_library().bm25x_index_get_info(h, C.byref(info)))
        return cls._adopt(h, info.n_docs, info.n_terms)

    @classmethod
    def _adopt(cls, handle, n_docs, n_terms):
        self = cls.__new__(cls)
        self.h, self._keep, self.n_docs, self.n_terms = handle, None, int(n_docs), int(n_terms)
        return self

    def export_blocks(self, doc_fieldnorm=True, payload=True, term_keys=False):
        """This index as the reference's stored segment, encoded on its GPU (bm25x_index_export_blocks).  Returns
        (args, extra): `Index.from_blocks(**args)` rebuilds the index (stored-norm form, SummaryTuple wand pairs included);
        extra holds the rest of what flush writes: blk_max_doc and the TokenTuple fields tok_df, tok_wand_fieldnorm,
        tok_wand_tf.  doc_fieldnorm / payload = False skip the per-document outputs (None in args); term_keys = True
        exports the keys (refused on an index without them)."""
        L = load_library()
        info = self.info()
        N, T, NB = int(info.n_docs), int(info.n_terms), int(info.n_blocks)
        e = Export()
        # sizing call: it runs the directory pass that the export runs again (about 17 ms at 10M blocks on an H100)
        _check(L.bm25x_index_export_blocks(self.h, C.byref(e)))
        a = {"n_docs": N, "n_terms": T, "term_blk_off": np.empty(T + 1, np.uint64),
             "blk_min_doc": np.empty(NB, np.uint32), "blk_n": np.empty(NB, np.uint32),
             "blk_meta_doc": np.empty(NB, np.uint8), "blk_meta_tf": np.empty(NB, np.uint8),
             "blk_doc_off": np.empty(NB, np.uint64), "blk_tf_off": np.empty(NB, np.uint64),
             "data": np.empty(max(int(e.n_bytes), 1), np.uint8)[:int(e.n_bytes)], "doc_fieldnorm": np.empty(N, np.uint8) if doc_fieldnorm else None,
             "sum_doc_len": 0, "k1": float(info.k1), "b": float(info.b),
             "payload": np.empty(N * 3, np.uint16) if payload else None,
             "term_keys": np.empty((T, 16), np.uint8) if term_keys else None,
             "blk_wand_fieldnorm": np.empty(NB, np.uint8), "blk_wand_tf": np.empty(NB, np.uint32)}
        x = {"blk_max_doc": np.empty(NB, np.uint32), "tok_df": np.empty(T, np.uint32),
             "tok_wand_fieldnorm": np.empty(T, np.uint8), "tok_wand_tf": np.empty(T, np.uint32)}
        e = Export()
        outputs = {"doc_fieldnorm": a["doc_fieldnorm"], "payload": a["payload"], "term_key": a["term_keys"],
                   "tok_df": x["tok_df"], "tok_wand_fieldnorm": x["tok_wand_fieldnorm"], "tok_wand_tf": x["tok_wand_tf"],
                   "term_blk_off": a["term_blk_off"], "blk_min_doc": a["blk_min_doc"], "blk_max_doc": x["blk_max_doc"],
                   "blk_n": a["blk_n"], "blk_meta_doc": a["blk_meta_doc"], "blk_meta_tf": a["blk_meta_tf"],
                   "blk_doc_off": a["blk_doc_off"], "blk_tf_off": a["blk_tf_off"],
                   "blk_wand_fieldnorm": a["blk_wand_fieldnorm"], "blk_wand_tf": a["blk_wand_tf"], "bytes": a["data"]}
        for name, arr in outputs.items():   # a None array stays a NULL pointer: not written
            if arr is not None:
                setattr(e, name, arr.ctypes.data_as(dict(Export._fields_)[name]))
        e.bytes_cap = len(a["data"])
        _check(L.bm25x_index_export_blocks(self.h, C.byref(e)))
        a["sum_doc_len"] = int(e.sum_doc_len)
        return a, x

    def layout(self) -> IndexLayout:
        out = IndexLayout()
        _check(load_library().bm25x_index_get_layout(self.h, C.byref(out)))
        return out

    @classmethod
    def alloc_replica(cls, like: IndexLayout, device: int) -> "Index":
        """Empty index of the same shape on `device`; fill the arrays of .layout() (e.g. by NCCL broadcast), then
        call finalize_replica()."""
        h = C.c_void_p()
        _check(load_library().bm25x_index_alloc_replica(C.byref(like), device, C.byref(h)))
        return cls._adopt(h, like.n_docs, like.n_terms)

    def finalize_replica(self):
        _check(load_library().bm25x_index_finalize_replica(self.h))

    def derived(self) -> IndexDerived:
        """Test hook: the doc-id copy, champion lists and s1f_min this handle built on its device (never replicated)."""
        out = IndexDerived()
        _check(load_library().bm25x_index_get_derived(self.h, C.byref(out)))
        return out

    def set_option(self, name: str, value: int):
        _check(load_library().bm25x_index_set_option(self.h, name.encode(), int(value)))

    def df(self):
        out = np.zeros(self.n_terms, np.uint32)
        _check(load_library().bm25x_index_get_df(self.h, _p(out, C.c_uint32)))
        return out

    @staticmethod
    def from_corpus(c, device=0, **kw):
        return Index(c.n_docs, c.doc_len, c.n_terms, c.post_off, c.post_doc, c.post_tf, getattr(c, "k1", 1.2),
                     getattr(c, "b", 0.75), device=device, **kw)

    def close(self):
        if getattr(self, "h", None):
            load_library().bm25x_index_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def info(self) -> IndexInfo:
        out = IndexInfo()
        _check(load_library().bm25x_index_get_info(self.h, C.byref(out)))
        return out

    def lookup_terms(self, keys):
        keys = np.ascontiguousarray(keys, dtype=np.uint8).reshape(-1, 16)
        out = np.zeros(len(keys), dtype=np.uint32)
        _check(load_library().bm25x_lookup_terms(self.h, _p(keys, C.c_uint8), len(keys), _p(out, C.c_uint32)))
        return out

    def tsvector_queries(self, seed, ent_off, entries, byte_off, data):
        """Queries from tsvectors (bm25x_tsvector_queries): the query cast of each vector and its keys' ordinals in
        this index's vocabulary (TERM_MISSING when absent), on the GPU.  Returns (q_off, q_terms) as search_batch and
        search_candidates take them."""
        keep = []
        t = _tsvectors(keep, ent_off, entries, byte_off, data)
        E = int(keep[0][-1]) if len(keep[0]) else 0
        q_off = np.zeros(t.n + 1, np.uint32)
        q_terms = np.zeros(max(E, 1), np.uint32)
        _check(load_library().bm25x_tsvector_queries(self.h, _seed(seed), C.byref(t), _p(q_off, C.c_uint32),
                                                     _p(q_terms, C.c_uint32)))
        return q_off, q_terms[:int(q_off[-1])].copy()

    # ---- bm25::search for a batch (host buffers in, host buffers out) ----
    def search_batch(self, q_off, q_terms, k, allow=None, want_f64=True, want_payload=False, out=None):
        return _search_batch(load_library().bm25x_search_batch, self.h, q_off, q_terms, k, allow, want_f64, want_payload,
                             out)

    def search_candidates(self, q_off, q_terms, c_off, c_docs, k, want_f64=True, want_payload=False):
        """Per-query candidate lists (bm25x_search_candidates): query i's top-k over the doc ids
        c_docs[c_off[i]:c_off[i+1]] (any order, duplicates counted once) — the rows search_batch returns for query i alone
        with allow = the bitmap of its candidates.  Returns what search_batch returns."""
        return _search_candidates(load_library().bm25x_search_candidates, self.h, q_off, q_terms, c_off, c_docs, k,
                                  want_f64, want_payload)

    def search(self, query, k, allow=None):
        """One query, the shape of bm25::search(&index, k, &query, filter): [(score f64, doc id)] best first."""
        terms = query.terms if isinstance(query, Query) else np.asarray(query, dtype=np.uint32)
        r = self.search_batch(np.array([0, len(terms)], np.uint32), terms, k, allow=allow)
        n = int(r["n"][0])
        return r["doc"][0, :n].copy(), r["score64"][0, :n].copy()

    # ---- growing segment (documents inserted since the last seal; search.rs:83-135) ----
    def growing(self, elem_off, elem_term, elem_tf, doc_len=None, doc_fieldnorm=None, payload=None,
                deleted=None) -> "Index":
        """Handle over the growing documents (doc-major: document g holds elements elem_off[g]..elem_off[g+1], term
        ordinals of THIS sealed index ascending, TERM_MISSING for tokens it does not know) that scores with this
        index's statistics (bm25x_growing_create).  Search it like any index; ids are growing ordinals."""
        keep = []
        g = _growing_docs(keep, elem_off, elem_term, elem_tf, doc_len, doc_fieldnorm, payload, deleted)
        h = C.c_void_p()
        _check(load_library().bm25x_growing_create(self.h, C.byref(g), C.byref(h)))
        return Index._adopt(h, g.n_docs, self.n_terms)

    def growing_segment(self) -> "GrowingSegment":
        """An empty mutable growing segment on this index's device (bm25x_growing_open): insert / delete in place,
        search sealed + growing in one call.  This index must stay open while the segment is."""
        return GrowingSegment(self)

    def search_batch_growing(self, growing, q_off, q_terms, k, allow=None, allow_growing=None, want_payload=False):
        """bm25::search over this sealed index + a growing handle (None = sealed only): ids >= n_docs are growing
        ordinal + n_docs."""
        q_off = np.ascontiguousarray(q_off, dtype=np.uint32)
        q_terms = np.ascontiguousarray(q_terms, dtype=np.uint32)
        nq, kk = len(q_off) - 1, int(k)
        out = _result_arrays(nq, kk, True, want_payload)
        al = np.ascontiguousarray(allow, dtype=np.uint8) if allow is not None else None
        alg = np.ascontiguousarray(allow_growing, dtype=np.uint8) if allow_growing is not None else None
        st = SearchStats()
        _check(load_library().bm25x_search_batch_growing(
            self.h, growing.h if growing is not None else None, nq, _p(q_off, C.c_uint32), _p(q_terms, C.c_uint32), kk,
            _p(al, C.c_uint8), _p(alg, C.c_uint8), *_rows_args(out), C.byref(st)))
        out["stats"] = st
        return out

    def prepare(self, q_off, q_terms, k, allow=None) -> "Batch":
        return Batch(self, q_off, q_terms, k, allow)

    # ---- bm25::evaluate for a batch of (document, query) pairs ----
    def evaluate_batch(self, docs, queries):
        return _evaluate_batch(load_library().bm25x_evaluate_batch, self.h, docs, queries)

    def evaluate(self, document: Document, query: Query) -> float:
        return float(self.evaluate_batch([document], [query])[0])

    def evaluate_tsvectors(self, seed, docs, queries, pair_query=None):
        """`<&>` from tsvectors (bm25x_evaluate_tsvectors): out[p] = bm25::evaluate of document tsvector p against query
        tsvector pair_query[p] (p when None), both cast on the GPU against this index's keys."""
        return _evaluate_tsvectors(load_library().bm25x_evaluate_tsvectors, self.h, seed, docs, queries, pair_query)


def _evaluate_batch(fn, h, docs, queries):
    """bm25x_evaluate_batch or its sharded form (the same signature) on lists of Document and Query."""
    d_off = np.zeros(len(docs) + 1, np.uint32)
    q_off = np.zeros(len(docs) + 1, np.uint32)
    for i, (d, q) in enumerate(zip(docs, queries)):
        d_off[i + 1] = d_off[i] + len(d.terms)
        q_off[i + 1] = q_off[i] + len(q.terms)
    cat = lambda xs: np.ascontiguousarray(np.concatenate(xs) if xs else np.zeros(0), dtype=np.uint32)
    d_terms, d_tfs, q_terms = cat([d.terms for d in docs]), cat([d.tfs for d in docs]), cat([q.terms for q in queries])
    out = np.zeros(len(docs), np.float64)
    _check(fn(h, len(docs), _p(d_off, C.c_uint32), _p(d_terms, C.c_uint32), _p(d_tfs, C.c_uint32),
              _p(q_off, C.c_uint32), _p(q_terms, C.c_uint32), _p(out, C.c_double)))
    return out


def _evaluate_tsvectors(fn, h, seed, docs, queries, pair_query):
    """bm25x_evaluate_tsvectors or its sharded form.  docs, queries: tsvector batches, each a dict of the arguments
    cast_tsvectors takes (ent_off, entries, byte_off, data); pair_query: u32 [docs n] or None."""
    keep = []
    d = _tsvectors(keep, **docs)
    q = _tsvectors(keep, **queries)
    pq = None if pair_query is None else _kept(keep, pair_query, np.uint32, C.c_uint32)
    out = np.zeros(max(d.n, 1), np.float64)
    _check(fn(h, _seed(seed), C.byref(d), C.byref(q), pq, _p(out, C.c_double)))
    return out[:d.n]


def _growing_docs(keep, elem_off, elem_term, elem_tf, doc_len, doc_fieldnorm, payload, deleted):
    g = _GrowingDocs()
    g.elem_off = _kept(keep, elem_off, np.uint64, C.c_uint64)
    g.n_docs = len(keep[-1]) - 1
    g.elem_term = _kept(keep, elem_term, np.uint32, C.c_uint32)
    g.elem_tf = _kept(keep, elem_tf, np.uint32, C.c_uint32)
    if doc_len is not None:
        g.doc_len = _kept(keep, doc_len, np.uint32, C.c_uint32)
    if doc_fieldnorm is not None:
        g.doc_fieldnorm = _kept(keep, doc_fieldnorm, np.uint8, C.c_uint8)
    if payload is not None:
        g.payload = _kept(keep, payload, np.uint16, C.c_uint16)
    if deleted is not None:
        g.deleted = _kept(keep, deleted, np.uint8, C.c_uint8)
    return g


class GrowingSegment:
    """The growing segment as the library keeps it (bm25x_growing_*): documents inserted and deleted in place, indexed on
    the sealed index's device by a refresh, searched together with the sealed index.  Growing ordinal o comes back as
    doc id sealed.n_docs + o.  The sealed side is an Index or a ShardedIndex (bm25x_growing_open_sharded: the segment
    lives on the last shard's device, ids and allow_sealed are global)."""

    def __init__(self, sealed):
        self.sealed = sealed
        self.sharded = isinstance(sealed, ShardedIndex)
        self.h = C.c_void_p()
        L = load_library()
        _check((L.bm25x_growing_open_sharded if self.sharded else L.bm25x_growing_open)(sealed.h, C.byref(self.h)))

    def insert(self, elem_off, elem_term, elem_tf, doc_len=None, doc_fieldnorm=None, payload=None, deleted=None):
        """Appends documents, arguments as Index.growing (bm25x_growing_insert)."""
        keep = []
        g = _growing_docs(keep, elem_off, elem_term, elem_tf, doc_len, doc_fieldnorm, payload, deleted)
        _check(load_library().bm25x_growing_insert(self.h, C.byref(g)))

    def insert_tsvectors(self, seed, ent_off, entries, byte_off, data, payload=None):
        """aminsert of tsvectors (bm25x_growing_insert_tsvectors): each vector cast on the GPU and appended as the next
        ordinal; keys the sealed vocabulary lacks are numbered by the segment (new_keys) and keyed by the seal.  The
        tsvectors as cast_tsvectors takes them; payload [n, 3] ctids or None."""
        keep = []
        t = _tsvectors(keep, ent_off, entries, byte_off, data)
        pay = _kept(keep, payload, np.uint16, C.c_uint16) if payload is not None else None
        _check(load_library().bm25x_growing_insert_tsvectors(self.h, _seed(seed), C.byref(t), pay))

    def new_keys(self):
        """The keys the segment numbered (bm25x_growing_get_new_keys): uint8 [K, 16], row i the key of token ordinal
        sealed.n_terms + i."""
        L = load_library()
        n = C.c_uint32()
        while True:  # tsvector inserts may add keys between the sizing call and the copy
            keys = np.zeros((max(n.value, 1), 16), np.uint8)
            cap = n.value
            rc = L.bm25x_growing_get_new_keys(self.h, cap, _p(keys, C.c_uint8), C.byref(n))
            if rc != 0 and n.value > cap:
                continue
            _check(rc)
            return keys[:n.value].copy()

    def tsvector_queries(self, seed, ent_off, entries, byte_off, data):
        """Queries from tsvectors for this segment's searches (bm25x_growing_tsvector_queries), shaped as
        Index.tsvector_queries: ordinals of the sealed vocabulary, TERM_MISSING for every other key (the segment's own
        included, until the seal)."""
        keep = []
        t = _tsvectors(keep, ent_off, entries, byte_off, data)
        E = int(keep[0][-1]) if len(keep[0]) else 0
        q_off = np.zeros(t.n + 1, np.uint32)
        q_terms = np.zeros(max(E, 1), np.uint32)
        _check(load_library().bm25x_growing_tsvector_queries(self.h, _seed(seed), C.byref(t), _p(q_off, C.c_uint32),
                                                             _p(q_terms, C.c_uint32)))
        return q_off, q_terms[:int(q_off[-1])].copy()

    def delete(self, ordinals):
        o = np.ascontiguousarray(ordinals, dtype=np.uint32)
        _check(load_library().bm25x_growing_delete(self.h, len(o), _p(o, C.c_uint32)))

    def refresh(self):
        _check(load_library().bm25x_growing_refresh(self.h))

    def info(self) -> GrowingInfo:
        out = GrowingInfo()
        _check(load_library().bm25x_growing_get_info(self.h, C.byref(out)))
        return out

    def arrays(self):
        """Test hook: (IndexLayout, IndexDerived) of the segment's current handle (bm25x_growing_get_index)."""
        lay, der = IndexLayout(), IndexDerived()
        _check(load_library().bm25x_growing_get_index(self.h, C.byref(lay), C.byref(der)))
        return lay, der

    def search_batch(self, q_off, q_terms, k, allow=None, allow_growing=None, allow_growing_docs=None,
                     want_payload=False):
        """Sealed + growing, the rows of Index.search_batch_growing.  allow_growing covers the ordinals
        [0, allow_growing_docs) (default: 8 x its length)."""
        q_off = np.ascontiguousarray(q_off, dtype=np.uint32)
        q_terms = np.ascontiguousarray(q_terms, dtype=np.uint32)
        nq, kk = len(q_off) - 1, int(k)
        out = _result_arrays(nq, max(kk, 1), True, want_payload)
        al = np.ascontiguousarray(allow, dtype=np.uint8) if allow is not None else None
        alg = np.ascontiguousarray(allow_growing, dtype=np.uint8) if allow_growing is not None else None
        n_alg = (8 * len(alg) if allow_growing_docs is None else int(allow_growing_docs)) if alg is not None else 0
        st = SearchStats()
        _check(load_library().bm25x_growing_search_batch(
            self.h, nq, _p(q_off, C.c_uint32), _p(q_terms, C.c_uint32), kk, _p(al, C.c_uint8), _p(alg, C.c_uint8), n_alg,
            *_rows_args(out), C.byref(st)))
        out["stats"] = st
        return out

    def search_candidates(self, q_off, q_terms, c_off, c_docs, k, want_f64=True, want_payload=False):
        """Index.search_candidates over sealed + growing (bm25x_growing_search_candidates): candidate ids in the result
        id space, growing ordinal o as sealed.n_docs + o."""
        return _search_candidates(load_library().bm25x_growing_search_candidates, self.h, q_off, q_terms, c_off, c_docs,
                                  k, want_f64, want_payload)

    def seal(self, sealed_deleted=None, new_keys=None):
        """`maintain` (bm25x_growing_seal): a new sealed Index of the surviving sealed documents (ascending old id) and
        the surviving growing ones (ascending ordinal).  sealed_deleted: bitmap over sealed ids, the layout of `allow`;
        new_keys: keyed index only, [n, 16] keys of the token ordinals sealed.n_terms + i.  Returns (index, sealed_map,
        growing_map, term_map): new id of each sealed id / growing ordinal (0xFFFFFFFF: deleted) and new ordinal of each
        source term (TERM_MISSING: vanished); growing_map covers the ordinals the seal took, which may be fewer than
        info().n_docs when other threads insert meanwhile.  The segment and this sealed index stay as they are.  Over a
        ShardedIndex (bm25x_growing_seal_sharded) the index returned is a new ShardedIndex and the ids are global."""
        L = load_library()
        dele = np.ascontiguousarray(sealed_deleted, dtype=np.uint8) if sealed_deleted is not None else None
        keys = np.ascontiguousarray(new_keys, dtype=np.uint8).reshape(-1, 16) if new_keys is not None else None
        n_keys = len(keys) if keys is not None else 0
        smap = np.empty(self.sealed.n_docs, np.uint32)
        g_cap, t_cap = int(self.info().n_docs), self.sealed.n_terms + n_keys
        while True:  # a cap below what the seal writes is refused with the sizes it needs (inserts may run meanwhile)
            gmap, tmap = np.empty(max(g_cap, 1), np.uint32), np.empty(max(t_cap, 1), np.uint32)
            a = SealArgs()
            a.sealed_deleted, a.new_keys, a.n_new_keys = _p(dele, C.c_uint8), _p(keys, C.c_uint8), n_keys
            a.sealed_map = _p(smap, C.c_uint32)
            a.growing_map, a.growing_cap = _p(gmap, C.c_uint32), g_cap
            a.term_map, a.term_cap = _p(tmap, C.c_uint32), t_cap
            h = C.c_void_p()
            rc = (L.bm25x_growing_seal_sharded if self.sharded else L.bm25x_growing_seal)(self.h, C.byref(a), C.byref(h))
            if rc != 0 and (a.n_growing > g_cap or a.n_source_terms > t_cap):
                g_cap, t_cap = max(g_cap, int(a.n_growing)), max(t_cap, int(a.n_source_terms))
                continue
            _check(rc)
            info = IndexInfo()
            if self.sharded:
                _check(L.bm25x_sharded_get_info(h, C.byref(info), None, None))
                ix = ShardedIndex._adopt(h, info.n_docs, info.n_terms)
            else:
                _check(L.bm25x_index_get_info(h, C.byref(info)))
                ix = Index._adopt(h, info.n_docs, info.n_terms)
            return ix, smap, gmap[:a.n_growing].copy(), tmap[:a.n_source_terms].copy()

    def rebind(self, new_index):
        """The segment goes on over new_index, the Index (or ShardedIndex) its latest seal returned
        (bm25x_growing_rebind / _sharded): the ordinals the seal folded in leave it, ordinal n_folded + i becomes i.
        Returns the new ids of the folded documents deleted after the seal's snapshot, ascending (to OR into
        allow_sealed and the next seal's sealed_deleted).  self.sealed then is new_index; the old index may be closed."""
        L = load_library()
        late = np.zeros(max((new_index.n_docs + 7) // 8, 1), np.uint8)
        a = RebindArgs()
        a.late_deleted = _p(late, C.c_uint8)
        call = L.bm25x_growing_rebind_sharded if self.sharded else L.bm25x_growing_rebind
        _check(call(self.h, new_index.h, C.byref(a)))
        self.sealed = new_index
        return np.flatnonzero(np.unpackbits(late, bitorder="little")[:new_index.n_docs]).astype(np.uint32)

    def close(self):
        if getattr(self, "h", None):
            load_library().bm25x_growing_close(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def merge_topk(a, b, doc_base_b, k):
    """Host-only bm25x_merge_topk of two result dicts (as returned by search_batch with f64 scores)."""
    nq = len(a["n"])
    assert a["doc"].shape == (nq, k) and b["doc"].shape == (nq, k)
    pay = a.get("payload") is not None and b.get("payload") is not None
    out = _result_arrays(nq, k, True, pay)
    c = lambda x, dt: np.ascontiguousarray(x, dtype=dt)
    keep = [c(a["doc"], np.uint32), c(a["score"], np.float32), c(a["score64"], np.float64),
            c(a["payload"], np.uint16) if pay else None, c(a["n"], np.uint32),
            c(b["doc"], np.uint32), c(b["score"], np.float32), c(b["score64"], np.float64),
            c(b["payload"], np.uint16) if pay else None, c(b["n"], np.uint32)]
    ty = [C.c_uint32, C.c_float, C.c_double, C.c_uint16, C.c_uint32] * 2
    _check(load_library().bm25x_merge_topk(nq, int(k), *[_p(x, t) for x, t in zip(keep[:5], ty[:5])],
                                           *[_p(x, t) for x, t in zip(keep[5:], ty[5:])], int(doc_base_b),
                                           *_rows_args(out)))
    return out


MAX_SHARDS = 16


class ShardedIndex:
    """One sealed segment split by document range into `n_shards` indexes (bm25x_sharded_*), on one GPU or several, so
    that it need not fit in one GPU's HBM.  Searches return exactly what Index.search_batch returns on the unsharded index
    built from the same corpus: global doc ids, `allow` over global ids."""

    def __init__(self, n_docs, doc_len, n_terms, post_off, post_doc, post_tf, k1=1.2, b=0.75, payload=None,
                 term_keys=None, n_shards=2, doc_bounds=None, devices=None):
        keep = []
        c = _corpus(keep, n_docs, doc_len, n_terms, post_off, post_doc, post_tf, k1, b, payload, term_keys)
        bounds = np.ascontiguousarray(doc_bounds, dtype=np.uint32) if doc_bounds is not None else None
        devs = (C.c_int * int(n_shards))(*[int(d) for d in devices]) if devices is not None else None
        self.h = C.c_void_p()
        _check(load_library().bm25x_sharded_create(C.byref(c), int(n_shards), _p(bounds, C.c_uint32), devs,
                                                   C.byref(self.h)))
        self.n_docs, self.n_terms = int(n_docs), int(n_terms)

    @classmethod
    def from_blocks(cls, n_docs, n_terms, term_blk_off, blk_min_doc, blk_n, blk_meta_doc, blk_meta_tf, blk_doc_off,
                    blk_tf_off, data, doc_len=None, doc_fieldnorm=None, sum_doc_len=0, k1=1.2, b=0.75, payload=None,
                    term_keys=None, blk_wand_fieldnorm=None, blk_wand_tf=None, n_shards=2, doc_bounds=None,
                    devices=None) -> "ShardedIndex":
        """The sharded index from the sealed segment as stored (Index.from_blocks' arguments): the blocks are checked
        once on devices[0], then each shard's device decodes only the stored blocks that hold its documents
        (bm25x_index_create_sharded_from_blocks)."""
        keep = []
        c = _blocks(keep, n_docs, n_terms, term_blk_off, blk_min_doc, blk_n, blk_meta_doc, blk_meta_tf, blk_doc_off,
                    blk_tf_off, data, doc_len, doc_fieldnorm, sum_doc_len, k1, b, payload, term_keys, blk_wand_fieldnorm,
                    blk_wand_tf)
        bounds = np.ascontiguousarray(doc_bounds, dtype=np.uint32) if doc_bounds is not None else None
        devs = (C.c_int * int(n_shards))(*[int(d) for d in devices]) if devices is not None else None
        self = cls.__new__(cls)
        self.h = C.c_void_p()
        _check(load_library().bm25x_index_create_sharded_from_blocks(C.byref(c), int(n_shards), _p(bounds, C.c_uint32),
                                                                     devs, C.byref(self.h)))
        self.n_docs, self.n_terms = int(n_docs), int(n_terms)
        return self

    @classmethod
    def from_documents(cls, elem_off, elem_tf, *, elem_term=None, elem_key=None, n_terms=0, payload=None, k1=1.2, b=0.75,
                       n_shards=2, doc_bounds=None, devices=None) -> "ShardedIndex":
        """The sharded index from documents (Index.from_documents' arguments, bm25x_index_create_sharded_from_documents):
        every shard's device inverts only its own documents' elements.  Equals ShardedIndex() on the Segment's CSR with the
        same n_shards / doc_bounds / devices."""
        keep = []
        c = _documents(keep, elem_off, elem_tf, elem_term, elem_key, n_terms, payload, k1, b)
        bounds = np.ascontiguousarray(doc_bounds, dtype=np.uint32) if doc_bounds is not None else None
        devs = (C.c_int * int(n_shards))(*[int(d) for d in devices]) if devices is not None else None
        h = C.c_void_p()
        _check(load_library().bm25x_index_create_sharded_from_documents(C.byref(c), int(n_shards), _p(bounds, C.c_uint32),
                                                                        devs, C.byref(h)))
        info = IndexInfo()
        _check(load_library().bm25x_sharded_get_info(h, C.byref(info), None, None))
        return cls._adopt(h, info.n_docs, info.n_terms)

    @classmethod
    def from_tsvectors(cls, seed, ent_off, entries, byte_off, data, *, payload=None, k1=1.2, b=0.75, n_shards=2,
                       doc_bounds=None, devices=None) -> "ShardedIndex":
        """The sharded index from tsvectors (Index.from_tsvectors' arguments, bm25x_index_create_sharded_from_tsvectors):
        every shard's device casts only its own tsvectors and the vocabulary is merged from the shards' distinct keys.
        Equals from_documents on the document cast with the same n_shards / devices and the bounds this index reports;
        doc_bounds=None balances the shards by tsvector entries."""
        keep = []
        t = _tsvectors(keep, ent_off, entries, byte_off, data)
        pay = _kept(keep, payload, np.uint16, C.c_uint16) if payload is not None else None
        bounds = np.ascontiguousarray(doc_bounds, dtype=np.uint32) if doc_bounds is not None else None
        devs = (C.c_int * int(n_shards))(*[int(d) for d in devices]) if devices is not None else None
        h = C.c_void_p()
        _check(load_library().bm25x_index_create_sharded_from_tsvectors(C.byref(t), _seed(seed), pay, float(k1), float(b),
                                                                        int(n_shards), _p(bounds, C.c_uint32), devs,
                                                                        C.byref(h)))
        info = IndexInfo()
        _check(load_library().bm25x_sharded_get_info(h, C.byref(info), None, None))
        return cls._adopt(h, info.n_docs, info.n_terms)

    @classmethod
    def _adopt(cls, handle, n_docs, n_terms):
        self = cls.__new__(cls)
        self.h, self.n_docs, self.n_terms = handle, int(n_docs), int(n_terms)
        return self

    def growing_segment(self) -> "GrowingSegment":
        """An empty mutable growing segment over this sharded index, on its last shard's device
        (bm25x_growing_open_sharded); seal() gives a new ShardedIndex.  This index must stay open while the segment is."""
        return GrowingSegment(self)

    @staticmethod
    def from_corpus(c, n_shards=2, doc_bounds=None, devices=None, **kw):
        return ShardedIndex(c.n_docs, c.doc_len, c.n_terms, c.post_off, c.post_doc, c.post_tf, getattr(c, "k1", 1.2),
                            getattr(c, "b", 0.75), n_shards=n_shards, doc_bounds=doc_bounds, devices=devices, **kw)

    def close(self):
        if getattr(self, "h", None):
            load_library().bm25x_sharded_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def info(self) -> IndexInfo:
        out = IndexInfo()
        _check(load_library().bm25x_sharded_get_info(self.h, C.byref(out), None, None))
        return out

    def doc_bounds(self):
        n = C.c_uint32(0)
        _check(load_library().bm25x_sharded_get_info(self.h, C.byref(IndexInfo()), C.byref(n), None))
        out = np.zeros(n.value + 1, np.uint32)
        _check(load_library().bm25x_sharded_get_info(self.h, C.byref(IndexInfo()), None, _p(out, C.c_uint32)))
        return out

    def set_option(self, name: str, value: int):
        _check(load_library().bm25x_sharded_set_option(self.h, name.encode(), int(value)))

    def shard_arrays(self, s: int):
        """Test hook: (IndexLayout, IndexDerived) of shard s, whose handle stays internal (bm25x_sharded_get_shard)."""
        lay, der = IndexLayout(), IndexDerived()
        _check(load_library().bm25x_sharded_get_shard(self.h, int(s), C.byref(lay), C.byref(der)))
        return lay, der

    def lookup_terms(self, keys):
        keys = np.ascontiguousarray(keys, dtype=np.uint8).reshape(-1, 16)
        out = np.zeros(len(keys), dtype=np.uint32)
        _check(load_library().bm25x_sharded_lookup_terms(self.h, _p(keys, C.c_uint8), len(keys), _p(out, C.c_uint32)))
        return out

    def tsvector_queries(self, seed, ent_off, entries, byte_off, data):
        """Index.tsvector_queries on this sharded index (bm25x_tsvector_queries_sharded): the query cast on shard 0's
        device against the segment's keys.  Returns (q_off, q_terms) as search_batch takes them."""
        keep = []
        t = _tsvectors(keep, ent_off, entries, byte_off, data)
        E = int(keep[0][-1]) if len(keep[0]) else 0
        q_off = np.zeros(t.n + 1, np.uint32)
        q_terms = np.zeros(max(E, 1), np.uint32)
        _check(load_library().bm25x_tsvector_queries_sharded(self.h, _seed(seed), C.byref(t), _p(q_off, C.c_uint32),
                                                             _p(q_terms, C.c_uint32)))
        return q_off, q_terms[:int(q_off[-1])].copy()

    def evaluate_batch(self, docs, queries):
        """Index.evaluate_batch with the whole segment's statistics (bm25x_evaluate_batch_sharded)."""
        return _evaluate_batch(load_library().bm25x_evaluate_batch_sharded, self.h, docs, queries)

    def evaluate_tsvectors(self, seed, docs, queries, pair_query=None):
        """Index.evaluate_tsvectors on this sharded index (bm25x_evaluate_tsvectors_sharded), on shard 0's device."""
        return _evaluate_tsvectors(load_library().bm25x_evaluate_tsvectors_sharded, self.h, seed, docs, queries,
                                   pair_query)

    def search_batch(self, q_off, q_terms, k, allow=None, want_f64=True, want_payload=False, out=None):
        return _search_batch(load_library().bm25x_sharded_search_batch, self.h, q_off, q_terms, k, allow, want_f64,
                             want_payload, out)

    def search_candidates(self, q_off, q_terms, c_off, c_docs, k, want_f64=True, want_payload=False):
        """Index.search_candidates with global ids (bm25x_search_candidates_sharded)."""
        return _search_candidates(load_library().bm25x_search_candidates_sharded, self.h, q_off, q_terms, c_off, c_docs,
                                  k, want_f64, want_payload)


def merge_shards(rows, doc_base, k, device=0):
    """bm25x_merge_shards: the device merge alone on host rows.  rows = list of S result dicts (doc, score, score64,
    payload [nq, k(, 3)] with local ids, n [nq]); returns the merged dict and the kernel's time in ms."""
    S, nq = len(rows), len(rows[0]["n"])
    cat = lambda key, dt: np.ascontiguousarray(np.stack([r[key] for r in rows]), dtype=dt)
    doc, sc, s64, pay, n = (cat("doc", np.uint32), cat("score", np.float32), cat("score64", np.float64),
                            cat("payload", np.uint16), cat("n", np.uint32))
    base = np.ascontiguousarray(doc_base, dtype=np.uint32)
    out = _result_arrays(nq, int(k), True, True)
    ms = C.c_float(0.0)
    _check(load_library().bm25x_merge_shards(int(device), S, nq, int(k), _p(base, C.c_uint32), _p(doc, C.c_uint32),
                                             _p(sc, C.c_float), _p(s64, C.c_double), _p(pay, C.c_uint16),
                                             _p(n, C.c_uint32), *_rows_args(out), C.byref(ms)))
    return out, ms.value


class Batch:
    """Split form: prepare (canonicalise + upload) / run (kernels only, inputs resident in HBM) / fetch (D2H)."""

    def __init__(self, index: Index, q_off, q_terms, k, allow=None):
        self.index = index
        q_off = np.ascontiguousarray(q_off, dtype=np.uint32)
        q_terms = np.ascontiguousarray(q_terms, dtype=np.uint32)
        self.nq, self.k = len(q_off) - 1, int(k)
        al = np.ascontiguousarray(allow, dtype=np.uint8) if allow is not None else None
        h = C.c_void_p()
        _check(load_library().bm25x_batch_prepare(index.h, self.nq, _p(q_off, C.c_uint32), _p(q_terms, C.c_uint32),
                                                  self.k, _p(al, C.c_uint8), C.byref(h)))
        self.h = h

    def run(self, stream=None, timed=True):
        st = SearchStats()
        _check(load_library().bm25x_batch_run(self.h, C.c_void_p(stream) if stream else None,
                                              C.byref(st) if timed else None))
        return st

    def fetch(self, want_f64=True, want_payload=False):
        out = _result_arrays(self.nq, self.k, want_f64, want_payload)
        _check(load_library().bm25x_batch_fetch(self.h, *_rows_args(out)))
        return out

    def device_results(self):
        """Raw device addresses of the result rows: {"doc": (ptr, nbytes), "score": ..., "score64": ..., "n": ...}
        (bm25x_batch_device_results) — for GPU → GPU transport of sharded results (shard.py)."""
        p = [C.c_void_p() for _ in range(5)]
        _check(load_library().bm25x_batch_device_results(self.h, *[C.byref(x) for x in p]))
        slots = self.nq * self.k
        return {"doc": (p[0].value, 4 * slots), "score": (p[1].value, 4 * slots), "score64": (p[2].value, 8 * slots),
                "payload": (p[3].value, 6 * slots), "n": (p[4].value, 4 * self.nq)}

    def close(self):
        if getattr(self, "h", None):
            load_library().bm25x_batch_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Broker:
    """Batching broker (include/bm25x_broker.h): concurrent single-query callers, one backend call per batch.
    Broker(index) batches into bm25x_search_batch; Broker(backend=callable) into any function of the backend signature
    (the callable receives raw ctypes pointers)."""

    def __init__(self, index=None, backend=None, max_batch=0, max_wait_us=0, ring_slots=0):
        L = load_library()
        opt = BrokerOptions(max_batch, max_wait_us, ring_slots, 0)
        self.h = C.c_void_p()
        self._keep = None
        if backend is not None:
            self._keep = BROKER_BACKEND(backend)
            _check(L.bm25x_broker_create_with_backend(self._keep, None, C.byref(opt), C.byref(self.h)))
        else:
            self._keep = index
            _check(L.bm25x_broker_create(index.h, C.byref(opt), C.byref(self.h)))

    def search(self, terms, k, want_payload=False):
        terms = np.ascontiguousarray(terms, dtype=np.uint32)
        kk = max(int(k), 1)
        doc, s64, n = np.empty(kk, np.uint32), np.empty(kk, np.float64), C.c_uint32(0)
        pay = np.empty((kk, 3), np.uint16) if want_payload else None
        _check(load_library().bm25x_broker_search(self.h, _p(terms, C.c_uint32), len(terms), int(k), _p(doc, C.c_uint32),
                                                  _p(s64, C.c_double), _p(pay, C.c_uint16), C.byref(n)))
        return (doc[:n.value], s64[:n.value]) + ((pay[:n.value],) if want_payload else ())

    def stats(self) -> BrokerStats:
        st = BrokerStats()
        _check(load_library().bm25x_broker_get_stats(self.h, C.byref(st)))
        return st

    def close(self):
        if self.h:
            load_library().bm25x_broker_destroy(self.h)
            self.h = C.c_void_p()
