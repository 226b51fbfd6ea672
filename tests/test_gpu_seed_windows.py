"""GPU: the seeded kernel's seeds where they meet its doc windows (RING_SEEDED, bm25x_search_ring.cuh).  A document that
holds one query term reaches the top k only as one of that term's seeds, so every seed must be listed once, in the
window that holds its doc id; a seed dropped, listed twice or left over from the previous query gives a wrong row that
no filter catches.  Each corpus is built from the CPU model of tests/util_seeds.py, and test_seed_windows.py asserts on
the CPU that each case reaches its branch:

  full slices   every term's 32 champions in one window, listed in one step at k <= 32 (256 seeds in the 8-lane class);
                champions held by no other query term (each enters alone) or by another one (the stream's business).
  list full     k = 33 .. 128 around the slice counts: the listing of one window pauses for verification passes inside
                a term's slices and between two terms, and resumes; the last term's seeds are the top rows.
  window edges  seeds on lo, hi - 1 and hi of a window another run bounds, in the last window (hi = INF, the last
                document) and of a term whose whole list lands in the first round.
  slot reset    thousands of queries per class (more than the launch's resident warps), alternately of terms with full
                champion lists and of terms with fewer postings than k: a seed slot left over from the previous query
                of a warp would be listed in the next one's windows.

Every case runs on the seeded kernel with nothing handed back (checked with the launch's hand-back test) and on the plain
kernel, with pruning on and off: doc ids, f32 and f64 scores and counts the same bits on every path, unused rows
0xFFFFFFFF, and equal to OracleIndex.search_exhaustive (every query; a sample of the slot-reset batch)."""
import time

import numpy as np
import pytest

import util_filter as uf
import util_prune as up
import util_seeds as us
from util_cuda import sm_count
from util_lib import gpu_library, set_options  # noqa: F401  (gpu_library: the module fixture m)
from util_parity import KERNEL_PATHS, PrefixOracle, compare, query_csr, same_rows
from util_sparse import peak_host_gb

pytestmark = pytest.mark.gpu

PATHS = dict(seeded=dict(KERNEL_PATHS["seeded"], seed_max_terms=8), plain=KERNEL_PATHS["plain"])


@pytest.fixture(scope="module", autouse=True)
def _wall_time():
    t0 = time.perf_counter()
    yield
    print(f"\n[seed windows] module wall time {time.perf_counter() - t0:.1f} s, host peak {peak_host_gb():.2f} GB")


def _index(m, c):
    return m.Index(c.n_docs, c.doc_len, c.n_terms, c.post_off, c.post_doc, c.post_tf, k1=up.K1, b=up.B)


def _oracle(orc, c):
    return orc.OracleIndex(orc.Corpus(c.n_docs, c.doc_len, c.n_terms, c.post_off, c.post_doc, c.post_tf, k1=up.K1, b=up.B))


def _rows(res, idx):
    return {key: res[key][idx] for key in ("doc", "score", "score64", "n")}


def _every_path(ix, oix, c, qs, ks, what, sample=None):
    """Seeded and plain launches, pruning on and off, at every limit: the same rows, unused rows 0xFFFFFFFF, equal to
    the oracle (on the queries `sample`, default all)."""
    for q in qs:
        for prune in (1, 0):
            assert not uf.hands_back(dict(df=[int(c.df[t]) for t in q], n_docs=c.n_docs), PATHS["seeded"], prune), q
    q_off, q_terms = query_csr(qs)
    sample = np.arange(len(qs)) if sample is None else np.asarray(sample)
    s_off, s_terms = query_csr([qs[i] for i in sample])
    for k in ks:
        got = {}
        for name, opts in PATHS.items():
            for prune in (1, 0):
                set_options(ix, prune=prune, **opts)
                got[name, prune] = ix.search_batch(q_off, q_terms, k)
        for key, res in got.items():
            same_rows(res, got["seeded", 0], f"{what} {key} k={k}")
            assert np.all(res["doc"][np.arange(k)[None, :] >= res["n"][:, None]] == 0xFFFFFFFF), f"{what} {key} k={k}"
        compare(_rows(got["seeded", 0], sample), oix, s_off, s_terms, k, what=f"{what} k={k}")


@pytest.mark.parametrize("shared", [0, 1], ids=["alone", "shared"])
def test_full_slices_in_one_window(m, orc, shared):
    c = us.full_slices_case(orc, shared)
    ix = _index(m, c)
    _every_path(ix, PrefixOracle(_oracle(orc, c), max(c.ks)), c, c.qs, c.ks, f"full slices shared={shared}")
    ix.close()


def test_list_full_between_slices(m, orc):
    """Each query at every limit of STOP_KS (the model's pauses are those of its own limit)."""
    c = us.slice_stops_case(orc)
    ix = _index(m, c)
    _every_path(ix, PrefixOracle(_oracle(orc, c), us.CHAMP_L), c, c.qs, us.STOP_KS, "list full")
    ix.close()


def test_seeds_on_window_edges(m, orc):
    c = us.edge_case(orc)
    ix = _index(m, c)
    _every_path(ix, PrefixOracle(_oracle(orc, c), max(us.EDGE_KS)), c, c.qs, us.EDGE_KS, "window edges")
    ix.close()


def test_seed_slots_of_the_previous_query(m, orc):
    """Per class twice as many queries as the most warps a launch keeps resident (BM25X_RING_MAXWARPS per SM), so every
    warp serves several; a sample of 64 per class against the oracle."""
    c = us.slot_reset_case(orc)
    per_class = 2 * us.MAX_WARPS * sm_count()
    qs = us.reset_queries(c, per_class)
    sample = np.concatenate([i * per_class + np.arange(64) * (per_class // 64) + np.arange(64) % 2 for i in range(len(us.CLASSES))])
    ix = _index(m, c)
    _every_path(ix, PrefixOracle(_oracle(orc, c), max(us.RESET_KS)), c, qs, us.RESET_KS, "slot reset", sample=sample)
    ix.close()
