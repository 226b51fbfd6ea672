"""GPU: the prepared-batch API (bm25x_batch_prepare / _run / _fetch / _device_results, Python `Batch`) that bench.py times —
one batch prepared once and run many times, on the library's stream and on caller streams, several batches and several
threads on one index at once — and the statistics of a run (bm25x_search_stats) restated on the CPU.

A rerun depends on what bm25x_batch_run resets (the per-class work counters, the hand-over lists of seeded and two-phase
launches, the `postings_fetched` counter) and on the kernels rewriting every row of every live query.  So before a rerun
the result rows of the live queries are poisoned on the device (n = 0xFFFFFFFF, doc ids and scores 0xAB bytes): a run that
answered nothing, or wrote only part of a row, leaves poison behind.  Rows of queries without a live term are set once by
prepare and written by no kernel: they keep what prepare gave them.  Bar: every fetch equals a fresh bm25x_search_batch bit for bit, and
the fresh results equal the oracle (OracleIndex.search_exhaustive over the canonical queries)."""
import threading

import numpy as np
import pytest

import _pkg
from test_gpu_parity import _compare, _live_queries, _oracle_index, _PrefixOracle, _rows_identical
from util_cuda import device_synchronize, download, memset

pytestmark = pytest.mark.gpu

KS = (10, 128, 224, 1025)
CLASSES = (1, 2, 3, 4, 8, 16, 32, 64)  # term-count classes of bm25x_batch_prepare (64: two passes of the 32-term kernel)
# kernel paths of the 2..8-term classes, as index options (every option set: BM25X_SEED_FORCE changes none of them)
_SEEDED = dict(seed=1, twophase=0, seed_max_terms=8)
PATHS = dict(seeded=dict(_SEEDED, seed_prune_min=0xFFFFFFFF, seed_dense_div=0),  # no hand-back
             handback=dict(_SEEDED, seed_prune_min=64, seed_dense_div=64),       # skewed and dense queries handed back
             twophase=dict(seed=0, twophase=1, seed_max_terms=8, seed_prune_min=32768, seed_dense_div=64),
             plain=dict(seed=0, twophase=0, seed_max_terms=8, seed_prune_min=32768, seed_dense_div=64))


@pytest.fixture(scope="module")
def m():
    mod = _pkg.load()
    mod.load_library()
    assert mod.device_count() >= 1, "no CUDA device: the engine has no CPU fallback"
    return mod


@pytest.fixture(scope="module")
def corpus(m):
    # Zipf: head terms next to rare ones, so that seeded launches hand queries back (seed_prune_min = 64)
    return m.synth_corpus(301, 8000, 3000, 8, 120, 1.0)


@pytest.fixture(scope="module")
def ix(m, corpus):
    index = m.Index.from_corpus(corpus)
    yield index
    index.close()


@pytest.fixture(scope="module")
def oix(orc, corpus):
    return _PrefixOracle(_oracle_index(orc, corpus), max(KS))


def _csr(qs):
    q_off = np.cumsum([0] + [len(q) for q in qs]).astype(np.uint32)
    return q_off, (np.concatenate(qs) if qs else np.zeros(0)).astype(np.uint32)


def _canonical(q, df):
    """bm25x_batch_prepare's canonical query: ascending, distinct, ids >= n_terms and df = 0 terms dropped."""
    q = np.asarray(q, dtype=np.uint32)
    q = q[q < len(df)]
    return np.unique(q[df[q] > 0]).astype(np.uint32)


@pytest.fixture(scope="module")
def mixed(m, corpus, ix):
    """~120 queries: every term-count class boundary (1 ... 64 live terms) with terms drawn uniformly, 1..8-term queries
    with terms drawn by df (head terms next to rare ones); raw forms with duplicate terms and unknown ids; repeated
    queries; queries without a live term.  Shuffled.  Returns (q_off, q_terms, canonical queries, live mask, prefilter
    bitmap)."""
    rng = np.random.default_rng(301)
    df = ix.df()
    T = corpus.n_terms
    qs = []
    for counts, weighted in (([1, 2, 3, 4, 5, 8, 9, 16, 17, 32, 33, 64] * 4, False), ([1, 2, 3, 4, 5, 8] * 8, True)):
        o, t = _live_queries(rng, df, counts, weighted=weighted)
        qs += [t[o[i]:o[i + 1]] for i in range(len(counts))]
    for i in rng.choice(len(qs), size=12, replace=False):  # duplicates and unknown ids around a live core
        junk = [m.TERM_MISSING, T, T + 9, 10 ** 7] + list(rng.choice(qs[i], size=min(len(qs[i]), 12)))
        qs.append(rng.permutation(np.concatenate([qs[i], np.array(junk)]).astype(np.uint32)))
    qs += [qs[5]] * 3 + [qs[60]] * 2
    zero = np.flatnonzero(df == 0)
    qs += [np.zeros(0, np.uint32), np.array([m.TERM_MISSING]), np.array([T, 10 ** 7]),
           np.array([m.TERM_MISSING, T, m.TERM_MISSING])] + ([zero[:2]] if len(zero) else [])
    qs = [np.asarray(qs[i], dtype=np.uint32) for i in rng.permutation(len(qs))]
    canon = [_canonical(q, df) for q in qs]
    n_live = np.array([len(c) for c in canon])
    assert n_live.max() == 64 and set(CLASSES) <= set(n_live.tolist())
    live = n_live > 0
    assert 4 <= (~live).sum() and any(len(q) != len(c) for q, c in zip(qs, canon) if len(c))
    allow = np.packbits(rng.random(corpus.n_docs) < 0.5, bitorder="little")
    return _csr(qs) + (canon, live, allow)


def _set(ix, **opts):
    for name, value in opts.items():
        ix.set_option(name, value)


def _runs(mask):
    """[a, b) ranges of consecutive True entries of `mask`."""
    edges = np.flatnonzero(np.diff(np.concatenate([[0], mask.astype(np.int8), [0]])))
    return list(zip(edges[0::2].tolist(), edges[1::2].tolist()))


def _poison(batch, live):
    """Overwrite the result rows of the live queries on the device: every row is poisoned, then the rows of queries
    without a live term get back what prepare gave them (few memsets: the rows of live queries are many short runs).  The
    batch's last run must have finished (fetch synchronises); the device synchronisation orders the memsets before the
    next run on a non-blocking stream."""
    dev, k = batch.device_results(), batch.k
    rows = (("doc", 4, 0xFF), ("score", 4, 0), ("score64", 8, 0), ("payload", 6, 0))
    for key, _, _ in rows:
        memset(dev[key][0], 0xAB, dev[key][1])
    memset(dev["n"][0], 0xFF, dev["n"][1])
    for a, b in _runs(~live):
        for key, width, value in rows:
            memset(dev[key][0] + a * k * width, value, (b - a) * k * width)
        memset(dev["n"][0] + 4 * a, 0, 4 * (b - a))
    device_synchronize()


def _same(got, want, what):
    _rows_identical(got, want, what)
    if got.get("payload") is not None:
        assert np.array_equal(got["payload"], want["payload"]), f"{what}: payload"


def _check_oracle(res, oix, canon, k, allow, what):
    c_off, c_terms = _csr(canon)
    _compare(res, oix, c_off, c_terms, k, allow=allow, what=what)


def _cls(n):
    return next(c for c in CLASSES if c >= n)


def _launches(canon, k, allow, prep, run=None):
    """Kernel launches of one bm25x_batch_run: one per non-empty term-count class, two where the class runs seeded (the
    seeded launch + the launch of its hand-back list) or two-phase.  prepare allocates the hand-over buffers under the
    options of its time (`prep`); run picks the launches under the options of its own (`run`) and falls back to the plain
    kernel where prepare allocated nothing for them."""
    run = prep if run is None else run

    def seeded(o, M):
        return o["seed"] and allow is None and 2 <= M <= o["seed_max_terms"] and k <= 128

    def two(o, M):
        return o["twophase"] and 2 <= M <= 4 and k <= 224

    total = 0
    for M in {_cls(len(c)) for c in canon if len(c)}:
        q2 = seeded(prep, M) or two(prep, M)
        total += 2 if q2 and (seeded(run, M) or (two(prep, M) and run["twophase"])) else 1
    return total


def _restated(canon, df, k, allow, opts):
    """(queries, postings, bytes_algo, launches) of a search over the canonical queries."""
    live = sum(1 for c in canon if len(c))
    postings = sum(int(df[c].astype(np.uint64).sum()) for c in canon)
    qterms = sum(len(c) for c in canon)
    return live, postings, 8 * postings + 8 * live * k + 16 * qterms, _launches(canon, k, allow, opts)


def _fields(st):
    return (st.queries, st.postings, st.bytes_algo, st.launches)


@pytest.mark.parametrize("path", list(PATHS))
def test_rerun_rewrites_every_row(m, ix, oix, mixed, path):
    """One prepared batch, run 3 times with a fetch in between and 5 times back to back: every run rewrites every row of
    every live query (the rows are poisoned before each sequence), and every fetch equals a fresh search_batch — for the
    seeded kernel with and without a hand-back list, the two-phase launches and the plain kernel, pruning on and off,
    limits of every pool class, with and without a prefilter bitmap.  The fresh results equal the oracle."""
    q_off, q_terms, canon, live, allow = mixed
    if path == "handback":  # the hand-back list is not empty, and not every query is on it
        df, n_docs = ix.df(), ix.n_docs
        eligible = [c for c in canon if 2 <= len(c) <= 8]
        back = [c for c in eligible if (df[c].max() >= 64 and df[c].max() // 8 >= df[c].min()) or
                df[c].max() >= n_docs // 64 + 1]
        assert 0 < len(back) < len(eligible), (len(back), len(eligible))
    for prune in (1, 0):
        _set(ix, prune=prune, **PATHS[path])
        for k in KS:
            for al in (None, allow):
                what = f"{path} prune={prune} k={k} allow={al is not None}"
                want = ix.search_batch(q_off, q_terms, k, allow=al, want_payload=True)
                if prune:
                    _check_oracle(want, oix, canon, k, al, what)
                b = ix.prepare(q_off, q_terms, k, allow=al)
                for r in range(3):
                    _poison(b, live)
                    b.run(timed=False)
                    _same(b.fetch(want_payload=True), want, f"{what} run {r}")
                _poison(b, live)
                for _ in range(5):
                    b.run(timed=False)
                _same(b.fetch(want_payload=True), want, f"{what} 5 runs back to back")
                b.close()
    ix.set_option("prune", 1)


def test_caller_streams_and_interleaved_batches(m, ix, mixed):
    """Three batches of different limit and path (seeded with hand-back; two-phase with a prefilter bitmap; HBM pools at
    k = 1025) run interleaved on two torch streams and the library's stream with no host synchronisation in between, as
    bench.py passes its stream: each fetch equals its own fresh result.  One batch run on a second stream after an event
    wait on the first (ordering the runs of one batch is the caller's job), and a batch run on a caller stream right after
    prepare (the run waits for the upload)."""
    import torch
    q_off, q_terms, canon, live, allow = mixed
    _set(ix, prune=1, **dict(PATHS["handback"], twophase=1))
    specs = [(10, None), (200, allow), (1025, None)]
    want = [ix.search_batch(q_off, q_terms, k, allow=al, want_payload=True) for k, al in specs]
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    streams = [s1.cuda_stream, s2.cuda_stream, None]
    bs = [ix.prepare(q_off, q_terms, k, allow=al) for k, al in specs]
    for b in bs:
        _poison(b, live)
    for _ in range(3):
        for b, s in zip(bs, streams):
            b.run(stream=s, timed=False)
    for b, w, (k, _) in zip(bs, want, specs):
        _same(b.fetch(want_payload=True), w, f"k={k} interleaved")

    b = bs[0]
    _poison(b, live)
    b.run(stream=s1.cuda_stream, timed=False)
    ev = torch.cuda.Event()
    ev.record(s1)
    s2.wait_event(ev)
    b.run(stream=s2.cuda_stream, timed=False)  # fetch reads on the stream of the last run
    _same(b.fetch(want_payload=True), want[0], "second stream after an event wait")
    for b in bs:
        b.close()

    fresh = ix.prepare(q_off, q_terms, 200, allow=allow)
    fresh.run(stream=s1.cuda_stream, timed=False)
    _same(fresh.fetch(want_payload=True), want[1], "caller stream right after prepare")
    st = fresh.run(stream=s2.cuda_stream, timed=True)
    assert _fields(st) == _fields(want[1]["stats"]) and st.kernel_ms > 0
    fresh.close()


def test_device_results_and_partial_fetch(m, ix, mixed):
    """device_results() rows read back with cudaMemcpy equal fetch(), at addresses that stay put across reruns; fetch
    without f64 scores and / or payloads returns the same subsets.  Options are read by run, buffers are allocated by
    prepare: a batch prepared under one option set and run under another returns the same rows, through the launches
    that prepare's buffers allow.  A batch prepared over a slice of an offset array (absolute offsets into the whole
    q_terms) returns those rows of the whole batch."""
    q_off, q_terms, canon, live, allow = mixed
    nq = len(q_off) - 1
    _set(ix, prune=1, **PATHS["handback"])
    k = 128
    b = ix.prepare(q_off, q_terms, k)
    b.run(timed=False)
    full = b.fetch(want_payload=True)
    dev = b.device_results()
    shape = dict(doc=(nq, k), score=(nq, k), score64=(nq, k), payload=(nq, k, 3), n=(nq,))
    dtype = dict(doc=np.uint32, score=np.float32, score64=np.float64, payload=np.uint16, n=np.uint32)
    for key, (ptr, nbytes) in dev.items():
        assert np.array_equal(download(ptr, nbytes, dtype[key]).reshape(shape[key]), full[key]), key
    for _ in range(2):
        b.run(timed=False)
    assert b.device_results() == dev
    for pay in (False, True):
        part = b.fetch(want_f64=False, want_payload=pay)
        assert part["score64"] is None and (part["payload"] is None) == (not pay)
        for key in ("doc", "score", "n") + (("payload",) if pay else ()):
            assert np.array_equal(part[key], full[key]), (key, pay)
    b.close()

    # prepare under `prep`, run under `run` (k = 10: every 2..8-term class may run seeded)
    k = 10
    _set(ix, **PATHS["plain"])
    want = ix.search_batch(q_off, q_terms, k, want_payload=True)
    smt4 = dict(PATHS["handback"], seed_max_terms=4)
    for prep, run in ((PATHS["handback"], PATHS["plain"]), (PATHS["plain"], PATHS["handback"]),
                      (PATHS["plain"], PATHS["twophase"]), (PATHS["twophase"], PATHS["plain"]),
                      (PATHS["twophase"], PATHS["handback"]), (smt4, PATHS["handback"]), (PATHS["handback"], smt4)):
        for prune_prep, prune_run in ((1, 0), (0, 1)):
            _set(ix, prune=prune_prep, **prep)
            b = ix.prepare(q_off, q_terms, k)
            _set(ix, prune=prune_run, **run)
            st = b.run(timed=True)
            what = f"prepared {prep} prune={prune_prep}, run {run} prune={prune_run}"
            _same(b.fetch(want_payload=True), want, what)
            assert st.launches == _launches(canon, k, None, prep, run), what
            b.close()
    assert _launches(canon, k, None, PATHS["handback"], PATHS["plain"]) == len({_cls(len(c)) for c in canon if len(c)})

    # a slice of the offset array: rows a .. b-1 of the whole batch
    _set(ix, prune=1, **PATHS["handback"])
    for a, e in ((37, 121), (0, 1), (nq - 5, nq), (60, 60)):
        sub = ix.prepare(q_off[a:e + 1], q_terms, k)
        st = sub.run(timed=True)
        got = sub.fetch(want_payload=True)
        _same(got, {key: want[key][a:e] for key in ("doc", "score", "score64", "payload", "n")}, f"slice [{a}, {e})")
        assert _fields(st) == _restated(canon[a:e], ix.df(), k, None, PATHS["handback"]), (a, e)
        sub.close()


@pytest.mark.parametrize("path", list(PATHS))
def test_search_stats_restated(m, ix, mixed, path):
    """bm25x_search_stats against a CPU restatement, for Batch.run(timed=True) and search_batch (one piece and sliced):
    `queries` = live queries, `postings` = sum of df over the canonical terms, `bytes_algo` = 8 * postings + 8 * live * k
    + 16 * live terms, `launches` per non-empty class.  Three timed reruns report the same numbers (postings_fetched is
    reset by each timed run).  With pruning off, postings_fetched = postings exactly for queries of <= 32 live terms on the
    plain and both seeded paths (refills count real postings only, a hand-back happens before the first refill); two-pass
    queries (probes of the other group) and two-phase runs (a resume re-reads its ring) fetch at least that many."""
    q_off, q_terms, canon, live, allow = mixed
    df = ix.df()
    nq = len(q_off) - 1
    short = [i for i in range(nq) if len(canon[i]) <= 32]
    s_off, s_terms = _csr([q_terms[q_off[i]:q_off[i + 1]] for i in short])
    sets = dict(mixed=(q_off, q_terms, canon), short=(s_off, s_terms, [canon[i] for i in short]))
    opts = PATHS[path]
    for prune in (1, 0):
        _set(ix, prune=prune, **opts)
        for k in KS:
            for al in (None, allow):
                for name, (qo, qt, cn) in sets.items():
                    if prune and name == "short":
                        continue
                    what = f"{path} prune={prune} k={k} allow={al is not None} {name}"
                    want = _restated(cn, df, k, al, opts)
                    b = ix.prepare(qo, qt, k, allow=al)
                    runs = [b.run(timed=True) for _ in range(3)]
                    b.close()
                    ix.set_option("slice_min", 0)
                    one = ix.search_batch(qo, qt, k, allow=al)["stats"]
                    for st in runs + [one]:
                        assert _fields(st) == want, what
                        assert st.kernel_ms > 0 and st.postings_fetched == runs[0].postings_fetched, what
                    assert runs[0].h2d_ms == runs[0].d2h_ms == 0.0
                    fetched = runs[0].postings_fetched
                    if prune == 0:
                        exact = name == "short" and not (opts["twophase"] and k <= 224)
                        if exact:
                            assert fetched == want[1], (what, fetched, want[1])
                        else:
                            assert fetched >= want[1], (what, fetched, want[1])
                    # sliced: slice s holds queries [nq * s / n, nq * (s + 1) / n), n = min(16, nq / slice_min)
                    ix.set_option("slice_min", 16)
                    cut = ix.search_batch(qo, qt, k, allow=al)["stats"]
                    n_sl = min(16, (len(qo) - 1) // 16)
                    edges = [(len(qo) - 1) * s // n_sl for s in range(n_sl + 1)]
                    launches = sum(_launches(cn[a:e], k, al, opts) for a, e in zip(edges[:-1], edges[1:]))
                    assert _fields(cut) == want[:3] + (launches,), what
                    assert cut.postings_fetched == fetched, what
    _set(ix, prune=1, slice_min=0)


def test_concurrent_threads_one_index(m, corpus, ix, mixed):
    """Eight threads on one index at once (ctypes releases the GIL), started on a barrier: single-piece search_batch,
    sliced search_batch (slice_min = 16) and prepare / run / fetch on the thread's own torch stream, batches growing so
    that the staging buffer of prepare is reallocated while other uploads are pending.  Every result equals the same call
    made alone.  One thread loops on refused calls: its error messages are its own, the other threads see none.  Then
    fresh indexes whose first calls are all sliced and concurrent (the download stream of sliced calls exists from the
    creation of the index: no first call creates it)."""
    import torch
    q_off, q_terms, canon, live, allow = mixed
    nq = len(q_off) - 1
    opts = dict(PATHS["handback"], prune=1, slice_min=16)
    _set(ix, **opts)
    rng = np.random.default_rng(311)

    def plan(t, sizes, first_kind):
        calls = []
        for j, size in enumerate(sizes):
            kind = ("sliced", "split", "single")[(first_kind + j) % 3]
            size = min(size, 31) if kind == "single" else max(size, 32)  # nq >= 2 * slice_min: sliced
            idx = rng.choice(nq, size=size)
            sub = _csr([q_terms[q_off[i]:q_off[i + 1]] for i in idx])
            k = (10, 100, 224)[(t + j) % 3]
            calls.append((kind, sub, k, allow if (t + j) % 4 == 0 else None))
        return calls

    def expected(calls):
        return [ix.search_batch(sub[0], sub[1], k, allow=al, want_payload=True) for _, sub, k, al in calls]

    live_terms = np.flatnonzero(ix.df() > 0)
    q65 = np.sort(rng.choice(live_terms, size=65, replace=False)).astype(np.uint32)
    refusals = [  # (call, code, message)
        (lambda x: x.search_batch(q_off, q_terms, 0), 5, "number of needed rows is set to 0"),
        (lambda x: x.prepare(np.array([0, 65], np.uint32), q65, 10), 4,
         "bm25x_batch_prepare: query 0 has 65 live terms > 64"),
        (lambda x: x.prepare(q_off, q_terms, m.MAX_K + 1), 4, f"bm25x_batch_prepare: k={m.MAX_K + 1} > BM25X_MAX_K=65535")]

    def run_threads(index, plans, refuse):
        n = len(plans) + (1 if refuse else 0)
        barrier, done = threading.Barrier(n), threading.Event()
        streams = [torch.cuda.Stream() for _ in plans]
        got, errs, refused = [None] * len(plans), [], [0]

        def worker(t):
            try:
                barrier.wait()
                out = []
                for kind, (so, st_), k, al in plans[t]:
                    if kind == "split":
                        b = index.prepare(so, st_, k, allow=al)
                        for _ in range(2):
                            b.run(stream=streams[t].cuda_stream, timed=False)
                        out.append(b.fetch(want_payload=True))
                        b.close()
                    else:
                        out.append(index.search_batch(so, st_, k, allow=al, want_payload=True))
                got[t] = out
            except Exception as e:  # pragma: no cover - reported below
                errs.append((t, repr(e)))

        def refuser():
            try:
                barrier.wait()
                i = 0
                while i < 60 or not done.is_set():
                    call, code, msg = refusals[i % len(refusals)]
                    with pytest.raises(m.Bm25xError) as e:
                        call(index)
                    assert e.value.code == code and str(e.value) == f"bm25x error {code}: {msg}", str(e.value)
                    i += 1
                refused[0] = i
            except BaseException as e:  # pragma: no cover - reported below
                errs.append(("refuser", repr(e)))

        ts = [threading.Thread(target=worker, args=(t,)) for t in range(len(plans))]
        if refuse:
            ts.append(threading.Thread(target=refuser))
        for t in ts:
            t.start()
        for t in ts[:len(plans)]:
            t.join()
        done.set()
        for t in ts[len(plans):]:
            t.join()
        assert not errs, errs
        assert not refuse or refused[0] >= 60
        return got

    sizes = (6, 24, 48, 100, 200, 400)
    plans = [plan(t, sizes, t % 3) for t in range(7)]
    wants = [expected(p) for p in plans]
    index = m.Index.from_corpus(corpus)  # fresh: its staging buffer grows during the threads
    _set(index, **opts)
    got = run_threads(index, plans, refuse=True)
    for t in range(len(plans)):
        for j, (g, w) in enumerate(zip(got[t], wants[t])):
            _same(g, w, f"thread {t} call {j} ({plans[t][j][0]}, k={plans[t][j][2]})")
    index.close()

    # every thread's first call is sliced, on indexes that have served no call yet
    plans = [plan(t, (64, 160), 0) for t in range(8)]
    wants = [expected(p) for p in plans]
    for r in range(2):
        index = m.Index.from_corpus(corpus)
        _set(index, **opts)
        got = run_threads(index, plans, refuse=False)
        for t in range(len(plans)):
            for j, (g, w) in enumerate(zip(got[t], wants[t])):
                _same(g, w, f"fresh index {r} thread {t} call {j}")
        index.close()
    _set(ix, slice_min=0)


def test_prepare_refusals(m, corpus, ix, mixed):
    """What prepare refuses, with its code: offsets that go backwards (1), more than 64 live terms (4), k = 0 (5),
    k > MAX_K (4), a replica that is not finalized (1).  A refused prepare leaves nothing behind: the next prepare on the
    same index works and answers as before."""
    q_off, q_terms, canon, live, allow = mixed
    _set(ix, prune=1, **PATHS["handback"])
    want = ix.search_batch(q_off, q_terms, 10, want_payload=True)
    rng = np.random.default_rng(321)
    q65 = np.sort(rng.choice(np.flatnonzero(ix.df() > 0), size=65, replace=False)).astype(np.uint32)
    dup64 = np.concatenate([q65[:64], q65[:64], [m.TERM_MISSING]]).astype(np.uint32)  # 129 raw, 64 live: accepted
    bad = [(np.array([0, 5, 3, 8], np.uint32), q_terms, 10, 1),
           (np.array([0, 3, 3 + 65], np.uint32), np.concatenate([q65[:3], q65]), 10, 4),
           (q_off, q_terms, 0, 5),
           (q_off, q_terms, m.MAX_K + 1, 4)]
    for qo, qt, k, code in bad:
        for _ in range(3):
            with pytest.raises(m.Bm25xError) as e:
                ix.prepare(qo, qt, k)
            assert e.value.code == code, (code, str(e.value))
        b = ix.prepare(q_off, q_terms, 10)
        b.run(timed=False)
        _same(b.fetch(want_payload=True), want, f"prepare after a code-{code} refusal")
        b.close()
    b = ix.prepare(np.array([0, len(dup64)], np.uint32), dup64, 10)
    assert b.run(timed=True).queries == 1
    b.close()
    rep = m.Index.alloc_replica(ix.layout(), 0)
    with pytest.raises(m.Bm25xError) as e:
        rep.prepare(q_off, q_terms, 10)
    assert e.value.code == 1 and "not finalized" in str(e.value)
    rep.close()
