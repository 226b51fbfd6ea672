"""GPU parity stress: many small random corpora / query shapes / limits against the exhaustive oracle, bit for bit —
ring wrap-around, single-posting terms, head terms next to rare ones (dense windows, and pruning where a draw happens to
reach it), duplicate-heavy vocabularies (tie floods), every term-count class, pruning on and off.  Nothing here asserts
that a query pruned or that its rings were split again: test_gpu_prune_points.py builds those cases on purpose."""
import numpy as np
import pytest

from util_lib import gpu_library  # noqa: F401  (gpu_library: the module fixture m)
from util_parity import compare, oracle_index

pytestmark = pytest.mark.gpu


def _cases():
    rng = np.random.default_rng(20260923)
    out = []
    for i in range(36):
        n = int(rng.choice([60, 300, 1500, 6000, 25000]))
        vocab = int(rng.choice([3, 12, 60, 400, 2500]))
        lmin = int(rng.integers(0, 6))
        lmax = lmin + int(rng.choice([0, 3, 30, 200]))
        out.append(dict(seed=1000 + i, n=n, vocab=vocab, lmin=lmin, lmax=lmax, zipf=float(rng.choice([0.0, 0.0, 0.7, 1.0, 1.4])),
                        tmax=int(rng.choice([1, 2, 3, 4, 7, 8, 13, 32])), k=int(rng.choice([1, 2, 7, 10, 31, 32, 33, 97, 224, 225, 1000])),
                        prune=int(rng.integers(0, 2))))
    return out


@pytest.mark.parametrize("cfg", _cases(), ids=lambda c: f"s{c['seed']}-n{c['n']}-v{c['vocab']}-t{c['tmax']}-k{c['k']}-p{c['prune']}")
def test_random_shapes_match_oracle(m, orc, cfg):
    c = m.synth_corpus(cfg["seed"], cfg["n"], cfg["vocab"], cfg["lmin"], max(cfg["lmax"], 1), cfg["zipf"])
    if int(c.post_off[-1]) == 0:
        pytest.skip("empty corpus")
    tmax = min(cfg["tmax"], max(1, int(np.count_nonzero(np.diff(c.post_off.astype(np.int64))))))
    q_off, q_terms = m.synth_queries(cfg["seed"] + 7, 24, cfg["vocab"], 1, tmax, c.post_off, cfg["zipf"])
    ix = m.Index.from_corpus(c)
    ix.set_option("prune", cfg["prune"])
    oix = oracle_index(orc, c)
    res = ix.search_batch(q_off, q_terms, cfg["k"])
    compare(res, oix, q_off, q_terms, cfg["k"], what=str(cfg))
    ix.close()
