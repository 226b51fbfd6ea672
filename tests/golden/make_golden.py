#!/usr/bin/env python
"""Regenerates tests/golden/reference_golden.json from the read-only reference tree.

Needs a checkout of the reference tree:
    python tests/golden/make_golden.py <path to tensorchord/VectorChord-bm25>
Extracts every golden / known answer the reference's own tests hold for the
BM25 top-k path (SURVEY.md §8c):
  * the literal FIELDNORM_TO_LENGTH table        crates/bm25/src/bm25.rs:15-272
  * the sqllogictest ranking goldens             tests/sqllogictest/bm25query.slt:35-82,
                                                 tests/sqllogictest/indexing.slt:30-41
  * the passages those goldens are computed on   tests/sqllogictest/bm25query.slt:11-21
Document lengths are derived with a restatement of PostgreSQL's
to_tsvector('english', ...) *length* rule only (stop words dropped; a hyphenated
compound yields the compound plus each part), which is all the golden ranking
depends on (N=10, df=6, tf=1 everywhere → rank = ascending length, all <= 40 so
the fieldnorm is exact).
"""
import json
import os
import re
import sys

REF = sys.argv[1] if len(sys.argv) > 1 else "."
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference_golden.json")

STOP = set("""i me my myself we our ours ourselves you your yours yourself yourselves he him his himself she her
hers herself it its itself they them their theirs themselves what which who whom this that these those am is are was
were be been being have has had having do does did doing a an the and but if or because as until while of at by for
with about against between into through during before after above below to from up down in out on off over under
again further then once here there when where why how all any both each few more most other some such no nor not
only own same so than too very s t can will just don should now""".split())


def lexemes(text):
    """Lower-cased lexeme occurrences (no stemming: it does not change lengths)."""
    out = []
    for tok in re.findall(r"[A-Za-z0-9]+(?:-[A-Za-z0-9]+)*", text):
        tok = tok.lower()
        if "-" in tok:
            out.append(tok)
            out.extend(p for p in tok.split("-") if p not in STOP)
        elif tok not in STOP:
            out.append(tok)
    return out


def main():
    src = open(os.path.join(REF, "crates/bm25/src/bm25.rs")).read()
    m = re.search(r"FIELDNORM_TO_LENGTH: \[u32; 256\] = \[(.*?)\];", src, re.S)
    table = [int(x.replace("_", "")) for x in re.findall(r"[\d_]+", m.group(1))]
    assert len(table) == 256

    slt = open(os.path.join(REF, "tests/sqllogictest/bm25query.slt")).read()
    passages = re.findall(r"^\('(.*)'\)[,;]$", slt, re.M)
    assert len(passages) == 10
    results = [list(map(int, blk.split())) for blk in re.findall(r"^----\n((?:\d+\n)+)", slt, re.M)]
    assert results == [[8, 9, 4, 1, 7, 2], [8, 4, 2], [9, 1, 7]], results
    slt2 = open(os.path.join(REF, "tests/sqllogictest/indexing.slt")).read()
    results2 = [list(map(int, blk.split())) for blk in re.findall(r"^----\n((?:\d+\n)+)", slt2, re.M)]

    docs = [lexemes(p) for p in passages]
    golden = {
        "source": "tensorchord/VectorChord-bm25 @ reference tree; see make_golden.py for file:line",
        "fieldnorm_to_length": table,
        "passages": passages,
        "doc_lexemes": docs,
        "doc_lengths": [len(d) for d in docs],
        "query": "postgresql",
        "ranking_full_index": results[0],       # ids are 1-based SERIAL
        "ranking_even_ids": results[1],
        "ranking_odd_ids": results[2],
        "ranking_indexing_slt": results2[0] if results2 else None,
    }
    json.dump(golden, open(OUT, "w"), indent=1)
    print("wrote", OUT, "lengths", golden["doc_lengths"])


if __name__ == "__main__":
    main()
