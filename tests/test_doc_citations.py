"""The documents cite tests as evidence (`tests/<file>.py::<name>`): every such citation must name a test that exists."""
import ast
import glob
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CITE = re.compile(r"tests/([A-Za-z0-9_]+\.py)::([A-Za-z_][A-Za-z0-9_]*)")
# where the project keeps its documents (not recursive: build and run outputs never count as documents)
DOC_DIRS = ("", "tests", "oracle", "tools", "vectorchord-bm25_b200")


def _citations():
    docs = sorted(md for d in DOC_DIRS for md in glob.glob(os.path.join(ROOT, d, "*.md")))
    for md in docs:
        with open(md, encoding="utf-8") as f:
            for line_no, line in enumerate(f, 1):
                for fname, name in CITE.findall(line):
                    yield os.path.relpath(md, ROOT), line_no, fname, name


def _functions(path):
    with open(path, encoding="utf-8") as f:
        tree = ast.parse(f.read())
    return {n.name for n in ast.walk(tree) if isinstance(n, (ast.FunctionDef, ast.AsyncFunctionDef))}


def test_cited_tests_exist():
    cites = list(_citations())
    assert cites, "no citation found: the pattern no longer matches how the documents cite tests"
    missing = []
    for md, line_no, fname, name in cites:
        path = os.path.join(ROOT, "tests", fname)
        if not os.path.exists(path) or name not in _functions(path):
            missing.append(f"{md}:{line_no}: tests/{fname}::{name}")
    assert not missing, "cited tests that do not exist:\n" + "\n".join(missing)
