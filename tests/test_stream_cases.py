"""Every entry point is in the stream-case table (tests/stream_cases.py) or exempt from it with a reason, so that a new
kernel cannot skip tests/test_gpu_streams.py.  Runs without a GPU."""
import os
import re

import stream_cases as SC

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(REPO, "deep-image-retrieval_b200")


def header_exports():
    with open(os.path.join(REPO, "include", "dirb200.h")) as f:
        return set(re.findall(r"^\s*(?:const\s+)?\w+\s*\*?\s*(dirb200_\w+)\s*\(", f.read(), re.M))


def python_calls():
    names = set()
    for fn in sorted(os.listdir(PKG)):
        if fn.endswith(".py"):
            with open(os.path.join(PKG, fn)) as f:
                names |= set(re.findall(r'lib\.call\(\s*"(dirb200_\w+)"', f.read()))
    return names


def missing(cases, exempt):
    covered = set().union(*(c.covers for c in cases))
    return sorted(n for n in header_exports() | python_calls() if n not in covered and n not in exempt)


def test_the_sources_are_found():
    exports, calls = header_exports(), python_calls()
    assert len(exports) > 100 and {"dirb200_index_search", "dirb200_whiten", "dirb200_graph_search"} <= exports
    assert len(calls) > 80 and calls <= exports


def test_every_entry_point_is_covered_or_exempt():
    assert missing(SC.STREAM_CASES, SC.EXEMPT) == []


def test_covers_and_exempt_name_real_exports_once():
    exports = header_exports()
    covered = set().union(*(c.covers for c in SC.STREAM_CASES))
    assert covered <= exports, sorted(covered - exports)
    assert set(SC.EXEMPT) <= exports, sorted(set(SC.EXEMPT) - exports)
    assert not covered & set(SC.EXEMPT), sorted(covered & set(SC.EXEMPT))
    assert all(reason.strip() for reason in SC.EXEMPT.values())


def test_case_names_are_unique():
    names = [c.name for c in SC.STREAM_CASES]
    assert len(names) == len(set(names))


def test_a_call_dropped_from_the_table_is_reported():
    """Removing any Python-called entry point from every case, without exempting it, makes the guard fail."""
    for name in sorted(python_calls() - set(SC.EXEMPT)):
        cases = [c._replace(covers=tuple(n for n in c.covers if n != name)) for c in SC.STREAM_CASES]
        assert missing(cases, SC.EXEMPT) == [name]
