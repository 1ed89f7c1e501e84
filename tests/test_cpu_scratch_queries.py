"""The hub-plan scratch an entry point needs is written down once, in the library's cogdl_b200_<family>_scratch_bytes
queries: each entry's check_plan calls its query, and the Python wrappers allocate what the same query returns.  These
tests read the sources for inline byte arithmetic and call every query through the loaded library (no GPU needed)."""
import os
import re

import pytest

from tests.test_cpu_oracle_and_host import declared_symbols

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "cogdl_b200", "csrc")


def sources(top, exts):
    for dirpath, _, files in os.walk(top):
        for f in sorted(files):
            if f.endswith(exts):
                path = os.path.join(dirpath, f)
                with open(path) as fh:
                    yield os.path.relpath(path, ROOT), fh.read()


def call_args(text, name):
    """The argument text of every call `name(...)` in text (balanced parentheses), skipping Python definitions."""
    for m in re.finditer(r"(?<![\w.])(def\s+)?(?:\w+\.)*" + name + r"\(", text):
        depth, i = 1, m.end()
        while depth:
            depth += {"(": 1, ")": -1}.get(text[i], 0)
            i += 1
        if not m.group(1):
            yield text[m.end():i - 1]


def test_every_check_plan_passes_zero_or_a_size_query():
    calls = [(path, args) for path, text in sources(CSRC, (".cu", ".cuh")) for args in call_args(text, "check_plan")
             if not args.lstrip().startswith("const ")]          # the declaration and the definition
    assert len(calls) >= 20
    queries = set(declared_symbols())
    for path, args in calls:
        need = args.split(",", 1)[1].strip()
        m = re.fullmatch(r"(cogdl_b200_\w+_scratch_bytes)\(.*\)", need, re.S)
        assert need == "0" or (m and m.group(1) in queries), f"{path}: check_plan({args})"


def test_no_plan_struct_call_passes_byte_arithmetic():
    calls = [(path, args.strip()) for path, text in sources(os.path.join(ROOT, "cogdl_b200"), (".py",))
             for args in call_args(text, "plan_struct")]
    assert len(calls) >= 3
    for path, args in calls:
        assert args in ("", "0", "partial_bytes") or re.fullmatch(r"_scratch\([^()]*\)", args), \
            f"{path}: plan_struct({args})"


# family, shape after n_chunks, and the bytes per chunk the Python wrappers allocated before the library gave the size
QUERIES = [
    ("spmm", (48,), 48 * 4),
    ("mhspmm", (8, 16), 8 * 16 * 4),
    ("gat_fwd", (8, 16), max(8 * 16 * 4, 8 * 12)),
    ("gat_fwd", (8, 1), max(8 * 1 * 4, 8 * 12)),
    ("edge_softmax", (8,), 8 * 12),
    ("scatter_max", (48,), 48 * 8),
    ("edge_colsum", (8,), 8 * 4),
    ("gcn_fused", (128,), 128 * 4),
    ("sage_fused", (128, 0), 128 * 4),
    ("sage_fused", (128, 1), 128 * 8),
    ("softmax_aggr", (48,), 48 * 16),
    ("softmax_aggr_bwd", (48,), 48 * 4),
    ("genconv_edge_bwd", (48, 1), 48 * 4),
    ("genconv_edge_bwd", (48, 0), 0),
    ("disen_route", (64, 4), (2 * 64 + 2 * 4) * 4),
    ("comp_aggr", (48,), 48 * 4),
    ("rgcn_aggr", (3, 48), 3 * 48 * 4),
]


@pytest.mark.parametrize("family,shape,per_chunk", QUERIES, ids=[f"{q[0]}{q[1]}" for q in QUERIES])
def test_size_query_is_zero_without_chunks_and_within_the_old_allocation(family, shape, per_chunk):
    from cogdl_b200 import _cabi

    query = getattr(_cabi.load(), f"cogdl_b200_{family}_scratch_bytes")
    assert query(0, *shape) == 0
    n_chunks = 37
    need = query(n_chunks, *shape)
    assert 0 <= need <= n_chunks * per_chunk
    if per_chunk:
        assert need > 0


def test_every_plan_size_query_is_covered():
    """A query whose first argument is n_chunks sizes plan partials; each one has a row in QUERIES."""
    with open(os.path.join(ROOT, "include", "cogdl_b200.h")) as f:
        header = f.read()
    families = set(re.findall(r"\bcogdl_b200_(\w+)_scratch_bytes\(int64_t n_chunks", header))
    assert families == {q[0] for q in QUERIES}
