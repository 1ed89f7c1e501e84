"""Every gather kernel compiled into spmm.o, sddmm.o, mhspmm.o and scatter_max.o has a row in the dispatch table
(tests/dispatch_table.py) that the GPU suite runs and checks, and every kernel the table names is compiled.  A new
dispatch branch without a test case fails here, on a machine without a GPU.

The kernel entry points are read from the objects with cuobjdump and demangled with cu++filt; each instantiation
is mapped to the string its launcher records for cogdl_b200_last_kernel()."""
import os
import re
import shutil
import subprocess

import pytest

from tests.dispatch_table import EXEMPT, TABLE

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBJ_DIR = os.path.join(ROOT, "cogdl_b200", "csrc", "build")
OBJECTS = ("spmm", "sddmm", "mhspmm", "scatter_max")


def _tool(name):
    for d in (os.environ.get("CUDA_HOME"), "/usr/local/cuda"):
        if d and os.access(os.path.join(d, "bin", name), os.X_OK):
            return os.path.join(d, "bin", name)
    return shutil.which(name)


def compiled_kernels():
    """Demangled kernel entry points (global functions) of the four objects."""
    cuobjdump, cufilt = _tool("cuobjdump"), _tool("cu++filt")
    if not cuobjdump or not cufilt:
        pytest.skip("cuobjdump / cu++filt from the CUDA toolkit are not available")
    paths = [os.path.join(OBJ_DIR, f"{o}.o") for o in OBJECTS]
    missing = [p for p in paths if not os.path.exists(p)]
    if missing:
        pytest.skip(f"library objects not built (run build()): {', '.join(missing)}")
    mangled = []
    for p in paths:
        out = subprocess.run([cuobjdump, "-symbols", p], capture_output=True, text=True, check=True).stdout
        mangled += [ln.split()[-1] for ln in out.splitlines() if "STT_FUNC" in ln and "STB_GLOBAL" in ln]
    assert mangled, "no kernel symbols found"
    out = subprocess.run([cufilt], input="\n".join(mangled) + "\n", capture_output=True, text=True, check=True).stdout
    return [ln.strip() for ln in out.splitlines() if ln.strip()]


_SRC = {0: "SRC_ONE", 1: "SRC_TWO", 2: "SRC_PEERS"}


def _args(sig):
    """Template arguments of a demangled name: 'float4', '(int)32', '(bool)1' -> 'float4', 32, True."""
    inner = sig[sig.index("<") + 1: sig.rindex(">")]
    out = []
    for a in inner.split(","):
        a = a.strip()
        m = re.fullmatch(r"\((int|bool)\)(-?\d+)", a)
        out.append(a if m is None else (int(m.group(2)) if m.group(1) == "int" else m.group(2) != "0"))
    return out


def note_of(sym):
    """The cogdl_b200_last_kernel() string of one demangled instantiation (canonical form, see canonical())."""
    m = re.fullmatch(r"(?:void )?cogdl_b200::(\w+)(<.*>)?\(.*\)", sym)
    assert m, f"unexpected symbol {sym!r}"
    name = m.group(1)
    a = _args(m.group(2)) if m.group(2) else []
    w = lambda b: "weighted" if b else "unweighted"  # noqa: E731
    if name == "spmm_kernel":
        vec, group, nv, has_val = a
        return f"cogdl_b200::spmm_kernel<{vec},GROUP={group},NV={nv},{w(has_val)}>"
    if name == "spmm_half_kernel":
        has_val, vec = a
        return f"cogdl_b200::spmm_half_kernel<{w(has_val)},{'vec' if vec else 'scalar'}>"
    if name == "stream_kernel":
        vec, nv, mode, perm, src, u, minb, prefetch, panel, drop = a
        what = {0: "unweighted", 1: "weighted", 2: "multihead"}[mode]
        if mode == 2:
            what += ("+perm" if perm else "") + ("+drop" if drop else "")
        s = f"cogdl_b200::stream_kernel<{vec},NV={nv},{what},{_SRC[src]},U={u},MINB={minb}{',prefetch' if prefetch else ''}>"
        return s + (",panels" if panel else "")
    if name == "sddmm_kernel":
        vec, group, sub, nv = a
        return f"cogdl_b200::sddmm_kernel<{vec},GROUP={group},SUB={sub},NV={nv}>"
    if name == "sddmm_stream_kernel":
        nv, u = a
        return f"cogdl_b200::sddmm_stream_kernel<NV={nv},U={u}>"
    if name == "mhspmm_kernel":
        vec, group, perm, drop = a
        return f"cogdl_b200::mhspmm_kernel<{vec},GROUP={group},{'perm' if perm else 'no_perm'}{',drop' if drop else ''}>"
    if name == "scatter_max_fwd_kernel":
        vec, group, nv = a
        return f"cogdl_b200::scatter_max_fwd_kernel<{vec},GROUP={group},NV={nv}>"
    if name == "scatter_max_stream_kernel":
        nv, u, argmax = a
        return f"cogdl_b200::scatter_max_stream_kernel<NV={nv},U={u}{'' if argmax else ',values_only'}>"
    if name == "scatter_max_bwd_kernel":
        return "cogdl_b200::scatter_max_bwd_kernel"
    raise AssertionError(f"no last_kernel() name is known for {sym!r}: add it to note_of() and a row to the table")


def canonical(note):
    """A recorded name without its launch-shape suffixes: the panel count becomes ',panels' (the instantiation is
    the same for every count) and ' block=N' goes."""
    return re.sub(r",panels=\d+", ",panels", re.sub(r" block=\d+$", "", note))


def test_note_of_maps_known_symbols():
    assert note_of("void cogdl_b200::spmm_kernel<float, (int)32, (int)4, (bool)1>(cogdl_b200::SpmmParams)") == \
        "cogdl_b200::spmm_kernel<float,GROUP=32,NV=4,weighted>"
    assert note_of("void cogdl_b200::stream_kernel<float2, (int)1, (int)0, (bool)0, (int)0, (int)8, (int)5, (bool)1, "
                   "(bool)1, (bool)0>(cogdl_b200::StreamParams)") == \
        "cogdl_b200::stream_kernel<float2,NV=1,unweighted,SRC_ONE,U=8,MINB=5,prefetch>,panels"
    assert canonical("cogdl_b200::stream_kernel<float2,NV=1,unweighted,SRC_ONE,U=8,MINB=5,prefetch>,panels=4 block=128") \
        == "cogdl_b200::stream_kernel<float2,NV=1,unweighted,SRC_ONE,U=8,MINB=5,prefetch>,panels"


def test_table_covers_every_compiled_kernel():
    compiled = {}
    for sym in compiled_kernels():
        compiled.setdefault(note_of(sym), sym)
    table = {canonical(c.kernel) for c in TABLE}
    untested = sorted(set(compiled) - table - set(EXEMPT))
    assert not untested, "compiled kernels without a row in tests/dispatch_table.py:\n" + "\n".join(
        f"  {n}   ({compiled[n]})" for n in untested)
    unknown = sorted(table - set(compiled))
    assert not unknown, "table rows name kernels that are not compiled:\n" + "\n".join(f"  {n}" for n in unknown)
    stale = sorted(set(EXEMPT) - set(compiled))
    assert not stale, f"exemptions for kernels that are not compiled: {stale}"


def test_table_rows_are_distinct():
    ids = [c.id for c in TABLE]
    dup = sorted({i for i in ids if ids.count(i) > 1})
    assert not dup, f"duplicate table rows: {dup}"
