"""One row per dispatch branch of cogdl_b200_spmm_residual_f32 (spmm_residual.cu): the fp32 SpMM's one-source
branches (tests/dispatch_table.py SPMM rows), each with the residual kernel it records, with Z and the row scale
switched on and off across the rows, and further rows for narrow widths, forced panel counts and the boundary-degree
graph.  test_gpu_spmm_residual.py runs every row; test_cpu_spmm_residual_inventory.py checks that the rows cover every
kernel compiled into spmm_residual.o and name no other.  Plain Python, no torch."""
from dataclasses import dataclass

from tests.dispatch_table import SPMM, spmm_k, stream_k


@dataclass(frozen=True)
class RCase:
    graph: str              # a name in tests/graphs.py CASES, or "bounds": boundary_csr(chunk)
    F: int
    kernel: str             # exact cogdl_b200_last_kernel() after the call
    aligned: bool = True    # False: X is a view one element past an aligned allocation
    plan: str = "default"   # none | chunks | default, as in dispatch_table.Case
    chunk: int = 64
    weighted: bool = True
    panels: int = 0
    z: bool = True          # Z given (else the output is a * (r * A @ X))
    row_scale: bool = False

    @property
    def id(self):
        s = f"{self.graph}-F{self.F}-{self.plan}-{'w' if self.weighted else 'u'}"
        s += "-z" if self.z else "-noz"
        s += "-rs" if self.row_scale else ""
        s += "" if self.aligned else "-misaligned"
        return s + (f"-P{self.panels}" if self.panels else "")


def residual_name(kernel):
    """The residual launch's name for the plain SpMM's: the same instantiation parameters under the residual kernel's
    name, and 4 blocks per SM (MINB=4) instead of 5 for the lean float4 loops, whose Z row needs more registers."""
    k = kernel.replace("::spmm_kernel<", "::spmm_residual_kernel<").replace("::stream_kernel<", "::stream_residual_kernel<")
    return k.replace("U=4,MINB=5", "U=4,MINB=4")


_EPI = [(True, False), (True, True), (False, True)]


def _rows():
    rows = []
    base = [c for c in SPMM if c.src == "one" and not c.partials_offset]
    for i, c in enumerate(base):
        z, rs = _EPI[i % 3]
        rows.append(RCase(c.graph, c.F, residual_name(c.kernel), c.aligned, c.plan, c.chunk, c.weighted, c.panels, z, rs))
    S = lambda vec, nv, w, u, minb, pf, panels=0: residual_name(stream_k(vec, nv, "weighted" if w else "unweighted",  # noqa: E731
                                                                         "SRC_ONE", u, minb, pf, panels))
    R = lambda vec, group, nv, w: residual_name(spmm_k(vec, group, nv, w))  # noqa: E731
    for w in (True, False):
        rows += [
            RCase("two_hubs", 7, R("float", 8, 1, w), weighted=w, z=True, row_scale=True),
            RCase("bounds", 1, R("float", 1, 1, w), weighted=w, z=True, row_scale=True),
            RCase("bounds", 16, R("float4", 4, 1, w), weighted=w, z=True, row_scale=False),
            RCase("bounds", 40, S("float4", 1, w, 4, 5, False), weighted=w, z=True, row_scale=True),
            RCase("bounds", 64, S("float4", 1, w, 4, 5, False), weighted=w, z=False, row_scale=True),
            RCase("bounds", 128, S("float2", 1, w, 8, 5, True, 2), weighted=w, panels=2, z=True, row_scale=True),
            RCase("bounds", 256, S("float4", 2, w, 4, 1, True), weighted=w, z=True, row_scale=False),
            RCase("ragged", 128, S("float", 1, w, 8, 6, True, 4), weighted=w, panels=4, z=True, row_scale=True),
            RCase("ragged", 256, S("float2", 1, w, 8, 5, True, 4), weighted=w, panels=4, z=False, row_scale=False),
        ]
    return rows


TABLE = _rows()
