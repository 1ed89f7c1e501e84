"""One row per dispatch branch of cogdl_b200_label_prop_f32 (label_prop.cu): every row of tests/spmm_residual_table.py
under the label-propagation kernel of the same instantiation, with the clamp and the pinned rows switched on and off
across the rows, and further rows for C = 47 (the products label width, not a multiple of 4) and every epilogue
combination on the boundary-degree graph.  test_gpu_label_prop.py runs every row; test_cpu_label_prop_inventory.py
checks that the rows cover every kernel compiled into label_prop.o and name no other.  Plain Python, no torch."""
from dataclasses import dataclass

from tests.dispatch_table import spmm_k, stream_k
from tests.spmm_residual_table import TABLE as RESIDUAL


@dataclass(frozen=True)
class LCase:
    graph: str              # a name in tests/graphs.py CASES, or "bounds": boundary_csr(chunk)
    F: int
    kernel: str             # exact cogdl_b200_last_kernel() after the call
    aligned: bool = True    # False: X is a view one element past an aligned allocation
    plan: str = "default"   # none | chunks | default, as in dispatch_table.Case
    chunk: int = 64
    weighted: bool = True
    panels: int = 0
    z: bool = True          # Z given
    row_scale: bool = False
    clamp: bool = False     # clamp to [CLAMP_LO, CLAMP_HI] (test_gpu_label_prop.py)
    pin: bool = False       # about a third of the rows pinned to Z (needs Z)

    @property
    def id(self):
        s = f"{self.graph}-F{self.F}-{self.plan}-{'w' if self.weighted else 'u'}"
        s += "-z" if self.z else "-noz"
        s += "-rs" if self.row_scale else ""
        s += "-clamp" if self.clamp else ""
        s += "-pin" if self.pin else ""
        s += "" if self.aligned else "-misaligned"
        return s + (f"-P{self.panels}" if self.panels else "")


def labelprop_name(residual_kernel):
    """The label-propagation launch's name for the residual one: the same instantiation parameters (MINB included)."""
    return residual_kernel.replace("::spmm_residual_kernel<", "::spmm_labelprop_kernel<").replace(
        "::stream_residual_kernel<", "::stream_labelprop_kernel<")


_POST = [(True, False), (False, True), (True, True), (False, False)]   # (clamp, pin)


def _rows():
    rows = []
    for i, c in enumerate(RESIDUAL):
        clamp, pin = _POST[i % 3]          # (False, False): the boundary-graph rows below
        if not c.z:                         # no Z to pin to: clamp
            clamp, pin = True, False
        rows.append(LCase(c.graph, c.F, labelprop_name(c.kernel), c.aligned, c.plan, c.chunk, c.weighted, c.panels,
                          c.z, c.row_scale, clamp, pin))
    L = lambda k: labelprop_name(k.replace("::spmm_kernel<", "::spmm_residual_kernel<").replace(  # noqa: E731
        "::stream_kernel<", "::stream_residual_kernel<"))
    nv2 = lambda w: L(stream_k("float", 2, "weighted" if w else "unweighted", "SRC_ONE", 4, 1, True))  # noqa: E731
    for w in (True, False):
        rows += [
            LCase("two_hubs", 47, nv2(w), weighted=w, z=True, row_scale=True, clamp=True, pin=True),
            LCase("two_hubs", 47, L(spmm_k("float", 32, 2, w)), plan="chunks", weighted=w, z=True, clamp=False, pin=True),
            LCase("ragged", 47, nv2(w), weighted=w, z=True, row_scale=False, clamp=True, pin=False),
        ]
        for clamp, pin in _POST:
            rows.append(LCase("bounds", 47, nv2(w), weighted=w, z=True, row_scale=True, clamp=clamp, pin=pin))
    return rows


TABLE = _rows()
