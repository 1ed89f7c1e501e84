"""One row per dispatch branch of cogdl_b200_spmm_residual_dcoef_f32 (gin.cu) and cogdl_b200_spmm_accum_f32
(spmm_accum.cu): every row of tests/spmm_residual_table.py under the device-coefficient kernel and under the
accumulating kernel of the same instantiation, plus C = 47 rows (not a multiple of 4) for the scalar two-vector loop.
The accumulating rows switch between the last hop and an inner one, and between ACC updated in place and read from a
separate buffer.  test_gpu_gin_grand.py runs every row; test_cpu_gin_grand_inventory.py checks that the rows cover
every kernel compiled into gin.o and spmm_accum.o and name no other.  Plain Python, no torch."""
from dataclasses import dataclass

from tests.dispatch_table import stream_k
from tests.spmm_residual_table import TABLE as RESIDUAL


@dataclass(frozen=True)
class GCase:
    epi: str                # "dcoef" (gin.cu) or "accum" (spmm_accum.cu)
    graph: str              # a name in tests/graphs.py CASES, or "bounds": boundary_csr(chunk)
    F: int
    kernel: str             # exact cogdl_b200_last_kernel() after the call
    aligned: bool = True    # False: X is a view one element past an aligned allocation
    plan: str = "default"   # none | chunks | default, as in dispatch_table.Case
    chunk: int = 64
    weighted: bool = True
    panels: int = 0
    z: bool = True          # dcoef: Z given
    row_scale: bool = False
    last: bool = False      # accum: the last hop (ACC scaled, Xn not stored)
    in_place: bool = True   # accum: ACC_in is ACC itself (else a separate buffer)

    @property
    def id(self):
        s = f"{self.epi}-{self.graph}-F{self.F}-{self.plan}-{'w' if self.weighted else 'u'}"
        if self.epi == "dcoef":
            s += "-z" if self.z else "-noz"
        else:
            s += ("-last" if self.last else "-hop") + ("" if self.in_place else "-accin")
        s += "-rs" if self.row_scale else ""
        s += "" if self.aligned else "-misaligned"
        return s + (f"-P{self.panels}" if self.panels else "")


def epi_name(residual_kernel, epi):
    """The launch's name for the residual one: the same instantiation parameters, except that the device-coefficient
    form runs the 64-float panel loop (float2, U=8) at 4 blocks per SM."""
    k = residual_kernel.replace("::spmm_residual_kernel<", f"::spmm_{epi}_kernel<").replace(
        "::stream_residual_kernel<", f"::stream_{epi}_kernel<")
    if epi == "dcoef":
        k = k.replace("<float2,NV=1,weighted,SRC_ONE,U=8,MINB=5,prefetch>", "<float2,NV=1,weighted,SRC_ONE,U=8,MINB=4,prefetch>")
        k = k.replace("<float2,NV=1,unweighted,SRC_ONE,U=8,MINB=5,prefetch>",
                      "<float2,NV=1,unweighted,SRC_ONE,U=8,MINB=4,prefetch>")
    return k


_ACC = [(False, True), (True, False), (True, True), (False, False)]   # (last, in_place)


def _rows():
    rows = []
    for i, c in enumerate(RESIDUAL):
        rows.append(GCase("dcoef", c.graph, c.F, epi_name(c.kernel, "dcoef"), c.aligned, c.plan, c.chunk, c.weighted,
                          c.panels, c.z, c.row_scale))
        last, in_place = _ACC[i % 4]
        rows.append(GCase("accum", c.graph, c.F, epi_name(c.kernel, "accum"), c.aligned, c.plan, c.chunk, c.weighted,
                          c.panels, True, c.row_scale, last, in_place))
    for w in (True, False):
        nv2 = lambda epi: epi_name(stream_k("float", 2, "weighted" if w else "unweighted", "SRC_ONE", 4, 1, True)  # noqa: E731
                                   .replace("::stream_kernel<", "::stream_residual_kernel<"), epi)
        rows += [
            GCase("dcoef", "two_hubs", 47, nv2("dcoef"), weighted=w, z=True, row_scale=True),
            GCase("accum", "two_hubs", 47, nv2("accum"), weighted=w, row_scale=True, last=True, in_place=False),
            GCase("accum", "bounds", 47, nv2("accum"), weighted=w, row_scale=False, last=False, in_place=True),
        ]
    return rows


TABLE = _rows()
