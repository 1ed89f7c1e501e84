"""Graph / Adjacency with the attribute surface of `cogdl.data.Graph` that the hot path touches
(cogdl/data/data.py:134-451 Adjacency, :474-959 Graph), for use where the `cogdl` package is not
importable (the GPU machine) and as the place where device-side structure caches live.

Same names and meaning: row_indptr / col_indices / edge_index / edge_weight / raw_edge_weight / edge_attr /
in_norm / out_norm / is_symmetric / sym_norm / row_norm / col_norm / local_graph /
add_remaining_self_loops / degrees / num_nodes / num_edges / to(device).  Index tensors are int64
as in the reference; the kernels' int32 copy, the hub plan and the transpose are cached in
`Adjacency.structure()` and shared by `local_graph()` copies (which only swap weights).

Not a port: storage is CSR-first, COO rows are derived on demand, and COO->CSR runs on the device
(cogdl_b200_coo2csr_index) when the tensors are CUDA tensors.
"""
import copy
from contextlib import contextmanager

import torch

from .structure import CSRStructure


def coo2csr_index(row, num_nodes):
    """(row_ptr [num_nodes+1] int64, reindex [E] int64): stable counting sort by row -- the edge
    order every edge-aligned tensor lives in (reference: cogdl/utils/graph_utils.py:133-142 ->
    cogdl/operators/sample/sample.cpp:234-270, single-thread CPU even for CUDA graphs)."""
    row = row.long().contiguous()
    if row.is_cuda:
        from . import _cabi
        from .structure import _ptr, _stream

        dev = row.device
        nnz = row.numel()
        with torch.cuda.device(dev):
            row_ptr = torch.empty(num_nodes + 1, dtype=torch.int64, device=dev)
            reindex = torch.empty(nnz, dtype=torch.int64, device=dev)
            wbytes = int(_cabi.load().cogdl_b200_coo2csr_workspace_bytes(nnz, num_nodes))
            ws = torch.empty(max(wbytes, 16), dtype=torch.uint8, device=dev)
            _cabi.call("cogdl_b200_coo2csr_index", _ptr(row), nnz, num_nodes, _ptr(row_ptr), _ptr(reindex),
                       _ptr(ws), ws.numel(), _stream(dev))
        return row_ptr, reindex
    # host tensors: graph construction is host logic (stable sort == counting sort order)
    reindex = torch.sort(row, stable=True).indices
    counts = torch.bincount(row, minlength=num_nodes)
    row_ptr = torch.zeros(num_nodes + 1, dtype=torch.int64)
    torch.cumsum(counts, 0, out=row_ptr[1:])
    return row_ptr, reindex


def _degrees_from_ptr(row_ptr):
    return (row_ptr[1:] - row_ptr[:-1]).float()


class Adjacency:
    def __init__(self, row=None, col=None, row_ptr=None, weight=None, num_nodes=None, attr=None):
        self.row, self.col, self.row_ptr, self.weight = row, col, row_ptr, weight
        self.attr = attr                   # edge-aligned, reordered with the edges (reference data.py:279-287)
        self.__num_nodes__ = num_nodes
        self.__normed__ = None
        self.__in_norm__ = self.__out_norm__ = None
        self.__symmetric__ = True          # reference default, data.py:146
        self._structure = None             # CSRStructure cache (shared with local copies)

    # ----------------------------------------------------------------- sizes
    @property
    def num_nodes(self):
        if self.__num_nodes__ is not None:
            return self.__num_nodes__
        if self.row_ptr is not None:
            return self.row_ptr.shape[0] - 1
        self.__num_nodes__ = int(max(self.row.max().item(), self.col.max().item())) + 1
        return self.__num_nodes__

    @property
    def num_edges(self):
        return self.col.shape[0]

    @property
    def device(self):
        return self.col.device

    # ----------------------------------------------------------------- CSR
    def _to_csr(self):
        row_ptr, reindex = coo2csr_index(self.row, self.num_nodes)
        self.row_ptr = row_ptr
        self.row, self.col = self.row[reindex], self.col[reindex]
        if self.weight is not None:
            self.weight = self.weight[reindex]
        if self.attr is not None:
            self.attr = self.attr[reindex]
        self._structure = None

    @property
    def row_indptr(self):
        if self.row_ptr is None:
            self._to_csr()
        return self.row_ptr

    @property
    def edge_index(self):
        if self.row is None:
            n = self.row_ptr.shape[0] - 1
            counts = self.row_ptr[1:] - self.row_ptr[:-1]
            self.row = torch.repeat_interleave(torch.arange(n, device=self.row_ptr.device), counts)
        return self.row, self.col

    def structure(self):
        """int32 CSR + hub plan + transpose on the device, built once per structure."""
        if self._structure is None:
            self._structure = CSRStructure.from_int64(self.row_indptr, self.col, n_cols=self.num_nodes)
        return self._structure

    def degrees(self):
        return _degrees_from_ptr(self.row_indptr)

    # ----------------------------------------------------------------- weights / norms
    def set_weight(self, weight):
        # reference data.py:150-154: a user-set weight clears the norms and the symmetric flag
        self.weight = weight
        self.__normed__ = None
        self.__in_norm__ = self.__out_norm__ = None
        self.__symmetric__ = False

    def get_weight(self, indicator=None):
        if self.weight is None or self.weight.shape[0] != self.col.shape[0]:
            self.weight = torch.ones(self.num_edges, device=self.device)
        weight = self.weight
        if indicator is not None:
            return weight
        # reference data.py:163-173 (note: out_norm overwrites in_norm there too)
        if self.__in_norm__ is not None:
            weight = self.__in_norm__[self.edge_index[0]].view(-1)
        if self.__out_norm__ is not None:
            weight = self.__out_norm__[self.col].view(-1)
        return weight

    def is_symmetric(self):
        return self.__symmetric__

    def set_symmetric(self, val):
        assert val in (True, False)
        self.__symmetric__ = val

    def _normalize(self, norm):
        if self.__normed__:
            return
        if self.row is None and norm != "col":
            # CSR-only graph: keep weights raw, put the scaling in in/out norms (data.py:240-258)
            deg = _degrees_from_ptr(self.row_ptr)
            s = deg.pow(-0.5 if norm == "sym" else -1)
            s[torch.isinf(s)] = 0
            self.__in_norm__ = s.view(-1, 1)
            self.__out_norm__ = s.view(-1, 1) if norm == "sym" else None
        else:
            self.edge_index  # materialise COO rows if the graph was CSR-only
            # COO present: bake the scaling into the edge weights (data.py:260-274)
            w = self.get_weight("raw")
            row, col = self.row, self.col
            n = self.num_nodes
            if norm == "sym":
                d = torch.zeros(n, device=w.device).scatter_add_(0, row, torch.ones_like(w))
                s = d.pow(-0.5)
                s[torch.isinf(s)] = 0
                self.weight = s[col] * w * s[row]
            else:
                key = row if norm == "row" else col
                d = torch.zeros(n, device=w.device).scatter_add_(0, key, torch.ones_like(w))
                s = d.pow(-1)
                s[torch.isinf(s)] = 0
                self.weight = w * s[key]
        self.__normed__ = norm

    def sym_norm(self):
        self._normalize("sym")

    def row_norm(self):
        self._normalize("row")
        if self.row is not None:
            self.__symmetric__ = False

    def col_norm(self):
        self._normalize("col")
        self.__symmetric__ = False

    def add_remaining_self_loops(self):
        """Drop existing self loops, append one (i, i) per node with weight 1, rebuild the CSR
        (reference data.py:175-191 / graph_utils.py:40-69)."""
        row, col = self.edge_index
        n = self.num_nodes
        w = self.get_weight("raw")
        mask = row != col
        loop = torch.arange(n, dtype=row.dtype, device=row.device)
        loop_w = torch.ones(n, dtype=w.dtype, device=w.device)
        inv = ~mask
        if inv.any():
            loop_w[row[inv]] = w[inv]
        self.row = torch.cat([row[mask], loop])
        self.col = torch.cat([col[mask], loop])
        self.weight = torch.cat([w[mask], loop_w])
        if self.attr is not None:          # a new loop's attribute is 0, an existing loop keeps its own
            loop_a = torch.zeros((n,) + tuple(self.attr.shape[1:]), dtype=self.attr.dtype, device=self.attr.device)
            if inv.any():
                loop_a[row[inv]] = self.attr[inv]
            self.attr = torch.cat([self.attr[mask], loop_a])
        self.row_ptr = None
        self._to_csr()

    # ----------------------------------------------------------------- misc
    def to(self, device):
        for k in ("row", "col", "row_ptr", "weight", "attr", "__in_norm__", "__out_norm__"):
            v = getattr(self, k)
            if torch.is_tensor(v):
                setattr(self, k, v.to(device))
        self._structure = None
        return self

    def __copy__(self):
        # local_graph(): new tensor OBJECTS sharing storage (copy.copy(t).data_ptr() == t.data_ptr()),
        # same device structure cache -- only the weight is expected to be swapped.
        out = Adjacency.__new__(Adjacency)
        out.__dict__.update(self.__dict__)
        return out


class Graph:
    def __init__(self, x=None, y=None, edge_index=None, edge_weight=None, row_ptr=None, col=None, num_nodes=None,
                 edge_attr=None, **kw):
        self.x, self.y = x, y
        self.grb_adj = None
        if num_nodes is None and x is not None:
            num_nodes = x.shape[0]
        if edge_index is not None:
            row, col_ = edge_index
            self._adj = Adjacency(row=row, col=col_, weight=edge_weight, num_nodes=num_nodes, attr=edge_attr)
        else:
            self._adj = Adjacency(col=col, row_ptr=row_ptr, weight=edge_weight, num_nodes=num_nodes, attr=edge_attr)
        self.__temp_adj_stack__ = []
        for k, v in kw.items():
            setattr(self, k, v)

    # structure
    @property
    def num_nodes(self):
        return self._adj.num_nodes

    @property
    def num_edges(self):
        return self._adj.num_edges

    @property
    def device(self):
        return self._adj.device

    @property
    def row_indptr(self):
        return self._adj.row_indptr

    @property
    def col_indices(self):
        if self._adj.row_ptr is None:
            self._adj._to_csr()
        return self._adj.col

    @property
    def edge_index(self):
        return self._adj.edge_index

    def structure(self):
        return self._adj.structure()

    def degrees(self):
        return self._adj.degrees()

    # weights
    @property
    def edge_weight(self):
        return self._adj.get_weight()

    @edge_weight.setter
    def edge_weight(self, w):
        self._adj.set_weight(w)

    @property
    def raw_edge_weight(self):
        return self._adj.get_weight("raw")

    @property
    def edge_attr(self):
        """Edge-aligned attributes (R-GCN / CompGCN edge types), in the graph's current edge order: building the CSR
        of a graph held as COO reorders them with the edges, as it reorders the weights."""
        return self._adj.attr

    @edge_attr.setter
    def edge_attr(self, attr):
        self._adj.attr = attr

    @property
    def in_norm(self):
        return self._adj.__in_norm__

    @property
    def out_norm(self):
        return self._adj.__out_norm__

    def is_symmetric(self):
        return self._adj.is_symmetric()

    def set_symmetric(self):
        self._adj.set_symmetric(True)

    def set_asymmetric(self):
        self._adj.set_symmetric(False)

    def sym_norm(self):
        self._adj.sym_norm()

    def row_norm(self):
        self._adj.row_norm()

    def col_norm(self):
        self._adj.col_norm()

    def normalize(self, key="sym"):
        assert key in ("row", "sym", "col")
        getattr(self, f"{key}_norm")()

    def add_remaining_self_loops(self):
        self._adj.add_remaining_self_loops()
        return self

    @contextmanager
    def local_graph(self):
        """Temporary weight swaps (reference data.py:594-604): a shallow copy of the adjacency is
        active inside the block and discarded afterwards."""
        self.__temp_adj_stack__.append(self._adj)
        self._adj = copy.copy(self._adj)
        try:
            yield
        finally:
            self._adj = self.__temp_adj_stack__.pop()

    def to(self, device):
        for k, v in list(self.__dict__.items()):
            if torch.is_tensor(v):
                setattr(self, k, v.to(device))
        self._adj.to(device)
        return self

    def cuda(self, device="cuda"):
        return self.to(device)
