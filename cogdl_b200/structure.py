"""Device-resident CSR structure in the kernels' format (int32), with everything that is derived
from the structure alone cached next to it: the hub plan and the transpose (CSC + permutation).

Why this exists: the reference re-casts `row_ptr.int(), col_indices.int()` on EVERY spmm call
(cogdl/utils/spmm_utils.py:106) and re-runs cuSPARSE csr2csc on EVERY backward of a non-symmetric
graph (cogdl/operators/spmm.py:67).  Here both are computed once per structure.

All device work goes through the C ABI (cogdl_b200._cabi); torch only owns the memory.
"""
import ctypes
from collections import OrderedDict
from typing import NamedTuple, Optional

import torch

from . import _cabi

import os

# rows with more edges than this are cut into chunks of this many edges (hub plan)
DEFAULT_CHUNK_EDGES = 64
# rows + edges streamed by one warp of the row-stream kernels (0 disables the stream form)
DEFAULT_SEG_COST = 128


_EMPTY = {}


def _ptr(t):
    """Raw device pointer of a tensor (None -> NULL).  A zero-element tensor has data_ptr() == 0;
    the C ABI treats NULL as "argument missing", so hand it a valid dummy address instead."""
    if t is None:
        return None
    if t.numel() == 0 and t.is_cuda:
        d = _EMPTY.get(t.device)
        if d is None:
            d = _EMPTY[t.device] = torch.zeros(16, dtype=torch.uint8, device=t.device)
        return ctypes.c_void_p(d.data_ptr())
    return ctypes.c_void_p(t.data_ptr())


def _stream(device):
    return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def require_cuda(*tensors):
    """No CPU fallback: fail loudly when handed a CPU tensor (the reference silently takes a
    slow torch path, cogdl/operators/spmm.py:11-40 `except Exception: csrspmm = None`)."""
    dev = None
    for t in tensors:
        if t is None:
            continue
        if not t.is_cuda:
            raise RuntimeError(
                "cogdl_b200 operators run on CUDA (sm_90a) only and have no CPU fallback; "
                f"got a tensor on {t.device}"
            )
        if dev is None:
            dev = t.device
        elif t.device != dev:
            raise RuntimeError(f"tensors on different devices: {dev} vs {t.device}")
    return dev


class HubPlan:
    """Which rows are cut into edge chunks (see cogdl_b200_hub_plan_t in include/cogdl_b200.h)."""

    def __init__(self, rowptr32, chunk_edges=DEFAULT_CHUNK_EDGES, nnz=None, seg_cost=None):
        dev = rowptr32.device
        n_rows = rowptr32.numel() - 1
        self.chunk_edges = int(chunk_edges)
        self.seg_cost = int(DEFAULT_SEG_COST if seg_cost is None else seg_cost)
        if nnz is None or n_rows == 0:
            self.seg_cost = 0
        self.device = dev
        self.segs = self.edge_row = None
        with torch.cuda.device(dev):
            counts = torch.empty(4, dtype=torch.int32, device=dev)
            _cabi.call("cogdl_b200_hub_plan_count", _ptr(rowptr32), n_rows, self.chunk_edges, self.seg_cost,
                       _ptr(counts), _stream(dev))
            n_hub, n_chunks, n_empty, n_segs = (int(v) for v in counts.tolist())  # one sync per structure
            self.n_hub_rows, self.n_chunks, self.n_empty_rows, self.n_segs = n_hub, n_chunks, n_empty, n_segs
            self.hub_rows = torch.empty(max(n_hub, 1), dtype=torch.int32, device=dev)
            self.chunks = torch.empty(max(2 * n_chunks, 2), dtype=torch.int32, device=dev)
            # one set of arrival counters per column panel of the SpMM's panel form (COGDL_B200_MAX_PANELS)
            self.counters = torch.zeros(max(n_chunks, 1) * _cabi.MAX_PANELS, dtype=torch.int32, device=dev)
            if self.seg_cost > 0 and n_segs > 0:
                self.segs = torch.empty(2 * n_segs, dtype=torch.int32, device=dev)
                self.edge_row = torch.empty(int(nnz), dtype=torch.int32, device=dev)
                _cabi.call("cogdl_b200_edge_rows", _ptr(rowptr32), n_rows, int(nnz), _ptr(self.edge_row), _stream(dev))
            else:
                self.n_segs = 0
            if n_chunks > 0 or self.n_segs > 0:
                _cabi.call("cogdl_b200_hub_plan_fill", _ptr(rowptr32), n_rows, self.chunk_edges,
                           self.seg_cost if self.segs is not None else 0, _ptr(counts), _ptr(self.hub_rows),
                           _ptr(self.chunks), _ptr(self.segs), _stream(dev))
            # hub rows by descending degree + a host copy of the degrees (row-tiered ops size their
            # block / cluster launches from it); the chunk table refers to rows, not to list positions
            self.hub_degrees_host = None
            if n_hub > 0:
                hr = self.hub_rows[:n_hub].long()
                deg = (rowptr32[hr + 1] - rowptr32[hr]).to(torch.int32)
                order = torch.argsort(deg, descending=True, stable=True)
                self.hub_rows[:n_hub] = self.hub_rows[:n_hub][order]
                self._hub_deg_np = deg[order].cpu().numpy().astype("int32")
                self.hub_degrees_host = self._hub_deg_np.ctypes.data

    def struct(self, partial_bytes=0):
        """ctypes struct for one call; partial scratch comes from torch's caching allocator.
        Returns (struct, keepalive)."""
        s = _cabi.HubPlanStruct()
        s.chunk_edges = self.chunk_edges
        s.n_hub_rows = self.n_hub_rows
        s.n_chunks = self.n_chunks
        s.hub_rows = self.hub_rows.data_ptr()
        s.chunks = self.chunks.data_ptr()
        s.counters = self.counters.data_ptr()
        s.n_empty_rows = self.n_empty_rows
        s.hub_degrees_host = self.hub_degrees_host
        if self.segs is not None:
            s.seg_cost, s.n_segs = self.seg_cost, self.n_segs
            s.segs, s.edge_row = self.segs.data_ptr(), self.edge_row.data_ptr()
        scratch = None
        if self.n_chunks > 0 and partial_bytes > 0:
            scratch = torch.empty((partial_bytes + 15) // 16 * 4, dtype=torch.float32, device=self.device)
            s.partials = scratch.data_ptr()
            s.partials_bytes = scratch.numel() * 4
        return s, scratch


class CSRStructure:
    """int32 CSR on the device + cached hub plan + cached transpose."""

    def __init__(self, rowptr32, colind32, n_cols=None, chunk_edges=DEFAULT_CHUNK_EDGES, seg_cost=None):
        dev = require_cuda(rowptr32, colind32)
        self.seg_cost = seg_cost
        if rowptr32.dtype != torch.int32 or colind32.dtype != torch.int32:
            raise ValueError("rowptr / colind must be int32 (use CSRStructure.from_int64 for Graph tensors)")
        if not (rowptr32.is_contiguous() and colind32.is_contiguous()):
            raise ValueError("rowptr / colind must be contiguous")
        self.rowptr, self.colind = rowptr32, colind32
        self.device = dev
        self.n_rows = rowptr32.numel() - 1
        self.nnz = colind32.numel()
        self.n_cols = self.n_rows if n_cols is None else int(n_cols)
        self.chunk_edges = int(chunk_edges)
        self._plan = None
        self._csc = None

    @staticmethod
    def from_int64(row_ptr, col, n_cols=None, chunk_edges=DEFAULT_CHUNK_EDGES):
        """Narrow Graph-style int64 (row_ptr, col) once, on the device."""
        dev = require_cuda(row_ptr, col)
        if row_ptr.dtype == torch.int32 and col.dtype == torch.int32:
            return CSRStructure(row_ptr.contiguous(), col.contiguous(), n_cols, chunk_edges)
        if row_ptr.dtype != torch.int64 or col.dtype != torch.int64:
            raise ValueError("row_ptr / col must both be int64 or both be int32")
        if col.numel() >= 2**31 or row_ptr.numel() >= 2**31:
            raise ValueError("graph too large for int32 indices on one device")
        row_ptr, col = row_ptr.contiguous(), col.contiguous()
        rp = torch.empty(row_ptr.numel(), dtype=torch.int32, device=dev)
        ci = torch.empty(col.numel(), dtype=torch.int32, device=dev)
        with torch.cuda.device(dev):
            _cabi.call("cogdl_b200_narrow_i64_i32", _ptr(row_ptr), _ptr(rp), row_ptr.numel(), _stream(dev))
            _cabi.call("cogdl_b200_narrow_i64_i32", _ptr(col), _ptr(ci), col.numel(), _stream(dev))
        return CSRStructure(rp, ci, n_cols, chunk_edges)

    @property
    def plan(self):
        if self._plan is None:
            self._plan = HubPlan(self.rowptr, self.chunk_edges, nnz=self.nnz, seg_cost=self.seg_cost)
        return self._plan

    def plan_struct(self, partial_bytes=0):
        """(ctypes pointer or None, keepalive) for one kernel call."""
        if self.chunk_edges <= 0:
            return None, None
        s, scratch = self.plan.struct(partial_bytes)
        return ctypes.byref(s), (s, scratch)

    def csc(self):
        """(CSRStructure of A^T, perm) with perm[q] = CSR position of CSC entry q.  Cached."""
        if self._csc is None:
            dev = self.device
            with torch.cuda.device(dev):
                colptr = torch.empty(self.n_cols + 1, dtype=torch.int32, device=dev)
                rowind = torch.empty(self.nnz, dtype=torch.int32, device=dev)
                perm = torch.empty(self.nnz, dtype=torch.int32, device=dev)
                wbytes = int(_cabi.load().cogdl_b200_csr2csc_workspace_bytes(self.nnz, self.n_cols))
                ws = torch.empty(max(wbytes, 16), dtype=torch.uint8, device=dev)
                _cabi.call("cogdl_b200_csr2csc", _ptr(self.rowptr), _ptr(self.colind), self.n_rows, self.n_cols,
                           self.nnz, _ptr(colptr), _ptr(rowind), _ptr(perm), _ptr(ws), ws.numel(), _stream(dev))
            t = CSRStructure(colptr, rowind, n_cols=self.n_rows, chunk_edges=self.chunk_edges, seg_cost=self.seg_cost)
            self._csc = (t, perm)
        return self._csc


class _Entry(NamedTuple):
    value: object
    tensors: tuple          # the key tensors, kept alive so their addresses cannot be reused under the key
    versions: tuple         # their in-place version counters when the entry was made
    nbytes: int

    def fresh(self):
        return self.versions == tuple(t._version for t in self.tensors)


class IdentityCache:
    """An LRU of values derived from tensors, keyed on the tensors' storage identity (address, sizes, device and
    whatever else the caller puts in the key).  An entry keeps its key tensors alive, and is dropped as stale once
    any of them has been modified in place.  A hit moves the entry to the end; past `cap` entries, or past
    `max_bytes` of the entries' declared sizes, the oldest entries are evicted (the newest one always stays).
    `stats["hit"]` counts hits; what counts as a miss is the caller's to say."""

    def __init__(self, cap, stats, max_bytes=None):
        self.entries = OrderedDict()
        self.cap, self.stats, self.max_bytes = cap, stats, max_bytes

    def get(self, key):
        ent = self.entries.get(key)
        if ent is None:
            return None
        if not ent.fresh():
            del self.entries[key]
            return None
        self.entries.move_to_end(key)
        self.stats["hit"] += 1
        return ent.value

    def put(self, key, tensors, value, nbytes=0):
        self.entries[key] = _Entry(value, tensors, tuple(t._version for t in tensors), nbytes)
        total = sum(e.nbytes for e in self.entries.values())
        while len(self.entries) > 1 and (len(self.entries) > self.cap
                                         or (self.max_bytes is not None and total > self.max_bytes)):
            total -= self.entries.popitem(last=False)[1].nbytes

    def clear(self):
        self.entries.clear()


# ---------------------------------------------------------------------------------------------
# Structure cache for the operator-level API, where the caller hands us bare (rowptr, colind)
# tensors (reference signature csrspmm(rowptr, colind, x, csr_data, sym), operators/spmm.py:24).
#
# Fast path: the identity lookup of IdentityCache.
#
# Slow path: the reference's own dispatch passes `graph.row_indptr.int(), graph.col_indices.int()`
# -- FRESH tensors on every call (cogdl/utils/spmm_utils.py:106) -- so identity never matches for a
# module that captured the reference `spmm` before install().  Those calls are matched by CONTENT
# against the most recent entries of the same shape (two device compares + one sync, ~tens of us)
# instead of rebuilding the int32 copy, the hub plan (three kernels + a host sync + an argsort) and
# possibly the transpose, and no entry is created for the short-lived tensors (no dead CSR copies
# pinned by the cache).  The cache is bounded by entries AND by bytes.
# ---------------------------------------------------------------------------------------------
_CONTENT_SCAN = 4
cache_stats = {"hit": 0, "content_hit": 0, "miss": 0}
_CACHE = IdentityCache(8, cache_stats, int(os.environ.get("COGDL_B200_STRUCT_CACHE_BYTES", str(8 << 30))))


def _entry_bytes(st, rp, ci):
    b = rp.numel() * rp.element_size() + ci.numel() * ci.element_size()
    if st.rowptr.data_ptr() != rp.data_ptr():
        b += st.rowptr.numel() * 4 + st.colind.numel() * 4
    return b + 4 * st.nnz  # + edge_row of the plan, roughly


def structure_for(rowptr, colind, n_cols=None):
    key = (rowptr.data_ptr(), colind.data_ptr(), rowptr.numel(), colind.numel(), str(rowptr.device),
           rowptr.dtype, n_cols)
    st = _CACHE.get(key)
    if st is not None:
        return st
    # content match against recent entries of the same shape (the `.int()`-per-call caller)
    scanned = 0
    for k in reversed(_CACHE.entries):
        if scanned >= _CONTENT_SCAN:
            break
        if k[2:5] != key[2:5] or k[6] != n_cols:
            continue
        scanned += 1
        ent = _CACHE.entries[k]
        if not ent.fresh():
            continue
        st, (rp, ci) = ent.value, ent.tensors
        a_rp = rp if rp.dtype == rowptr.dtype else (st.rowptr if rowptr.dtype == torch.int32 else None)
        a_ci = ci if ci.dtype == colind.dtype else (st.colind if colind.dtype == torch.int32 else None)
        if a_rp is None or a_ci is None:
            continue
        if torch.equal(a_rp, rowptr) and torch.equal(a_ci, colind):
            _CACHE.entries.move_to_end(k)
            cache_stats["content_hit"] += 1
            return st
    cache_stats["miss"] += 1
    st = CSRStructure.from_int64(rowptr, colind, n_cols)
    _CACHE.put(key, (rowptr, colind), st, _entry_bytes(st, rowptr, colind))
    return st


class GraphOperands(NamedTuple):
    st: CSRStructure
    val: Optional[torch.Tensor]         # edge weights in CSR order (raw: without the norms)
    out_norm: Optional[torch.Tensor]
    in_norm: Optional[torch.Tensor]
    sym: bool


def csr_order(graph):
    """(row_indptr, col_indices, raw_edge_weight) of a cogdl_b200.Graph or a cogdl.data.Graph, after putting the
    graph in CSR order.  Host tensors are fine: nothing here needs the device.

    The order is what makes it correct.  Building the CSR of a graph held as COO reorders every edge-aligned tensor
    the graph holds (its edge weights, and a cogdl.data.Graph's edge_attr) by the sort that builds it.  So the
    weights are read only once the CSR exists: a weight tensor read before would stay in COO order and pair the
    CSR's columns with other edges' weights."""
    rowptr, colind = graph.row_indptr, graph.col_indices
    return rowptr, colind, graph.raw_edge_weight


def graph_operands(graph):
    """What a graph-level entry point hands its kernels: the cached CSRStructure, the edge weights in CSR order,
    out_norm, in_norm and is_symmetric(), in that order (see csr_order).

    A cogdl_b200.Graph caches its structure on its adjacency.  A real cogdl.data.Graph filters attribute names
    (cogdl/data/data.py:352-375: a single leading underscore is stripped, only `keys` survive copy.copy in
    local_graph()), so nothing can be parked on it; its structure comes from structure_for instead.  Its
    row_indptr / col_indices are the same tensors on every call and local_graph()'s copies share their storage,
    so that is a dictionary hit per call, never a rebuild."""
    rowptr, colind, val = csr_order(graph)
    st = graph.structure() if hasattr(graph, "structure") else structure_for(rowptr, colind, graph.num_nodes)
    return GraphOperands(st, val, graph.out_norm, graph.in_norm, graph.is_symmetric())


def unsupported_operands(graph, *tensors, entry="", what="features"):
    """The error a graph-level fp32 entry point raises for operands it has no kernel for, or None: a dense grb_adj
    on the graph (ValueError), a tensor off the GPU (RuntimeError) or not float32 (TypeError).  `entry` and `what`
    name the entry point and its tensors in the message."""
    tensors = [t for t in tensors if t is not None]
    if getattr(graph, "grb_adj", None) is not None:
        return ValueError(f"{entry}: graphs carrying a dense grb_adj are not supported; use spmm")
    if not all(t.is_cuda for t in tensors):
        return RuntimeError(f"cogdl_b200.{entry}: CPU tensors are not supported (no CPU fallback); move the graph "
                            f"and {what} to an H100 device")
    if any(t.dtype != torch.float32 for t in tensors):
        return TypeError(f"{entry} takes float32 {what}, got {' and '.join(str(t.dtype) for t in tensors)}")
    return None


def clear_structure_cache():
    _CACHE.clear()
    _COMP_CACHE.clear()
    _COO_CACHE.clear()
    _RGCN_CACHE.clear()
    _MEMBER_CACHE.clear()


class Membership(NamedTuple):
    """What the readouts of one `batch` vector read: `st`, the membership CSR (B rows, one per graph, whose columns are
    that graph's nodes in ascending order); `st_t`, its transpose (N rows, one edge per node: the node's graph), with
    `perm` its permutation; `inv_count` [B], 1 / n_g in fp32 (0 for an empty graph: the mean's row scale) and
    `inv_count_node` [N], inv_count of each node's graph (the mean's backward over st_t)."""
    st: CSRStructure
    st_t: CSRStructure
    perm: torch.Tensor
    inv_count: torch.Tensor
    inv_count_node: torch.Tensor

    @property
    def num_graphs(self):
        return self.st.n_rows


# Membership cache, keyed on the storage identity, size and stride of the batch vector and the graph count asked for:
# every readout of a forward and its backward share one entry, and the entry made when the graph count is read from
# the device serves every later call on that batch without a host read.
member_cache_stats = {"hit": 0, "miss": 0}
_MEMBER_CACHE = IdentityCache(8, member_cache_stats)


def membership_for(batch, num_graphs=None):
    """The cached Membership of a graph-id vector `batch` ([N] integers on the device, node i in graph batch[i], sorted
    or not).  B = num_graphs, or max(batch) + 1 when None; graph ids without nodes are empty rows.

    Built on the device with the stable COO -> CSR sort (a sorted batch gives colind = arange(N)); the CSR's hub plan
    is built here too, and the transpose needs none, so the readouts and their backward never read the host.  Building
    reads the batch's smallest and largest id once (one host sync per batch vector, which also checks them) and the
    plan's sizes; `batch` itself is never copied to the host."""
    from .data import coo2csr_index

    require_cuda(batch)
    if batch.dim() != 1 or batch.dtype.is_floating_point or batch.dtype.is_complex or batch.dtype == torch.bool:
        raise TypeError(f"batch must be a 1-D integer tensor, got {batch.dtype} {tuple(batch.shape)}")
    key = (batch.data_ptr(), batch.numel(), tuple(batch.stride()), str(batch.device), batch.dtype,
           None if num_graphs is None else int(num_graphs))
    mb = _MEMBER_CACHE.get(key)
    if mb is not None:
        return mb
    member_cache_stats["miss"] += 1
    dev, N = batch.device, batch.numel()
    if N >= 2**31:
        raise ValueError("batch too large for int32 indices on one device")
    lo, hi = (int(v) for v in torch.stack([batch.min(), batch.max()]).tolist()) if N > 0 else (0, -1)
    B = hi + 1 if num_graphs is None else int(num_graphs)
    if lo < 0 or hi >= B:
        raise ValueError(f"graph id {lo if lo < 0 else hi} is out of range for {B} graphs")
    if B >= 2**31:
        raise ValueError(f"{B} graphs do not fit int32 indices")
    rowptr, reindex = coo2csr_index(batch, B)
    st = CSRStructure.from_int64(rowptr, reindex, n_cols=N)
    st.plan                                             # built now: its sizes are read on the host
    # The transpose needs no sort: row q is node q with its one edge, column batch[q], and perm[q] is node q's CSR
    # slot.  With one edge per row it has no hub rows, so it runs without a plan (no host read).
    perm = torch.empty(N, dtype=torch.int32, device=dev)
    perm[st.colind.long()] = torch.arange(N, dtype=torch.int32, device=dev)
    st_t = CSRStructure(torch.arange(N + 1, dtype=torch.int32, device=dev), batch.to(torch.int32).contiguous(),
                        n_cols=B, chunk_edges=0)
    st._csc = (st_t, perm)
    count = (rowptr[1:] - rowptr[:-1]).float()
    inv_count = torch.where(count > 0, 1.0 / count.clamp_min(1.0), torch.zeros_like(count))
    inv_count_node = inv_count[st_t.colind.long()].contiguous()
    mb = Membership(st, st_t, perm, inv_count, inv_count_node)
    _MEMBER_CACHE.put(key, (batch,), mb, 4 * (3 * N + 3 * B))
    return mb


class CompStructure:
    """CompGCN's typed COO (cogdl/models/nn/compgcn.py:94-151) in the form the composition aggregation reads.

    The COO is taken in the order given and never reordered in place: edges [0, E // 2) are the "in" half and
    [E // 2, E) the "out" half.  Owns
      * `csr`: the two halves stacked into one CSR of 2N rows (rows [0, N) "in", [N, 2N) "out"), built with the
        stable device COO -> CSR, so each row keeps its edges in COO order, with per-slot `type` and weight
        `w` = 1 / deg_h(row) (CompGCN's per-half row normalisation);
      * `transpose()`: the N x 2N transpose with the permuted type and weight (for dx), built on first use;
      * `by_type(T)`: the CSR with edge types as rows, per slot the stacked row, the column and the weight (for
        dR'), built on first use.
    Index bounds are checked once here (one host sync) and raise ValueError, as the reference's indexing raises
    IndexError; `max_type` lets every call check its relation table's size on the host."""

    def __init__(self, row, col, etype, num_nodes, chunk_edges=DEFAULT_CHUNK_EDGES):
        from .data import coo2csr_index

        dev = require_cuda(row, col)
        etype = etype.reshape(-1)
        E, N = row.numel(), int(num_nodes)
        if col.numel() != E or etype.numel() != E:
            raise ValueError(f"edge_index has {E} / {col.numel()} entries and the edge types {etype.numel()}")
        if 2 * N >= 2**31 or E >= 2**31:
            raise ValueError("graph too large for int32 indices on one device")
        row, col = row.to(dev, torch.int64).contiguous(), col.to(dev, torch.int64).contiguous()
        etype = etype.to(dev, torch.int64).contiguous()   # edge types may come from the host: one copy per build
        self.device, self.n_nodes, self.nnz, self.chunk_edges = dev, N, E, int(chunk_edges)
        self.max_type = -1
        if E > 0:
            lo_i, lo_t, hi_i, hi_t = (int(v) for v in torch.stack([
                torch.minimum(row.min(), col.min()), etype.min(), torch.maximum(row.max(), col.max()), etype.max()
            ]).tolist())                                  # one sync per structure
            if lo_i < 0 or hi_i >= N:
                raise ValueError(f"edge index {lo_i if lo_i < 0 else hi_i} is out of range for {N} nodes")
            if lo_t < 0:
                raise ValueError(f"edge type {lo_t} is negative")
            self.max_type = hi_t
        srow = row + N * (torch.arange(E, device=dev) >= E // 2)   # stacked row: the "out" half is rows [N, 2N)
        rowptr, reindex = coo2csr_index(srow, 2 * N)
        self.srow = srow[reindex].int()
        self.type = etype[reindex].int()
        deg = rowptr[1:] - rowptr[:-1]
        self.w = torch.repeat_interleave(1.0 / deg.float(), deg, output_size=E)
        self.csr = CSRStructure(rowptr.int(), col[reindex].int(), n_cols=N, chunk_edges=self.chunk_edges)
        self._transpose = None
        self._by_type = {}

    def transpose(self):
        """(CSRStructure of the N x 2N transpose, type, w) with type / w in the transpose's slot order."""
        if self._transpose is None:
            t, perm = self.csr.csc()
            p = perm.long()
            self._transpose = (t, self.type[p], self.w[p])
        return self._transpose

    def by_type(self, T):
        """(CSRStructure with T type rows whose colind is the stacked row, col, w) in type-then-COO slot order."""
        from .data import coo2csr_index

        ent = self._by_type.get(T)
        if ent is None:
            if self.max_type >= T:
                raise ValueError(f"edge type {self.max_type} is out of range for {T} relation rows")
            rowptr, reindex = coo2csr_index(self.type.long(), T)
            st = CSRStructure(rowptr.int(), self.srow[reindex], n_cols=2 * self.n_nodes, chunk_edges=self.chunk_edges)
            ent = self._by_type[T] = (st, self.csr.colind[reindex], self.w[reindex])
        return ent


# CompStructure cache: keyed on the storage identity and size of the (row, col, type) tensors, the node count and
# the chunk size.  Both layers of a model, and repeated predict() calls on one graph, share one entry.
comp_cache_stats = {"hit": 0, "miss": 0}
_COMP_CACHE = IdentityCache(4, comp_cache_stats)


def comp_structure_for(row, col, etype, num_nodes, chunk_edges=DEFAULT_CHUNK_EDGES):
    keys = (row, col, etype)
    key = tuple((t.data_ptr(), t.numel(), str(t.device), t.dtype) for t in keys) + (int(num_nodes), int(chunk_edges))
    cs = _COMP_CACHE.get(key)
    if cs is None:
        comp_cache_stats["miss"] += 1
        cs = CompStructure(row, col, etype, num_nodes, chunk_edges)
        _COMP_CACHE.put(key, keys, cs)
    return cs


def _coo_bounds(row, col, n_rows, n_cols):
    """Raise ValueError unless every row index is in [0, n_rows) and every column in [0, n_cols) (one host sync)."""
    if row.numel() == 0:
        return
    lo_r, lo_c, hi_r, hi_c = (int(v) for v in torch.stack([row.min(), col.min(), row.max(), col.max()]).tolist())
    if lo_r < 0 or hi_r >= n_rows:
        raise ValueError(f"row index {lo_r if lo_r < 0 else hi_r} is out of range for {n_rows} rows")
    if lo_c < 0 or hi_c >= n_cols:
        raise ValueError(f"column index {lo_c if lo_c < 0 else hi_c} is out of range for {n_cols} columns")


class CooStructure:
    """A COO index [2, E] (torch_sparse's `index` argument) in the forms the sparse products read.

    * `csr`: the (row, col)-sorted, duplicate-merged CSR (ascending unique columns per row) that the sparse x sparse
      product needs, built with two stable device sorts (by column, then by row), so entries of one (row, col) keep
      their input order; `slot[e]` is the CSR slot input entry e was merged into.  `merge(value)` sums the values of
      each slot in input order (deterministic) and `spread(g)` hands every input entry its slot's gradient.
    * `coo_csr()`: the stable COO -> CSR with duplicates kept (row order, then input order) and `reindex`, for the
      sparse x dense product; built on first use.
    Index bounds are checked once here and raise ValueError."""

    def __init__(self, index, n_rows, n_cols):
        from .data import coo2csr_index

        require_cuda(index)
        if index.dim() != 2 or index.shape[0] != 2:
            raise ValueError(f"index must be [2, E], got {tuple(index.shape)}")
        n_rows, n_cols = int(n_rows), int(n_cols)
        E = index.shape[1]
        if n_rows < 0 or n_cols < 0:
            raise ValueError(f"negative size {n_rows} x {n_cols}")
        if n_rows >= 2**31 or n_cols >= 2**31 or E >= 2**31:
            raise ValueError("sparse matrix too large for int32 indices on one device")
        dev = index.device
        row, col = index[0].to(torch.int64).contiguous(), index[1].to(torch.int64).contiguous()
        _coo_bounds(row, col, n_rows, n_cols)
        self.device, self.n_rows, self.n_cols, self.nnz_in = dev, n_rows, n_cols, E
        self._row, self._col = row, col
        self._coo_csr = None
        by_col = coo2csr_index(col, n_cols)[1]
        rowptr_all, by_row = coo2csr_index(row[by_col], n_rows)
        order = by_col[by_row]                        # input positions in (row, col, input) order
        srow, scol = row[order], col[order]
        new = torch.ones(E, dtype=torch.bool, device=dev)
        if E > 1:
            new[1:] = (srow[1:] != srow[:-1]) | (scol[1:] != scol[:-1])
        sorted_slot = torch.cumsum(new, 0) - 1
        self.nnz = int(sorted_slot[-1]) + 1 if E > 0 else 0       # one host read per structure
        self.slot = torch.empty(E, dtype=torch.int64, device=dev)
        self.slot[order] = sorted_slot
        urow = srow[new]
        rowptr = torch.searchsorted(urow, torch.arange(n_rows + 1, device=dev))
        self.csr = CSRStructure(rowptr.to(torch.int32), scol[new].to(torch.int32), n_cols=n_cols)
        # merge plan: the r-th entry (in input order) of every slot, for r = 0 .. max multiplicity - 1
        self._groups = []
        if self.nnz < E:
            first = torch.nonzero(new).view(-1)
            rank = torch.arange(E, device=dev) - first[sorted_slot]
            for r in range(int(rank.max()) + 1):
                sel = torch.nonzero(rank == r).view(-1)
                self._groups.append((order[sel], sorted_slot[sel]))
        else:
            self._order = order

    def merge(self, value):
        """[nnz] fp32 CSR values: the input values of each slot summed in input order."""
        value = value.reshape(-1)
        if not self._groups:
            return value[self._order].float().contiguous()
        out = torch.empty(self.nnz, dtype=torch.float32, device=value.device)
        src, dst = self._groups[0]
        out[dst] = value[src].float()
        for src, dst in self._groups[1:]:
            out[dst] = out[dst] + value[src].float()
        return out

    def spread(self, g):
        """Gradient of the input values from the gradient `g` [nnz] of the merged CSR values."""
        return g[self.slot]

    def coo_csr(self):
        """(CSRStructure with duplicates kept, reindex [E] int64: CSR slot -> input position)."""
        if self._coo_csr is None:
            from .data import coo2csr_index

            rowptr, reindex = coo2csr_index(self._row, self.n_rows)
            st = CSRStructure(rowptr.to(torch.int32), self._col[reindex].to(torch.int32), n_cols=self.n_cols)
            self._coo_csr = (st, reindex)
        return self._coo_csr


# CooStructure cache, keyed on the storage, size and strides of the index tensor and the matrix shape: SRGCN reuses
# one index across its heads and calls the products on it several times per forward.
coo_cache_stats = {"hit": 0, "miss": 0}
_COO_CACHE = IdentityCache(8, coo_cache_stats)


def coo_structure_for(index, n_rows, n_cols):
    key = (index.data_ptr(), tuple(index.shape), tuple(index.stride()), str(index.device), index.dtype, int(n_rows),
           int(n_cols))
    cs = _COO_CACHE.get(key)
    if cs is None:
        coo_cache_stats["miss"] += 1
        cs = CooStructure(index, n_rows, n_cols)
        _COO_CACHE.put(key, (index,), cs)
    return cs


class RgcnStructure:
    """R-GCN's typed CSR: a graph's CSRStructure `st` with its edge types `type` (int32, in CSR slot order), in the
    form the fan-out aggregation reads.  Built from the types a graph holds once its CSR exists (graph_operands, then
    edge_attr), so every type stays paired with its edge.  Owns, built on first use:
      * `transpose()`: the cached transpose of `st`, the types permuted to it and the permutation (the feature gradient);
      * `by_type(T)`: the CSR with T type rows whose colind is the CSR slot, in slot order (the coefficient gradient
        reduces per-slot products over it with the SpMM).
    The types are checked once here (one host sync): a negative type raises ValueError, and `max_type` lets every call
    check its coefficient table's size on the host."""

    def __init__(self, st, etype):
        etype = etype.reshape(-1)
        if etype.numel() != st.nnz:
            raise ValueError(f"edge_attr holds {etype.numel()} edge types, the graph has {st.nnz} edges")
        if etype.dtype.is_floating_point or etype.dtype.is_complex or etype.dtype == torch.bool:
            raise TypeError(f"edge types must be integers, got {etype.dtype}")
        self.st, self.device, self.nnz = st, st.device, st.nnz
        etype = etype.to(st.device, torch.int64)
        self.max_type = -1
        if st.nnz > 0:
            lo, hi = (int(v) for v in torch.stack([etype.min(), etype.max()]).tolist())   # one sync per structure
            if lo < 0:
                raise ValueError(f"edge type {lo} is negative")
            if hi >= 2**31:
                raise ValueError(f"edge type {hi} does not fit int32")
            self.max_type = hi
        self.type = etype.to(torch.int32).contiguous()
        self._transpose = None
        self._by_type = {}

    def transpose(self):
        """(CSRStructure of A^T, type in its slot order, perm [nnz] int64: CSR slot of each transpose slot)."""
        if self._transpose is None:
            t, perm = self.st.csc()
            p = perm.long()
            self._transpose = (t, self.type[p].contiguous(), p)
        return self._transpose

    def by_type(self, T):
        """CSRStructure with T rows (types) whose colind lists the CSR slots of that type in slot order."""
        from .data import coo2csr_index

        st = self._by_type.get(T)
        if st is None:
            if self.max_type >= T:
                raise ValueError(f"edge type {self.max_type} is out of range for {T} relations")
            rowptr, reindex = coo2csr_index(self.type.long(), T)
            st = self._by_type[T] = CSRStructure(rowptr.int(), reindex.int(), n_cols=self.nnz)
        return st


# RgcnStructure cache, keyed on the storage identity of the graph structure's int32 CSR and of the edge-type tensor:
# both layers of a model, and repeated predict() calls on one graph, share one entry.
rgcn_cache_stats = {"hit": 0, "miss": 0}
_RGCN_CACHE = IdentityCache(4, rgcn_cache_stats)


def rgcn_structure_for(st, etype):
    keys = (st.rowptr, st.colind, etype)
    key = tuple((t.data_ptr(), t.numel(), str(t.device), t.dtype) for t in keys)
    rs = _RGCN_CACHE.get(key)
    if rs is None or rs.st is not st:
        rgcn_cache_stats["miss"] += 1
        rs = RgcnStructure(st, etype)
        _RGCN_CACHE.put(key, keys, rs)
    return rs
