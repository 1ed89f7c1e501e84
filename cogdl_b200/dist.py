"""Node-range partitioned SpMM across the GPUs of one box (SURVEY 8e; new functionality -- the
reference's sparse ops are single-GPU only, SURVEY 2.3/2.4).

One process per GPU (torch.distributed, NCCL over NVLink 5 / NVSwitch).  Rank p owns a contiguous
range of destination rows [lo_p, hi_p) of A together with the matching rows of X and Y.  Output
rows are independent, so the only coupling is the gather of X rows owned by other ranks:

    setup (once per structure)   columns outside [lo_p, hi_p) are renumbered to n_local + k where k
                                 indexes this rank's sorted, de-duplicated halo list; the halo lists
                                 are exchanged so every owner knows which of its rows each peer needs
    step                         pack   : send_buf = X_local[send_index]          (gather kernel)
                                 move   : all-to-all of the packed rows over NVLink (NCCL)
                                 compute: Y_local = A_local @ [X_local ; X_halo]   (two-source SpMM,
                                          cogdl_b200_spmm_csr_f32_2src -- no concatenation copy)

This is the pull form of the boundary exchange and the default: there is no reduction on the data
path, a row's sum is completed by exactly one rank.

The push form named in the north star ("reduce of boundary partial sums") is `PushSpMM` below: rank
p keeps the COLUMN slice A[:, lo_p:hi_p], multiplies it by its own X shard, and the partial sums of
destination rows owned by other ranks are reduce-scattered -- a ragged all-to-all of the packed
boundary rows followed by an in-order add that is folded into the interior SpMM (the received
partials are a second source of a two-source SpMM with unit weights).  Same order of bytes as the
pull form ((#distinct boundary rows) * 4F per rank), two SpMM launches instead of one; kept for
comparison (opt-in).
"""
import torch
import torch.distributed as dist

from . import synth
from .structure import CSRStructure


def balanced_row_ranges(row_ptr, parts):
    """Contiguous row ranges balanced by cost = nnz + rows (power-law graphs: NOT by row count)."""
    n = row_ptr.numel() - 1
    cost = row_ptr.to(torch.int64) + torch.arange(n + 1, device=row_ptr.device, dtype=torch.int64)
    total = int(cost[-1])
    targets = torch.tensor([total * k // parts for k in range(parts + 1)], device=row_ptr.device, dtype=torch.int64)
    bounds = torch.searchsorted(cost, targets).clamp_(max=n)
    bounds[0], bounds[-1] = 0, n
    return [int(b) for b in bounds.tolist()]


class LocalPartition:
    """What one rank holds of the partitioned graph (index arithmetic only; device agnostic)."""

    def __init__(self, rank, world, bounds, row_ptr_local, col_global, val_local):
        self.rank, self.world, self.bounds = rank, world, list(bounds)
        lo, hi = bounds[rank], bounds[rank + 1]
        self.lo, self.hi, self.n_local = lo, hi, hi - lo
        col_global = col_global.to(torch.int64)
        is_local = (col_global >= lo) & (col_global < hi)
        remote = col_global[~is_local]
        self.halo = torch.unique(remote)                                # sorted global ids this rank must fetch
        self.n_halo = int(self.halo.numel())
        col_local = torch.empty_like(col_global)
        col_local[is_local] = col_global[is_local] - lo
        col_local[~is_local] = self.n_local + torch.searchsorted(self.halo, remote)
        self.row_ptr = row_ptr_local
        self.col = col_local
        self.val = val_local
        self.nnz_local = int(col_global.numel())
        bt = torch.tensor(self.bounds, device=self.halo.device, dtype=torch.int64)
        owner = torch.searchsorted(bt, self.halo, right=True) - 1       # owner rank of every halo row
        self.recv_counts = torch.bincount(owner, minlength=world).tolist()   # rows I receive from each rank
        self.halo_owner_local = self.halo - bt[owner]                   # row index inside the owner's shard
        # peer encoding (fused NVLink gather): remote column -> n_local + (owner << shift | row in owner's shard)
        max_rows = max(bounds[k + 1] - bounds[k] for k in range(world))
        self.peer_shift = max(1, int(max_rows - 1).bit_length())
        if self.n_local + (world << self.peer_shift) >= 2**31:
            self.col_peer = None      # does not fit int32: only the halo form is available
        else:
            rem_owner = torch.searchsorted(bt, remote, right=True) - 1
            col_peer = col_local.clone()
            col_peer[~is_local] = self.n_local + (rem_owner << self.peer_shift) + (remote - bt[rem_owner])
            self.col_peer = col_peer


def exchange_index_lists(part, group=None, comm_device=None):
    """Tell every owner which of its rows this rank needs.  Returns (send_index, send_counts):
    send_index = my local row ids to pack, concatenated in peer order.  comm_device: where the
    (small) index lists live during the exchange -- NCCL needs CUDA tensors even when the
    partition was computed on the host."""
    world = part.world
    dev = part.halo.device if comm_device is None else comm_device
    recv_counts = torch.tensor(part.recv_counts, dtype=torch.int64, device=dev)
    send_counts = torch.empty(world, dtype=torch.int64, device=dev)
    _all_to_all(send_counts, recv_counts, [1] * world, [1] * world, group)
    send_counts_l = [int(v) for v in send_counts.tolist()]
    send_index = torch.empty(sum(send_counts_l), dtype=torch.int64, device=dev)
    _all_to_all(send_index, part.halo_owner_local.to(dev).contiguous(), send_counts_l, part.recv_counts, group)
    return send_index.to(part.halo.device), send_counts_l


def _all_to_all(out, inp, out_splits, in_splits, group=None):
    """all_to_all_single on NCCL; point-to-point batch on backends without it (gloo in CPU tests)."""
    backend = dist.get_backend(group)
    if backend == "nccl":
        dist.all_to_all_single(out, inp, output_split_sizes=out_splits, input_split_sizes=in_splits, group=group)
        return
    if out.is_cuda or inp.is_cuda:
        # gloo has no device point-to-point: stage through the host (tests that run two ranks on one GPU;
        # a real multi-GPU job uses NCCL above)
        out_h = torch.empty(out.shape, dtype=out.dtype)
        _all_to_all(out_h, inp.cpu(), out_splits, in_splits, group)
        out.copy_(out_h)
        return
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    outs = list(out.split(out_splits)) if sum(out_splits) else [out[:0]] * world
    ins = list(inp.split(in_splits)) if sum(in_splits) else [inp[:0]] * world
    outs[rank].copy_(ins[rank])
    ops = []
    for peer in range(world):
        if peer == rank:
            continue
        if in_splits[peer]:
            ops.append(dist.P2POp(dist.isend, ins[peer].contiguous(), peer, group))
        if out_splits[peer]:
            ops.append(dist.P2POp(dist.irecv, outs[peer], peer, group))
    if ops:
        for w in dist.batch_isend_irecv(ops):
            w.wait()


class PartitionedSpMM:
    """Per-rank state + the step  y_local = A_local @ X  of the node-range partitioned SpMM.

    mode "p2p"  (default on CUDA): feature shards live in torch symmetric memory; the SpMM kernel
                reads remote rows straight from the owner's HBM over NVLink
                (cogdl_b200_spmm_csr_f32_peers) -- gather and compute are ONE kernel.
    mode "nccl": pack (gather kernel) -> all_to_all_single -> two-source SpMM on [X_local ; X_halo].
    """

    def __init__(self, part: LocalPartition, device, group=None, global_nnz=None, description="", mode=None):
        self.part, self.device, self.group = part, device, group
        self.n_local, self.n_halo, self.nnz_local = part.n_local, part.n_halo, part.nnz_local
        self.global_nnz = global_nnz
        self._desc = description
        self.world = part.world
        nccl = dist.get_backend(group) == "nccl"
        if mode is None:
            mode = "p2p" if (device.type == "cuda" and nccl and part.col_peer is not None) else "nccl"
        if mode not in ("p2p", "nccl"):
            raise ValueError(f"PartitionedSpMM mode must be 'p2p' or 'nccl', got {mode!r} (the push form is dist.PushSpMM)")
        self.mode = mode
        self.x_local = None
        self._symm = None
        self._symm_by_F = {}
        if mode == "p2p":
            self.exchange = "fused: remote rows read from peer HBM inside the SpMM kernel (symmetric memory, NVLink P2P)"
            self.st = CSRStructure.from_int64(part.row_ptr.to(device), part.col_peer.to(device),
                                              n_cols=part.n_local)
            self.st.plan
            self.val = None if part.val is None else part.val.to(device).float().contiguous()
            rows = torch.tensor([part.n_local], device=device, dtype=torch.int64)
            dist.all_reduce(rows, op=dist.ReduceOp.MAX, group=group)
            self._symm_rows = int(rows)
            return
        comm_dev = device if nccl else None
        self.send_index, self.send_counts = exchange_index_lists(part, group, comm_dev)
        self.recv_counts = part.recv_counts
        self.exchange = "NCCL all_to_all_single of packed halo rows" if nccl else "p2p isend/irecv (gloo)"
        if device.type == "cuda":
            self.st = CSRStructure.from_int64(part.row_ptr.to(device), part.col.to(device),
                                              n_cols=part.n_local + part.n_halo)
            self.st.plan
            self.val = None if part.val is None else part.val.to(device).float().contiguous()
            self.send_index32 = self.send_index.to(device).to(torch.int32).contiguous()

    def describe(self):
        return self._desc

    # ------------------------------------------------------------------ p2p form
    def features(self, F):
        """The local feature shard [n_local, F] inside symmetric memory (write X here; peers read it).
        One symmetric buffer per feature width, kept for the life of the object (a multi-layer model
        alternates widths; re-allocating + re-rendezvousing while a slower peer's kernel still reads
        the old shard would be a use-after-free across ranks)."""
        ent = self._symm_by_F.get(F)
        if ent is None:
            import ctypes

            import torch.distributed._symmetric_memory as symm

            buf = symm.empty((self._symm_rows, F), dtype=torch.float32, device=self.device)
            hdl = symm.rendezvous(buf, self.group if self.group is not None else dist.group.WORLD)
            ptrs = (ctypes.c_void_p * self.world)(*[int(p) for p in hdl.buffer_ptrs])
            ent = self._symm_by_F[F] = (buf, hdl, ptrs)
        self._symm = ent
        return ent[0][: self.n_local]

    def release(self):
        """Barrier that must precede ANY write to a shard returned by features(): a faster rank may
        only overwrite its shard once every peer's previous SpMM kernel has finished gathering from
        it (write-after-read across ranks).  spmm(x) does this itself when it copies x in."""
        if self._symm is not None:
            self._symm[1].barrier(channel=1)

    def spmm_p2p(self):
        """Y_local from the features currently in the symmetric shards (barrier, then ONE kernel)."""
        import ctypes

        from .operators._raw import _launch, _scratch, _spmm_out
        from .structure import _ptr

        buf, hdl, ptrs = self._symm
        hdl.barrier()   # every rank's shard is written before anyone gathers from it
        st = self.st
        y = _spmm_out(st, self.val, buf)
        _launch("cogdl_b200_spmm_csr_f32_peers", st, _scratch("spmm", st, buf.shape[1]), _ptr(st.rowptr),
                _ptr(st.colind), _ptr(self.val), _ptr(buf), self.n_local, ctypes.cast(ptrs, ctypes.c_void_p), self.world,
                self.part.peer_shift, _ptr(y), st.n_rows, buf.shape[1])
        return y

    # ------------------------------------------------------------------ nccl (halo) form: three stages
    def pack(self, x_local):
        if x_local.is_cuda:
            from .operators._raw import gather_rows_raw

            return gather_rows_raw(self.send_index32, x_local)
        return x_local.index_select(0, self.send_index)   # host tensors: gloo plumbing tests only

    def exchange_rows(self, send_buf, F):
        halo = torch.empty((self.n_halo, F), dtype=send_buf.dtype, device=send_buf.device)
        _all_to_all(halo.view(-1), send_buf.view(-1), [c * F for c in self.recv_counts],
                    [c * F for c in self.send_counts], self.group)
        return halo

    def local_spmm(self, x_local, x_halo):
        from .operators._raw import spmm_2src_raw

        return spmm_2src_raw(self.st, self.val, x_local, x_halo)

    # ------------------------------------------------------------------ the step
    def spmm(self, x_local):
        if self.mode == "p2p":
            shard = self.features(x_local.shape[1])
            if x_local.data_ptr() != shard.data_ptr():
                self.release()              # peers' previous kernels are done reading this shard
                shard.copy_(x_local)        # callers that keep X in features() skip barrier + copy
            return self.spmm_p2p()
        F = x_local.shape[1]
        halo = self.exchange_rows(self.pack(x_local), F)
        return self.local_spmm(x_local, halo)

    def last_kernel_seconds(self, step, torch_mod, iters=5):
        """Mean duration of the SpMM kernel alone (CUDA events, max over ranks), for the roofline."""
        if self.mode == "p2p":
            fn = self.spmm_p2p
        else:
            F = self.x_local.shape[1]
            halo = self.exchange_rows(self.pack(self.x_local), F)
            fn = lambda: self.local_spmm(self.x_local, halo)
        for _ in range(2):
            fn()
        a, b = torch_mod.cuda.Event(enable_timing=True), torch_mod.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            fn()
        b.record()
        torch_mod.cuda.synchronize()
        t = torch.tensor([a.elapsed_time(b) / iters / 1e3], device=self.device, dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX, group=self.group)
        return float(t)


def partition_global_csr(row_ptr, col, val, rank, world, device, group=None, mode=None):
    """Slice a (replicated, host or device) global CSR into this rank's LocalPartition."""
    bounds = balanced_row_ranges(row_ptr, world)
    lo, hi = bounds[rank], bounds[rank + 1]
    e0, e1 = int(row_ptr[lo]), int(row_ptr[hi])
    part = LocalPartition(rank, world, bounds, (row_ptr[lo:hi + 1] - e0).clone(), col[e0:e1].clone(),
                          None if val is None else val[e0:e1].clone())
    return PartitionedSpMM(part, device, group, global_nnz=int(row_ptr[-1]), mode=mode)


# papers100M-shaped graph, 1/8 of it per GPU (BASELINE configs[4]): fixed per-GPU work => weak scaling
PAPERS_ROWS_PER_GPU = synth.PAPERS_ROWS_PER_GPU
PAPERS_EDGES_PER_GPU = synth.PAPERS_EDGES_PER_GPU


def synthetic_partition(rank, world, device, seed=0, rows=PAPERS_ROWS_PER_GPU, edges=PAPERS_EDGES_PER_GPU,
                        beta=0.05, hidden=128, group=None, mode=None, scaling="weak"):
    """Generate this rank's shard directly on its GPU (synth.shard_csr: the locality-controlled
    generator of SURVEY 8d) and wrap it in a PartitionedSpMM with X resident in the feature shard."""
    row_ptr, col = synth.shard_csr(rank, world, rows, edges, beta, seed=seed, device=device)
    bounds = [k * rows for k in range(world + 1)]
    part = LocalPartition(rank, world, bounds, row_ptr, col, None)
    del col
    desc = synth.shard_description(rows, edges, world, beta, seed, hidden, scaling)
    ps = PartitionedSpMM(part, device, group, global_nnz=edges * world, description=desc, mode=mode)
    gen = torch.Generator(device=device).manual_seed(seed + rank)
    if ps.mode == "p2p":
        ps.x_local = ps.features(hidden)          # X lives in the symmetric shard: no copy per step
        ps.x_local.normal_(generator=gen)
    else:
        ps.x_local = torch.randn(rows, hidden, device=device, generator=gen)
    return ps


# =============================================================================================
# Push form: reduce of boundary partial sums (the exchange the north star names; SURVEY 8e row 3)
# =============================================================================================
class PushPartition:
    """What rank p holds in the push form (index arithmetic only; device agnostic).

    Rank p owns destination rows AND source columns [lo_p, hi_p) and keeps every edge (r, c) whose
    column it owns, i.e. the column slice A[:, lo_p:hi_p], as two CSR blocks:

      boundary  B  [n_brow x n_local]  one row per DISTINCT destination row owned by another rank
                                       (ascending global id => grouped by owner rank), columns local;
                                       P = B @ X_local are the boundary partial sums this rank sends
      combined  C  [n_local x (n_local + n_recv)]
                                       row i = its interior edges in CSR order (columns < n_local),
                                       then one unit-weight entry per received partial that belongs
                                       to row i, in (source rank, position) order (columns
                                       n_local + k) => Y_local = C @ [X_local ; R] completes the
                                       sums in a fixed order: deterministic, no atomics.

    `rows_global` must be non-decreasing inside every source rank's block (true for edges kept in
    CSR order); `cols_global` all lie inside [lo_p, hi_p)."""

    def __init__(self, rank, world, bounds, rows_global, cols_global, val, group=None, comm_device=None):
        self.rank, self.world, self.bounds = rank, world, list(bounds)
        lo, hi = bounds[rank], bounds[rank + 1]
        self.lo, self.hi, self.n_local = lo, hi, hi - lo
        rows_global, cols_global = rows_global.to(torch.int64), cols_global.to(torch.int64)
        dev = rows_global.device
        if cols_global.numel() and (int(cols_global.min()) < lo or int(cols_global.max()) >= hi):
            raise ValueError("push form: every edge kept by a rank must have its column inside the rank's own range")
        self.weighted = val is not None
        interior = (rows_global >= lo) & (rows_global < hi)
        # ---- boundary block B
        rb, cb = rows_global[~interior], cols_global[~interior] - lo
        if rb.numel() > 1 and not bool((rb[1:] >= rb[:-1]).all()):
            order = torch.sort(rb, stable=True).indices            # keeps the CSR order inside a destination row
            rb, cb = rb[order], cb[order]
            vb = None if val is None else val[~interior][order]
        else:
            vb = None if val is None else val[~interior]
        self.brow, counts = torch.unique_consecutive(rb, return_counts=True)     # ascending global row ids
        self.n_brow = int(self.brow.numel())
        self.b_rowptr = torch.zeros(self.n_brow + 1, dtype=torch.int64, device=dev)
        torch.cumsum(counts, 0, out=self.b_rowptr[1:])
        self.b_col, self.b_val = cb, vb
        bt = torch.tensor(self.bounds, device=dev, dtype=torch.int64)
        owner = torch.searchsorted(bt, self.brow, right=True) - 1
        self.send_counts = torch.bincount(owner, minlength=world).tolist()       # partial rows I send to each rank
        assert self.send_counts[rank] == 0
        dest_local = self.brow - bt[owner]                                       # row inside the owner's shard
        # ---- tell every owner which of its rows my partials belong to (once per structure)
        cdev = dev if comm_device is None else comm_device
        sc = torch.tensor(self.send_counts, dtype=torch.int64, device=cdev)
        rc = torch.empty(world, dtype=torch.int64, device=cdev)
        _all_to_all(rc, sc, [1] * world, [1] * world, group)
        self.recv_counts = [int(v) for v in rc.tolist()]                         # partial rows I receive from each rank
        self.n_recv = sum(self.recv_counts)
        recv_row = torch.empty(self.n_recv, dtype=torch.int64, device=cdev)
        _all_to_all(recv_row, dest_local.to(cdev).contiguous(), self.recv_counts, self.send_counts, group)
        self.recv_row = recv_row.to(dev)                                         # local row of received partial k
        if self.n_recv and (int(self.recv_row.min()) < 0 or int(self.recv_row.max()) >= self.n_local):
            raise RuntimeError("push form: a peer sent a partial sum for a row this rank does not own")
        # ---- combined block C: interior edges first, then the partial slots, row by row (stable sort)
        ri, ci = rows_global[interior] - lo, cols_global[interior] - lo
        n_int = int(ri.numel())
        rows_c = torch.cat([ri, self.recv_row])
        cols_c = torch.cat([ci, self.n_local + torch.arange(self.n_recv, device=dev, dtype=torch.int64)])
        order = torch.sort(rows_c, stable=True).indices
        self.c_col = cols_c[order]
        self.c_rowptr = torch.zeros(self.n_local + 1, dtype=torch.int64, device=dev)
        torch.cumsum(torch.bincount(rows_c, minlength=self.n_local), 0, out=self.c_rowptr[1:])
        if val is None:
            self.c_val = None                     # unweighted kernel: a partial enters as 1.0 * r == r exactly
        else:
            self.c_val = torch.cat([val[interior].to(torch.float32),
                                    torch.ones(self.n_recv, dtype=torch.float32, device=dev)])[order]
        self.nnz_interior, self.nnz_boundary = n_int, int(cb.numel())

    # -------------------------------------------------------------------- constructors
    @staticmethod
    def from_global_csr(row_ptr, col, val, rank, world, bounds=None, group=None, comm_device=None):
        """Column slice of a replicated global CSR (host or device tensors), edges kept in CSR order."""
        bounds = balanced_row_ranges(row_ptr, world) if bounds is None else bounds
        lo, hi = bounds[rank], bounds[rank + 1]
        col = col.to(torch.int64)
        mine = ((col >= lo) & (col < hi)).nonzero().view(-1)
        deg = (row_ptr[1:] - row_ptr[:-1]).to(torch.int64)
        rows = torch.repeat_interleave(torch.arange(deg.numel(), device=col.device, dtype=torch.int64), deg)
        return PushPartition(rank, world, bounds, rows[mine], col[mine], None if val is None else val[mine],
                             group=group, comm_device=comm_device)

    @staticmethod
    def from_row_shard(rank, world, bounds, row_ptr_local, col_global, val_local, group=None, comm_device=None):
        """From the ROW shard a rank already holds (rows [lo, hi), global column ids): every boundary edge
        (r, c, v) is shipped once, at setup, to the rank that owns column c (ragged all-to-all of int64
        pairs); received blocks arrive in source-rank order, each in its sender's CSR order."""
        lo, hi = bounds[rank], bounds[rank + 1]
        dev = col_global.device
        cdev = dev if comm_device is None else comm_device
        col_global = col_global.to(torch.int64)
        deg = (row_ptr_local[1:] - row_ptr_local[:-1]).to(torch.int64)
        rows = lo + torch.repeat_interleave(torch.arange(deg.numel(), device=dev, dtype=torch.int64), deg)
        bt = torch.tensor(list(bounds), device=dev, dtype=torch.int64)
        owner = torch.searchsorted(bt, col_global, right=True) - 1
        away = owner != rank
        order = torch.sort(owner[away], stable=True).indices                     # group by owner, CSR order inside
        send = torch.stack([rows[away][order], col_global[away][order]], 1).contiguous()
        sc_l = torch.bincount(owner[away], minlength=world).tolist()
        sc = torch.tensor(sc_l, dtype=torch.int64, device=cdev)
        rc = torch.empty(world, dtype=torch.int64, device=cdev)
        _all_to_all(rc, sc, [1] * world, [1] * world, group)
        rc_l = [int(v) for v in rc.tolist()]
        recv = torch.empty((sum(rc_l), 2), dtype=torch.int64, device=cdev)
        _all_to_all(recv.view(-1), send.to(cdev).view(-1), [2 * c for c in rc_l], [2 * c for c in sc_l], group)
        recv = recv.to(dev)
        rv = None
        if val_local is not None:
            rv = torch.empty(sum(rc_l), dtype=torch.float32, device=cdev)
            _all_to_all(rv, val_local.to(torch.float32)[away][order].to(cdev).contiguous(), rc_l, sc_l, group)
            rv = rv.to(dev)
        # interior edges (mine, CSR order) + received boundary edges (source-rank order = ascending rows)
        rows_all = torch.cat([rows[~away], recv[:, 0]])
        cols_all = torch.cat([col_global[~away], recv[:, 1]])
        val_all = None if val_local is None else torch.cat([val_local.to(torch.float32)[~away], rv])
        return PushPartition(rank, world, bounds, rows_all, cols_all, val_all, group=group, comm_device=comm_device)


class PushSpMM:
    """The step of the push form:  P = B @ X_local  ->  reduce-scatter of the boundary partial sums
    (ragged all-to-all over NCCL/NVLink)  ->  Y_local = C @ [X_local ; R]  (two-source SpMM; the unit-weight
    columns of C add the received partials to their rows in a fixed order).  Both products run on the
    row-stream SpMM kernel (cogdl_b200_spmm_csr_f32 / _2src); there is no other kernel and no atomic."""

    def __init__(self, part: PushPartition, device, group=None):
        self.part, self.device, self.group = part, device, group
        self.mode = "push"
        self.n_local = part.n_local
        self.exchange = ("push: boundary partial sums reduce-scattered by a ragged all_to_all_single, added in "
                         "(source rank, row) order inside the interior SpMM")
        if device.type == "cuda":
            self.st_b = CSRStructure.from_int64(part.b_rowptr.to(device), part.b_col.to(device), n_cols=part.n_local)
            self.st_c = CSRStructure.from_int64(part.c_rowptr.to(device), part.c_col.to(device),
                                                n_cols=part.n_local + part.n_recv)
            self.st_b.plan, self.st_c.plan
            self.val_b = None if part.b_val is None else part.b_val.to(device).float().contiguous()
            self.val_c = None if part.c_val is None else part.c_val.to(device).float().contiguous()

    def partials(self, x_local):
        """P [n_brow, F]: this rank's contribution to rows owned by other ranks, packed in send order."""
        from .operators._raw import spmm_raw

        return spmm_raw(self.st_b, self.val_b, x_local)

    def reduce_scatter(self, p_send, F):
        """Ragged all-to-all of the packed partial rows; returns R [n_recv, F] in (source rank, row) order."""
        part = self.part
        r = torch.empty((part.n_recv, F), dtype=p_send.dtype, device=p_send.device)
        _all_to_all(r.view(-1), p_send.contiguous().view(-1), [c * F for c in part.recv_counts],
                    [c * F for c in part.send_counts], self.group)
        return r

    def combine(self, x_local, r):
        from .operators._raw import spmm_2src_raw

        return spmm_2src_raw(self.st_c, self.val_c, x_local, r)

    def spmm(self, x_local):
        F = x_local.shape[1]
        return self.combine(x_local, self.reduce_scatter(self.partials(x_local), F))
