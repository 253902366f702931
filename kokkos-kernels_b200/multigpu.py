"""Row-block-partitioned SpMV across the GPUs of one box with the all-gather of y pipelined behind
the compute (BASELINE.json configs[4]; no reference counterpart -- the reference is single-process).

Each rank owns rows [r0, r1) of A (row_ptr rebased, global columns) and a full copy of x.  The local
rows are cut into `chunks` pieces; piece c is computed by the TMA-tiled SpMV kernel straight into this
rank's slot of the next-x buffer and, as soon as it is done, pushed to the same slot of every peer's
next-x buffer by copy-engine transfers over NVLink (peer buffers are mapped through symmetric memory),
while piece c+1 is being computed.  A device-side barrier closes the step.  Results are bit-identical
to the single-GPU SpMV (same kernel, same per-row order).

modes: "pipelined" (default), "fused" (P2P stores issued by the SpMV kernel itself,
b200sp_spmv_scatter_f64_i32), "multicast" (as fused, but ONE store per y value to the NVSwitch multicast
address of the symmetric buffer -- on sm_90 multimem.st is a plain st.global to a multicast mapping, the
switch replicates it into all 8 copies, so every GPU sends its 80 MB once instead of 7 times; falls back
to "fused" when the symmetric-memory handle has no multicast pointer; not yet measured on H100 machines),
"pipelined_mc" (pieces like "pipelined", but each finished piece is pushed ONCE to the multicast address by a
small SM kernel with 16-byte stores, b200sp_multicast_push, on one communication stream; falls back to
"pipelined" without a multicast pointer),
"multicast_fwd" (one launch like "multicast", but the values reach the multicast address tile by tile from the kernel's
PRODUCER warp -- finished tiles of y are read back from L2 and stored with 256 contiguous bytes per instruction,
b200sp_spmv_forward_f64_i32: whole 128-byte NVLink writes instead of one 8-byte packet per row, no separate push kernel, no
SM taken from the compute),
"pipelined_sm" (pieces pushed to the 7 peers' unicast mappings by a small SM kernel, every 16 bytes read once and stored
7 times, b200sp_peer_push_sm), "nccl" (SpMV then all_gather_into_tensor)."""
import ctypes as C

import numpy as np
import torch
import torch.distributed as dist

from . import _lib, partition, sparse as sp


MODES = ("pipelined", "pipelined_mc", "pipelined_sm", "multicast", "multicast_fwd", "fused", "nccl")


class RowBlockSpMV:
    """y-slice = A[r0:r1, :] @ x on every rank, all-gathered into the next x.

    Two next-x buffers are used alternately (step k writes buffer k % 2), so `x = op.step(x)` is safe: the kernel never
    reads the buffer it -- or a peer that is one step ahead -- is writing (the closing barrier of step k orders every
    rank's reads of step k before any write of step k + 1 into the other buffer, and its writes before the reads of
    step k + 1).  `shared` = another RowBlockSpMV of the same shard whose device copy of the matrix is reused."""

    def __init__(self, rp, ci, va, n_total, r0, r1, device, mode="pipelined", chunks=8, tune=(-1, -1, -1), shared=None,
                 push_ctas=32):
        assert mode in MODES, mode
        self.world, self.rank = dist.get_world_size(), dist.get_rank()
        self.n_total, self.r0, self.r1, self.dev, self.mode = n_total, r0, r1, device, mode
        self.push_ctas = push_ctas
        nrows = r1 - r0
        assert n_total % self.world == 0 and nrows == n_total // self.world, "equal row blocks expected"
        if shared is not None:
            self.ci_d, self.va_d = shared.ci_d, shared.va_d
        else:
            self.ci_d = torch.from_numpy(ci).to(device)
            self.va_d = torch.from_numpy(va).to(device)
        self.symm = [None, None]
        self.bufs = []
        self.peer_ptrs = [[], []]
        self.mc_ptr = [0, 0]
        if mode != "nccl":
            import torch.distributed._symmetric_memory as symm_mem

            for b in range(2):
                buf = symm_mem.empty(n_total, dtype=torch.float64, device=device)
                hdl = symm_mem.rendezvous(buf, dist.group.WORLD)
                self.bufs.append(buf)
                self.symm[b] = hdl
                self.peer_ptrs[b] = [int(p) for p in hdl.buffer_ptrs]
                self.mc_ptr[b] = int(getattr(hdl, "multicast_ptr", 0) or 0)
            if mode in ("multicast", "multicast_fwd", "pipelined_mc") and (self.mc_ptr[0] == 0 or self.mc_ptr[1] == 0):
                raise RuntimeError("no NVSwitch multicast mapping for the symmetric buffer on this box")
        else:
            self.bufs = [torch.empty(n_total, dtype=torch.float64, device=device) for _ in range(2)]
        self.parity = 0  # buffer the next step writes
        self.x_next = self.bufs[0]
        self.y = self.x_next[r0:r1]
        # chunk boundaries on rows whose first entry is 16-byte aligned in col_idx / vals (TMA path)
        if not mode.startswith("pipelined"):
            chunks = 1
        bounds = partition.piece_bounds(rp, chunks, row_offset=r0, even_rows=(mode in ("pipelined_mc", "pipelined_sm")))
        self.pieces = []
        for c0, c1 in zip(bounds[:-1], bounds[1:]):
            s0, s1 = int(rp[c0]), int(rp[c1])
            rpc = torch.from_numpy((rp[c0:c1 + 1].astype(np.int64) - s0).astype(np.int32)).to(device)
            A = sp.CrsMatrix(rpc, self.ci_d[s0:s1], self.va_d[s0:s1], n_total)
            h = sp.SPMVHandle(sp.SPMV_DEFAULT)
            h.tune(*tune)
            per_buf = []
            for b in range(2):
                yv = self.bufs[b][r0 + c0: r0 + c1]
                dsts = []
                if mode in ("multicast", "multicast_fwd", "pipelined_mc"):
                    dsts = [self.mc_ptr[b] + (r0 + c0) * 8]  # one store, replicated by the switch (incl. this rank's copy)
                elif mode != "nccl":
                    dsts = [self.peer_ptrs[b][q] + (r0 + c0) * 8 for q in range(self.world) if q != self.rank]
                arr = (C.c_void_p * max(len(dsts), 1))(*[C.c_void_p(d) for d in dsts])
                per_buf.append((yv, dsts, arr))
            self.pieces.append((A, h, per_buf, torch.cuda.Event()))
        # whole-shard view (host-vector end-to-end path, parity checks)
        if shared is not None:
            self.A_full, self.h_full = shared.A_full, shared.h_full
        else:
            self.A_full = sp.CrsMatrix(torch.from_numpy(np.ascontiguousarray(rp)).to(device), self.ci_d, self.va_d, n_total)
            self.h_full = sp.SPMVHandle(sp.SPMV_DEFAULT)
        # communication streams (high priority: a push that becomes runnable is placed before the next piece's CTAs):
        # one per peer for the copy-engine pushes, the first one for the SM push kernels
        self.comm = [torch.cuda.Stream(device=device, priority=-1) for _ in range(max(self.world - 1, 1))]
        self.comm_arr = (C.c_void_p * len(self.comm))(*[C.c_void_p(s.cuda_stream) for s in self.comm])

    def kernel_name(self):
        return self.pieces[0][1].last_kernel()

    def nnz(self):
        return self.ci_d.numel()

    def step(self, x):
        """next x <- all-gather(A_local @ x); returns the buffer written (valid on every rank once the call's stream work
        has completed); self.y is this rank's slice of it."""
        lib = _lib.sparse()
        cur = torch.cuda.current_stream()
        b = self.parity
        out = self.bufs[b]
        assert x.data_ptr() != out.data_ptr(), "RowBlockSpMV.step: x is the buffer this step writes"
        if self.mode == "multicast_fwd":
            A, h, per_buf, ev = self.pieces[0]
            yv, dsts, arr = per_buf[b]
            sp.spmv_forward(h, 1.0, A, x, yv, dsts[0])
            self.symm[b].barrier(channel=0)
        elif self.mode in ("fused", "multicast"):
            A, h, per_buf, ev = self.pieces[0]
            yv, dsts, arr = per_buf[b]
            sp.spmv_scatter(h, 1.0, A, x, yv, dsts)
            self.symm[b].barrier(channel=0)
        elif self.mode in ("pipelined_mc", "pipelined_sm"):
            cs = C.c_void_p(cur.cuda_stream)
            comm = self.comm[0]
            for A, h, per_buf, ev in self.pieces:
                yv, dsts, arr = per_buf[b]
                sp.spmv(h, "N", 1.0, A, x, 0.0, yv)
                ev.record(cur)
                comm.wait_event(ev)
                if self.mode == "pipelined_mc":
                    _lib.check(lib.b200sp_multicast_push(C.c_void_p(comm.cuda_stream), C.c_void_p(yv.data_ptr()),
                                                         C.c_void_p(dsts[0]), yv.numel() * 8, self.push_ctas))
                else:
                    _lib.check(lib.b200sp_peer_push_sm(C.c_void_p(comm.cuda_stream), C.c_void_p(yv.data_ptr()), yv.numel() * 8,
                                                       len(dsts), arr, self.push_ctas))
            _lib.check(lib.b200sp_peer_join(cs, self.comm_arr, 1))
            self.symm[b].barrier(channel=0)
        elif self.mode == "pipelined":
            cs = C.c_void_p(cur.cuda_stream)
            for A, h, per_buf, ev in self.pieces:
                yv, dsts, arr = per_buf[b]
                sp.spmv(h, "N", 1.0, A, x, 0.0, yv)
                _lib.check(lib.b200sp_peer_push_async(cs, self.comm_arr, len(dsts), arr, C.c_void_p(yv.data_ptr()),
                                                      yv.numel() * 8))
            _lib.check(lib.b200sp_peer_join(cs, self.comm_arr, len(self.comm) if self.world > 1 else 0))
            self.symm[b].barrier(channel=0)
        else:
            A, h, per_buf, ev = self.pieces[0]
            yv, dsts, arr = per_buf[b]
            sp.spmv(h, "N", 1.0, A, x, 0.0, yv)
            dist.all_gather_into_tensor(out, yv)
        self.x_next = out
        self.y = out[self.r0:self.r1]
        self.parity ^= 1
        return out

    def allgather_slices(self, buf_index=None):
        """All-gather of the ranks' own slices of a next-x buffer WITHOUT compute (the slice of every rank is already in
        its own copy): what the end-to-end leg uses after uploading only this rank's part of x.  Same transport as step()."""
        lib = _lib.sparse()
        cur = torch.cuda.current_stream()
        b = self.parity if buf_index is None else buf_index
        out = self.bufs[b]
        mine = out[self.r0:self.r1]
        if self.mode == "nccl":
            dist.all_gather_into_tensor(out, mine)
            return out
        cs = C.c_void_p(cur.cuda_stream)
        if self.mode in ("multicast", "multicast_fwd", "pipelined_mc"):
            _lib.check(lib.b200sp_multicast_push(cs, C.c_void_p(mine.data_ptr()), C.c_void_p(self.mc_ptr[b] + self.r0 * 8),
                                                 mine.numel() * 8, 4 * self.push_ctas))
        elif self.mode == "pipelined":
            dsts = [self.peer_ptrs[b][q] + self.r0 * 8 for q in range(self.world) if q != self.rank]
            arr = (C.c_void_p * max(len(dsts), 1))(*[C.c_void_p(d) for d in dsts])
            _lib.check(lib.b200sp_peer_push_async(cs, self.comm_arr, len(dsts), arr, C.c_void_p(mine.data_ptr()), mine.numel() * 8))
            _lib.check(lib.b200sp_peer_join(cs, self.comm_arr, len(self.comm) if self.world > 1 else 0))
        else:
            dsts = [self.peer_ptrs[b][q] + self.r0 * 8 for q in range(self.world) if q != self.rank]
            arr = (C.c_void_p * max(len(dsts), 1))(*[C.c_void_p(d) for d in dsts])
            _lib.check(lib.b200sp_peer_push_sm(cs, C.c_void_p(mine.data_ptr()), mine.numel() * 8, len(dsts), arr, 4 * self.push_ctas))
        self.symm[b].barrier(channel=0)
        return out

    # ---- end-to-end form: host vectors in, host vectors out -------------------------------------------------------------
    def step_host(self, x_host_slice, y_host_slice):
        """One SpMV of the row-partitioned matrix with HOST vectors: this rank uploads only ITS slice of x (rows r0:r1, pinned
        host memory) into its slot of a next-x buffer, the all-gather over NVLink completes x on every GPU, the local rows are
        multiplied and this rank's slice of y is downloaded.  Calls are pipelined over the two buffers: upload k + 1 runs
        while call k computes and call k - 1 downloads; y_host_slice is valid after host_flush() and a synchronisation of
        the current stream."""
        if not hasattr(self, "_hs"):
            dev = self.dev
            self._hs = {
                "sH": torch.cuda.Stream(device=dev), "sD": torch.cuda.Stream(device=dev), "k": 0,
                "up": [torch.cuda.Event() for _ in range(2)], "sp": [torch.cuda.Event() for _ in range(2)],
                "dn": [torch.cuda.Event() for _ in range(2)],
                "y": [torch.empty(self.r1 - self.r0, dtype=torch.float64, device=dev) for _ in range(2)],
            }
        hs = self._hs
        k, b = hs["k"], hs["k"] % 2
        cur = torch.cuda.current_stream()
        buf = self.bufs[b]
        if k >= 2:
            hs["sH"].wait_event(hs["sp"][b])  # call k - 2 read this buffer
        else:
            hs["sH"].wait_stream(cur)
        with torch.cuda.stream(hs["sH"]):
            buf[self.r0:self.r1].copy_(x_host_slice, non_blocking=True)
            hs["up"][b].record(hs["sH"])
        cur.wait_event(hs["up"][b])
        self.allgather_slices(b)
        if k >= 2:
            cur.wait_event(hs["dn"][b])  # the download of call k - 2 has left y[b]
        sp.spmv(self.h_full, "N", 1.0, self.A_full, buf, 0.0, hs["y"][b])
        hs["sp"][b].record(cur)
        hs["sD"].wait_event(hs["sp"][b])
        with torch.cuda.stream(hs["sD"]):
            y_host_slice.copy_(hs["y"][b], non_blocking=True)
            hs["dn"][b].record(hs["sD"])
        hs["k"] = k + 1

    def host_flush(self):
        """Make the current stream wait for every outstanding download of step_host."""
        if hasattr(self, "_hs"):
            cur = torch.cuda.current_stream()
            for b in range(min(2, self._hs["k"])):
                cur.wait_event(self._hs["dn"][b])

    def local_spmv_only(self, x):
        b = self.parity
        for A, h, per_buf, ev in self.pieces:
            sp.spmv(h, "N", 1.0, A, x, 0.0, per_buf[b][0])


class RowBlockSpGEMM:
    """C = A * B with the rows of A (hence of C) sharded over the ranks and B replicated (SURVEY.md section 8e: "SpGEMM also
    shards by row blocks of A with B replicated; rowptr needs one exchange of P counts").  Every rank runs the single-GPU
    spgemm_symbolic / spgemm_numeric of the library on its row block -- the rows of C are independent, so the block is
    bit-identical to the same rows of the single-GPU product -- and ONE all_gather of the P block sizes gives each rank the
    offset of its block in the global C (no collective on the data path).  No reference counterpart (single-process library).

        op = RowBlockSpGEMM(A_local, B, group=None)   # A_local: rows [r0, r1) of A, row map rebased, global columns
        C_local = op.symbolic()                       # structure of this rank's rows; op.block_nnz / op.offset are known
        op.numeric()                                  # values; re-runnable with new values on the same structure
        op.global_row_map()                           # int64: C_local.row_map + op.offset (global nnz may exceed int32)
    """

    def __init__(self, A_local, B, group=None):
        if A_local.numCols() != B.numRows():
            raise sp.B200SparseError(f"RowBlockSpGEMM: inner dimensions differ: {A_local.numCols()} vs {B.numRows()}")
        self.A, self.B, self.group = A_local, B, group
        self.kh = sp.KokkosKernelsHandle()
        self.kh.create_spgemm_handle(sp.SPGEMM_KK)
        self.C = None
        self.block_nnz = None  # nnz of every rank's block of C
        self.offset = None     # where this rank's block starts in the global entries / values of C

    def symbolic(self):
        self.C = sp.spgemm_symbolic(self.kh, self.A, False, self.B, False)
        mine = int(self.kh.get_spgemm_handle().get_c_nnz())
        if dist.is_available() and dist.is_initialized():
            world = dist.get_world_size(self.group)
            counts = [None] * world
            dist.all_gather_object(counts, mine, group=self.group)
            rank = dist.get_rank(self.group)
        else:
            counts, rank = [mine], 0
        self.block_nnz = [int(c) for c in counts]
        self.offset = int(sum(self.block_nnz[:rank]))
        return self.C

    def numeric(self, A_values=None, B_values=None):
        if self.C is None:
            raise sp.B200SparseInvalidArgument("RowBlockSpGEMM.numeric: call symbolic first")
        A = self.A if A_values is None else sp.CrsMatrix(self.A.row_map, self.A.entries, A_values, self.A.numCols())
        B = self.B if B_values is None else sp.CrsMatrix(self.B.row_map, self.B.entries, B_values, self.B.numCols())
        sp.spgemm_numeric(self.kh, A, False, B, False, self.C)
        return self.C

    def global_row_map(self):
        return self.C.row_map.to(torch.int64) + self.offset
