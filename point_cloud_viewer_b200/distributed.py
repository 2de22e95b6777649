"""Multi-GPU build_octree: points shard by octree path prefix and move once to their owners (SURVEY.md 8e).

Every rank holds a contiguous slice of the global point index space.  The split phase of the reference is independent
below any octree prefix and the subsample phase only couples a parent with its 8 children, so:

  1. all-reduce the 8^k histogram of level-k prefix cells (first k steps of the re-quantising descent on the raw
     positions - the cell the single-GPU build would route the point to);
  2. greedily balance the non-empty cells over the ranks (largest first);
  3. ONE exchange; every receiver holds the source ranks' blocks in rank order, which is global index order, i.e. the
     reference's stable stream order.  On GPUs every rank first runs the ingest step of the build on its own points
     (level-1 codes + the digits of levels 1..2, whose histogram IS the cell histogram of step 1) and one kernel then
     ranks the records by destination and stores them straight into the owners' memory over NVLink (CUDA-IPC peer mapping,
     `CudaOps.ingest` / `exchange_records`): 21 bytes per point cross the link, and the owner's build starts at its first
     partition pass - no arithmetic is repeated.  The staged variant (raw points packed into send buffers +
     all_to_all_single) serves the CPU tests;
  4. every rank builds the sub-trees of its cells independently (global bounding cube; the nodes above level k take
     their split decision from the global counts);
  5. the <= 1 + 8 + 64 nodes above level k are assembled on rank 0 from the children's every-8th points (collected,
     already encoded in the parent's cube, by the level k-1 "collector" nodes of every rank).

The compute steps are CUDA kernels behind the C ABI (`CudaOps`); the collectives are torch.distributed (NCCL on GPUs).
The orchestration below is backend-neutral so that tests can run it on 2 CPU processes over gloo with the test-only
sequential stand-ins for the kernels.
"""
import sys

import numpy as np

from . import ENC_BYTES


# ---- pure planning helpers ----------------------------------------------------------------------------------------
def level_counts(counts_k, k):
    """Counts of the cells of levels 1..k from the level-k histogram."""
    c = np.asarray(counts_k, np.uint64)
    return [c.reshape(8 ** j, -1).sum(1).astype(np.uint64) for j in range(1, k + 1)]


def concat_counts(levels):
    return np.concatenate(levels).astype(np.uint64)


def usable_prefix_levels(counts_k, k, root_edge, resolution, max_points):
    """Largest k' <= k such that every non-empty node of levels 1..k'-1 is split by the reference's rule
    (count > MAX_POINTS_PER_NODE and edge > resolution, generation.rs:128-150), i.e. no leaf sits above the shard level."""
    levels = level_counts(counts_k, k)
    ok = 1
    edge = root_edge
    for j in range(1, k):
        edge = edge / 2.0
        c = levels[j - 1]
        nz = c[c > 0]
        if len(nz) and (nz > max_points).all() and edge > resolution:
            ok = j + 1
        else:
            break
    return ok


def assign_cells(counts, nranks):
    """Longest-processing-time greedy: cells by decreasing count (ties: lower cell first) to the least loaded rank
    (ties: lower rank).  Deterministic, identical on every rank.  Empty cells -> rank 0."""
    counts = np.asarray(counts, np.uint64)
    order = sorted(range(len(counts)), key=lambda c: (-int(counts[c]), c))
    load = [0] * nranks
    out = np.zeros(len(counts), np.int32)
    for c in order:
        if counts[c] == 0:
            continue
        r = min(range(nranks), key=lambda i: (load[i], i))
        out[c] = r
        load[r] += int(counts[c])
    return out


# ---- communication over torch.distributed ---------------------------------------------------------------------------
class TorchComm:
    def __init__(self, device):
        import torch.distributed as dist

        self.dist = dist
        self.rank = dist.get_rank()
        self.world = dist.get_world_size()
        self.device = device

    def all_reduce_sum_u64(self, arr):
        import torch

        t = torch.from_numpy(np.asarray(arr, np.uint64).astype(np.int64)).to(self.device)
        self.dist.all_reduce(t, op=self.dist.ReduceOp.SUM)
        return t.cpu().numpy().astype(np.uint64)

    def all_reduce_minmax(self, mn, mx):
        import torch

        a = torch.tensor(list(mn), dtype=torch.float64, device=self.device)
        b = torch.tensor(list(mx), dtype=torch.float64, device=self.device)
        self.dist.all_reduce(a, op=self.dist.ReduceOp.MIN)
        self.dist.all_reduce(b, op=self.dist.ReduceOp.MAX)
        return a.cpu().numpy(), b.cpu().numpy()

    def exchange_counts(self, send_counts):
        import torch

        s = torch.from_numpy(np.asarray(send_counts, np.int64)).to(self.device)
        r = torch.empty_like(s)
        self.dist.all_to_all_single(r, s)
        return r.cpu().numpy()

    def all_to_all(self, tensor, send_counts, recv_counts, alloc=None):
        import torch

        n = int(np.sum(recv_counts))
        out = alloc(tensor, n) if alloc is not None else torch.empty((n,) + tuple(tensor.shape[1:]), dtype=tensor.dtype, device=tensor.device)
        self.dist.all_to_all_single(out, tensor.contiguous(), output_split_sizes=[int(v) for v in recv_counts], input_split_sizes=[int(v) for v in send_counts])
        return out

    def all_gather_objects(self, obj):
        lst = [None] * self.world
        self.dist.all_gather_object(lst, obj)
        return lst

    def all_gather_counts(self, counts):
        """(world, len(counts)) int64 matrix: row s = the counts of rank s."""
        import torch

        s = torch.from_numpy(np.asarray(counts, np.int64)).to(self.device)
        out = torch.empty(self.world * s.numel(), dtype=torch.int64, device=self.device)  # flat: gloo takes no (world, n) output
        self.dist.all_gather_into_tensor(out, s)
        return out.cpu().numpy().reshape(self.world, -1)

    def all_gather_bytes(self, buf, nbytes_max):
        """(world, nbytes_max) uint8 matrix: row r = rank r's byte buffer, zero padded (one tensor collective, no pickling)."""
        import torch

        t = torch.zeros(nbytes_max, dtype=torch.uint8, device=self.device)
        if len(buf):
            t[: len(buf)] = torch.from_numpy(np.ascontiguousarray(buf, np.uint8)).to(self.device)
        out = torch.empty(self.world * nbytes_max, dtype=torch.uint8, device=self.device)
        self.dist.all_gather_into_tensor(out, t)
        return out.cpu().numpy().reshape(self.world, nbytes_max)

    def barrier(self):
        if self.device.type == "cuda":
            import torch

            torch.cuda.synchronize()
        self.dist.barrier()

    def done_with(self, *tensors):
        """The exchange that read these send buffers has completed: pool-backed buffers go back to the library's pool."""
        if self.device.type == "cuda":
            import torch

            torch.cuda.synchronize()
        for t in tensors:
            owner = getattr(t, "_pcv_owner", None) if t is not None else None
            if owner is not None:
                owner.free()


# ---- CUDA implementation of the compute steps ---------------------------------------------------------------------
class CudaOps:
    """x, y, z: torch cuda float64 tensors (SoA); rgb: uint8 (n*3); intensity: float32 or None."""

    def __init__(self, ctx, x, y, z, rgb, intensity, resolution, bmin, bmax, consume_input=False):
        self.consume_input = consume_input  # release pool-backed input tensors as soon as they have been packed
        self.ctx, self.x, self.y, self.z, self.rgb, self.intensity = ctx, x, y, z, rgb, intensity
        self.res, self.bmin, self.bmax = resolution, bmin, bmax
        self.n = x.numel()
        self.device = x.device

    def local_bbox(self):
        return self.ctx.bbox(self.x.data_ptr(), self.y.data_ptr(), self.z.data_ptr(), n=self.n, device=True)

    def prefix_histogram(self, k):
        return self.ctx.prefix_histogram_device(self.x.data_ptr(), self.y.data_ptr(), self.z.data_ptr(), self.n, self.res, self.bmin, self.bmax, k)

    def prefix_histogram_bbox(self, k):
        """(histogram, data min, data max): the bounding box rides on the histogram's read of the positions."""
        return self.ctx.prefix_histogram_bbox_device(self.x.data_ptr(), self.y.data_ptr(), self.z.data_ptr(), self.n, self.res, self.bmin, self.bmax, k)

    def pack(self, k, cell_to_rank, nranks, index_base):
        import torch

        n = self.n
        # staging buffers come from torch's caching allocator: identical sizes every step, so they are reused without any
        # driver call (pool-backed buffers were measured to fragment the stream-ordered pool: 2-5x slower steps)
        xyz = torch.empty((n, 3), dtype=torch.float64, device=self.device)
        rgb = torch.empty((n, 3), dtype=torch.uint8, device=self.device)
        inten = torch.empty(n, dtype=torch.float32, device=self.device) if self.intensity is not None else None
        idx = torch.empty(n, dtype=torch.int64, device=self.device)
        counts = self.ctx.prefix_pack_device(self.x.data_ptr(), self.y.data_ptr(), self.z.data_ptr(), self.rgb.data_ptr(),
                                             self.intensity.data_ptr() if self.intensity is not None else None, None, index_base, n, self.res, self.bmin,
                                             self.bmax, k, cell_to_rank, nranks, xyz.data_ptr(), rgb.data_ptr(), inten.data_ptr() if inten is not None else None,
                                             idx.data_ptr())
        if self.consume_input:
            for t in (self.x, self.y, self.z, self.rgb, self.intensity):
                owner = getattr(t, "_pcv_owner", None) if t is not None else None
                if owner is not None:
                    owner.free()
            self.x = self.y = self.z = self.rgb = self.intensity = None
        return xyz, rgb, inten, idx, counts.astype(np.int64)

    # ---- fused pack + exchange over peer memory (NVLink / NVSwitch), see kernels_shard.cuh::k_pack_exchange ----
    def pack_exchange(self, k, cell_to_rank, nranks, index_base, comm, send_counts):
        """Returns a PeerReceive: this rank's received points (SoA device arrays inside its exportable slab)."""
        import torch

        M = comm.all_gather_counts(send_counts)  # M[s][d]: points rank s sends to rank d; identical on every rank
        need = M.sum(0)  # per destination
        slab = PeerSlab.get(self.ctx, comm, int(need.max()), self.intensity is not None)
        rank = comm.rank
        first = [int(M[:rank, d].sum()) for d in range(nranks)]
        A = [slab.arrays(d) for d in range(nranks)]
        counts = self.ctx.prefix_pack_exchange_device(self.x.data_ptr(), self.y.data_ptr(), self.z.data_ptr(), self.rgb.data_ptr(),
                                                      self.intensity.data_ptr() if self.intensity is not None else None, index_base, self.n, self.res,
                                                      self.bmin, self.bmax, k, cell_to_rank, nranks, first, [a["x"] for a in A], [a["y"] for a in A],
                                                      [a["z"] for a in A], [a["idx"] for a in A],
                                                      [a["intensity"] for a in A] if self.intensity is not None else None, [a["col"] for a in A])
        assert [int(c) for c in counts] == [int(v) for v in M[rank]], "local histogram and pack disagree"
        if self.consume_input:
            for t in (self.x, self.y, self.z, self.rgb, self.intensity):
                owner = getattr(t, "_pcv_owner", None) if t is not None else None
                if owner is not None:
                    owner.free()
            self.x = self.y = self.z = self.rgb = self.intensity = None
        comm.barrier()  # every rank's stores have landed (each kernel completed before its rank entered the barrier)
        n = int(need[rank])
        mine = slab.arrays(rank)
        rgb = torch.empty(max(3 * n, 1), dtype=torch.uint8, device=self.device)
        self.ctx.unpack_colours_device(mine["col"], n, rgb.data_ptr())
        idx = torch.as_tensor(_RawCuda(mine["idx"], (max(n, 1),), "<i8"), device=self.device)[:n].clone()  # the slab is reused by the next step
        return PeerReceive(n, mine["x"], mine["y"], mine["z"], rgb, mine["intensity"] if self.intensity is not None else None, idx)

    # ---- round 2: exchange of ingested records (pcv.h pcv_shard_*) ----
    def ingest(self, k):
        """Ingest step + digit histogram of the local points -> level-k cell counts (the send handle stays with the ops)."""
        counts, self.send = self.ctx.shard_ingest(self.x.data_ptr(), self.y.data_ptr(), self.z.data_ptr(), self.rgb.data_ptr(),
                                                  self.intensity.data_ptr() if self.intensity is not None else None, self.n, self.res, self.bmin, self.bmax, k)
        self.wide, self.digit_levels = self.ctx.shard_send_info(self.send)
        return counts

    def exchange_records(self, k, cell_to_rank, nranks, comm, send_counts):
        """One kernel: every local record into its owner's slab.  Returns (RecordSlab, n received, count matrix)."""
        M = comm.all_gather_counts(send_counts)  # M[s][d]: points rank s sends to rank d; identical on every rank
        need = M.sum(0)
        slab = RecordSlab.get(self.ctx, comm, int(need.max()), self.wide, self.intensity is not None)
        rank = comm.rank
        first = [int(M[:rank, d].sum()) for d in range(nranks)]
        A = [slab.arrays(d) for d in range(nranks)]
        comm.barrier()  # no peer is still using its slab as build scratch
        counts = self.ctx.shard_exchange(self.send, k, cell_to_rank, nranks, first, [a["rec"] for a in A], [a["col"] for a in A] if self.wide else None, [a["dig"] for a in A],
                                         [a["intensity"] for a in A] if self.intensity is not None else None)
        assert [int(c) for c in counts] == [int(v) for v in M[rank]], "local histogram and exchange disagree"
        comm.barrier()  # every rank's stores have landed (each kernel completed before its rank entered the barrier)
        return slab, int(need[rank]), M

    def build_from_records(self, slab, n, k, prefix_counts):
        a = slab.arrays(slab.rank)
        return self.ctx.build_octree_from_records(a["rec"] if n else 0, (a["col"] if n else 0) if slab.wide else None, a["dig"] if n else 0,
                                                  a["intensity"] if (self.intensity is not None and n) else None, n, self.res, self.bmin, self.bmax, k, prefix_counts)

    def build_sharded_soa(self, recv, k, prefix_counts):
        n = recv.n
        return self.ctx.build_octree_sharded_device_soa(recv.x if n else 0, recv.y if n else 0, recv.z if n else 0, recv.rgb.data_ptr() if n else 0,
                                                        recv.intensity if (recv.intensity and n) else None, n, self.res, self.bmin, self.bmax, k, prefix_counts)

    def build_sharded(self, xyz, rgb, inten, k, prefix_counts):
        n = xyz.shape[0]
        return self.ctx.build_octree_sharded_device(xyz.data_ptr() if n else 0, rgb.data_ptr() if n else 0, inten.data_ptr() if (inten is not None and n) else None, n,
                                                    self.res, self.bmin, self.bmax, k, prefix_counts)

    def assemble_top(self, k, prefix_counts, unit_nsub, xyz_codes, rgb, inten):
        return self.ctx.assemble_top(self.res, self.bmin, self.bmax, k, prefix_counts, unit_nsub, xyz_codes, rgb, inten)



class _RawCuda:
    """A device pointer as __cuda_array_interface__ (zero-copy torch view of slab memory)."""

    def __init__(self, ptr, shape, typestr):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": typestr, "data": (int(ptr), False), "version": 2, "strides": None}


class PeerReceive:
    def __init__(self, n, x, y, z, rgb, intensity, idx):
        self.n, self.x, self.y, self.z, self.rgb, self.intensity, self.idx = n, x, y, z, rgb, intensity, idx


class PeerSlab:
    """Per-rank receive slab in exportable device memory, mapped into every peer process through CUDA IPC.  All ranks use
    the same capacity (so that the sub-array offsets of a peer's slab are known): x | y | z | index (8 B each) | intensity |
    packed colour (4 B each).  Re-created collectively, and rarely, when a step needs more room (decided from the
    all-gathered count matrix, i.e. identically on every rank, without an extra collective)."""

    _cache = {}

    @classmethod
    def get(cls, ctx, comm, need_points, with_intensity):
        cur = cls._cache.get(id(ctx))
        if cur is not None and cur.cap >= need_points and cur.world == comm.world:
            return cur
        if cur is not None:
            cur.close(comm)
        cap = ((int(need_points * 1.05) + 4096 + 4095) // 4096) * 4096
        cls._cache[id(ctx)] = slab = cls(ctx, comm, cap)
        return slab

    def __init__(self, ctx, comm, cap):
        self.ctx, self.cap, self.world, self.rank = ctx, cap, comm.world, comm.rank
        self.ptr, handle = ctx.ipc_alloc(40 * cap)
        handles = comm.all_gather_objects(handle)
        self.peer = [self.ptr if r == self.rank else ctx.ipc_open(handles[r]) for r in range(self.world)]
        comm.barrier()

    def arrays(self, r):
        b, c = self.peer[r], self.cap
        return {"x": b, "y": b + 8 * c, "z": b + 16 * c, "idx": b + 24 * c, "intensity": b + 32 * c, "col": b + 36 * c}

    def close(self, comm):
        comm.barrier()  # nobody is still writing into a slab that is about to disappear
        for r, p in enumerate(self.peer):
            if r != self.rank:
                self.ctx.ipc_close(p)
        comm.barrier()
        self.ctx.ipc_free(self.ptr)
        PeerSlab._cache.pop(id(self.ctx), None)


class RecordSlab:
    """Per-rank receive slab for ingested records, in exportable device memory mapped into every peer process through CUDA IPC.
    All ranks use the same capacity (so that the sub-array offsets of a peer's slab are known): records (16 or 32 B) | packed
    colour (4 B) | intensity (4 B, optional) | digits (1 B), each section with 256 bytes of slack (bulk copies read whole
    16-byte granules).  Re-created collectively, and rarely, when a step needs more room."""

    _cache = {}

    @classmethod
    def get(cls, ctx, comm, need_points, wide, with_intensity):
        cur = cls._cache.get(id(ctx))
        if cur is not None and cur.cap >= need_points and cur.world == comm.world and cur.wide == wide and cur.with_intensity == with_intensity:
            return cur
        if cur is not None:
            cur.close(comm)
        cap = ((int(need_points * 1.05) + 4096 + 4095) // 4096) * 4096
        cls._cache[id(ctx)] = slab = cls(ctx, comm, cap, wide, with_intensity)
        return slab

    def __init__(self, ctx, comm, cap, wide, with_intensity):
        self.ctx, self.cap, self.world, self.rank, self.wide, self.with_intensity = ctx, cap, comm.world, comm.rank, wide, with_intensity
        rs = 32 if wide else 16
        # build scratch: the owner's partition passes ping-pong through the slab, so the colour section exists either way
        self.off_col = rs * cap + 256
        self.off_int = self.off_col + 4 * cap + 256
        self.off_dig = self.off_int + (4 * cap + 256 if with_intensity else 0)
        self.bytes = self.off_dig + cap + 256
        self.ptr, handle = ctx.ipc_alloc(self.bytes)
        handles = comm.all_gather_objects(handle)
        self.peer = [self.ptr if r == self.rank else ctx.ipc_open(handles[r]) for r in range(self.world)]
        comm.barrier()

    def arrays(self, r):
        b = self.peer[r]
        return {"rec": b, "col": b + self.off_col, "intensity": b + self.off_int, "dig": b + self.off_dig}

    def close(self, comm):
        comm.barrier()  # nobody is still writing into a slab that is about to disappear
        for r, p in enumerate(self.peer):
            if r != self.rank:
                self.ctx.ipc_close(p)
        comm.barrier()
        self.ctx.ipc_free(self.ptr)
        RecordSlab._cache.pop(id(self.ctx), None)


class LazyIndex:
    """Global source index of every received record, materialised on first use (a collective over `comm`): the exchange is stable,
    so the block a source rank wrote into this rank's slab holds, in order, exactly those of its points whose destination is
    this rank - each source lists their global indices from its per-point destination array and one all-to-all delivers them."""

    def __init__(self, ctx, send, index_base, n_local, M, comm, n_recv=None):
        self.ctx, self.send, self.base, self.n_local, self.M, self.comm = ctx, send, int(index_base), int(n_local), M, comm
        self.n_recv = n_recv
        self.value = None

    def resolve(self):
        if self.value is not None:
            return self.value
        import torch

        dev, comm = self.comm.device, self.comm
        ptr, n = self.ctx.shard_send_dest(self.send)
        dest = torch.as_tensor(_RawCuda(ptr, (max(n, 1),), "|u1"), device=dev)[:n] if n else torch.zeros(0, dtype=torch.uint8, device=dev)
        parts = [torch.nonzero(dest == d).flatten() + self.base for d in range(comm.world)]
        if self.M is None:  # count matrix from the per-point destinations (collective)
            self.M = np.asarray(comm.all_gather_counts(np.array([int(p.numel()) for p in parts], np.int64))).reshape(comm.world, comm.world)
        send = torch.cat(parts) if parts else torch.zeros(0, dtype=torch.int64, device=dev)
        sc, rc = [int(v) for v in self.M[comm.rank]], [int(v) for v in self.M[:, comm.rank]]
        assert [int(p.numel()) for p in parts] == sc, "destination array and count matrix disagree"
        self.value = comm.all_to_all(send, sc, rc)
        return self.value

    def numel(self):
        return int(self.n_recv) if self.M is None else int(self.M[:, self.comm.rank].sum())


class LazyCellIndex(LazyIndex):
    """Provenance after a fused exchange pass: a slot on an owner is (cell-major over the owner's cells, sender rank, local order),
    so each sender derives the slot of every local point from its level-2 cell (one byte per point, kept by the send handle) and
    the gathered per-sender histograms; one all-to-all delivers (slot, global index) pairs and the owner scatters them."""

    def __init__(self, ctx, send, index_base, n_local, cell_to_rank, n_slots, comm):
        self.ctx, self.send, self.base, self.n_local, self.c2r, self.n_slots, self.comm = ctx, send, int(index_base), int(n_local), cell_to_rank, int(n_slots), comm
        self.value = None

    def resolve(self):
        if self.value is not None:
            return self.value
        import torch

        dev, comm = self.comm.device, self.comm
        ptr, n = self.ctx.shard_send_cells(self.send)
        cells = (torch.as_tensor(_RawCuda(ptr, (max(n, 1),), "|u1"), device=dev)[:n] if n else torch.zeros(0, dtype=torch.uint8, device=dev)).to(torch.int64)
        mine = torch.bincount(cells, minlength=64)
        H = np.asarray(comm.all_gather_counts(mine.cpu().numpy()), np.int64).reshape(comm.world, 64)
        T, c2r = H.sum(0), np.asarray(self.c2r, np.int64)
        slot_start = np.zeros(64, np.int64)
        for r in range(comm.world):
            run = 0
            for c in range(64):
                if c2r[c] == r and T[c]:
                    slot_start[c] = run
                    run += int(T[c])
        pre = H[: comm.rank].sum(0)
        order = torch.argsort(cells, stable=True)
        sc = cells[order]
        first = torch.cumsum(mine, 0) - mine
        base = torch.from_numpy(slot_start + pre).to(dev)
        slot = base[sc] + (torch.arange(n, device=dev) - first[sc])
        owner = torch.from_numpy(c2r).to(dev)[sc]
        o2 = torch.argsort(owner, stable=True)
        send_counts = torch.bincount(owner, minlength=comm.world).cpu().numpy().astype(np.int64)
        recv_counts = np.asarray(comm.all_gather_counts(send_counts), np.int64).reshape(comm.world, comm.world)[:, comm.rank]
        sc_l, rc_l = [int(v) for v in send_counts], [int(v) for v in recv_counts]
        got_slot = comm.all_to_all(slot[o2].contiguous(), sc_l, rc_l)
        got_idx = comm.all_to_all((order[o2] + self.base).contiguous(), sc_l, rc_l)
        assert int(got_slot.numel()) == self.n_slots, "slots received and slots owned disagree"
        value = torch.full((self.n_slots,), -1, dtype=torch.int64, device=dev)
        value[got_slot] = got_idx
        assert self.n_slots == 0 or int(value.min()) >= 0, "a slot has no source"
        self.value = value
        return self.value

    def numel(self):
        return self.n_slots


class ShardedOctree:
    """The result on one rank: `local` holds the sub-trees of this rank's cells (levels >= k) plus its collector
    content; `top` (rank 0 only) holds the nodes of levels < k.  The global octree is the union of every rank's
    level >= k nodes and rank 0's `top` nodes."""

    def __init__(self, local, top, k, recv_index, top_index, cell_to_rank, rank, stats=None):
        self.local, self.top, self.k = local, top, k
        self._recv_index, self._top_index = recv_index, top_index
        self.send_handle = None  # (ctx, handle): the sender-side per-point destinations, kept for provenance look-ups
        self.cell_to_rank, self.rank = cell_to_rank, rank
        self.stats = stats or {}
        self._nodes = None
        self.num_nodes = (int((local.meta["level"] >= k).sum()) if hasattr(local, "meta") else sum(1 for m in local.nodes.values() if m["level"] >= k)) + (
            (top.num_nodes if hasattr(top, "num_nodes") else len(top.nodes)) if top is not None else 0)

    @property
    def nodes(self):
        if self._nodes is None:
            self._nodes = {name: m for name, m in self.local.nodes.items() if m["level"] >= self.k}
            if self.top is not None:
                self._nodes.update(self.top.nodes)
        return self._nodes

    @property
    def recv_index(self):
        """Global source index per received record.  COLLECTIVE on first use when the build exchanged ingested records."""
        if isinstance(self._recv_index, LazyIndex):
            self._recv_index = self._recv_index.resolve()
        return self._recv_index

    def resolve_provenance(self, comm):
        """Collective: global source indices of the received records (every rank) and of the top nodes' points (rank 0)."""
        r_idx = self.recv_index
        if isinstance(self._top_index, dict):  # lazily gathered: {(collector, child): (owner rank, slots)} of every rank's own pieces
            mine = {key: _take(r_idx, slots) for key, slots in self._top_index.get("mine", {}).items()}
            parts = comm.all_gather_objects(mine)
            if self.rank == 0:
                allp = {}
                for part in parts:
                    allp.update(part)
                keys = sorted(allp)
                self._top_index = np.concatenate([np.asarray(allp[kk], np.uint64) for kk in keys]) if keys else np.zeros(0, np.uint64)
            else:
                self._top_index = None
        return r_idx

    @property
    def top_index(self):
        assert not isinstance(self._top_index, dict), "call resolve_provenance(comm) first (collective)"
        return self._top_index

    def free(self):
        self.local.free()
        if self.top is not None:
            self.top.free()
        if self.send_handle is not None:
            ctx, h = self.send_handle
            ctx.shard_send_free(h)
            self.send_handle = None

    def node_arrays(self, name):
        """(xyz bytes, rgb, intensity, GLOBAL source index) of one of this rank's final nodes."""
        if len(name) - 1 >= self.k:
            xyz, rgb, inten, src = self.local.node_data(name)
            return xyz, rgb, inten, _take(self.recv_index, src)
        xyz, rgb, inten, src = self.top.node_data(name)
        return xyz, rgb, inten, np.asarray(self.top_index, np.uint64)[src.astype(np.int64)]

    def gather_all(self, comm):
        """Test helper: every final node with its content on rank 0 (small clouds only)."""
        self.resolve_provenance(comm)
        mine = {}
        for name, m in self.nodes.items():
            d = dict(num_points=m["num_points"], enc=m["enc"], cube=tuple(m["cube"]))
            if m["num_points"]:
                d["xyz"], d["rgb"], d["intensity"], d["src"] = self.node_arrays(name)
            mine[name] = d
        out = {}
        for part in comm.all_gather_objects(mine):
            for name, d in part.items():
                assert name not in out, "node %s owned twice" % name
                out[name] = d
        return out


def _take(index, src):
    idx = src.astype(np.int64)
    if hasattr(index, "cpu"):
        import torch

        return index[torch.from_numpy(idx).to(index.device)].cpu().numpy().astype(np.uint64)
    return np.asarray(index)[idx].astype(np.uint64)


def build_sharded(ops, comm, index_base, prefix_levels=2, max_points_per_node=100000):
    """Backend-neutral orchestration (see module docstring)."""
    import os
    import time

    marks = [("start", time.perf_counter())]

    def mark(name):  # every phase ends in a host-visible synchronisation of the library's stream, so wall marks are device times
        marks.append((name, time.perf_counter()))

    res, bmin, bmax = ops.res, np.asarray(ops.bmin, np.float64), np.asarray(ops.bmax, np.float64)
    lo, hi = np.minimum(bmin, bmax), np.maximum(bmin, bmax)
    root_edge = max(max(hi[0] - lo[0], hi[1] - lo[1]), hi[2] - lo[2])
    nranks, rank = comm.world, comm.rank

    # (0) the bounding box is an argument of build_octree (generation.rs:292); the all-reduced box of the data is only
    # checked against it (find_bounding_box would be the producer in build_octree_from_file).
    k = int(prefix_levels)
    records = hasattr(ops, "ingest") and not os.environ.get("PCV_NO_FUSED_EXCHANGE") and k <= 2
    if records:
        return _build_sharded_records(ops, comm, index_base, k, max_points_per_node, root_edge, marks, mark)
    if hasattr(ops, "prefix_histogram_bbox"):  # one pass over the positions for both
        local_hist, lmn, lmx = ops.prefix_histogram_bbox(k)
    else:
        lmn, lmx = ops.local_bbox()
        local_hist = ops.prefix_histogram(k)
    local_hist = np.asarray(local_hist, np.uint64)
    gmn, gmx = comm.all_reduce_minmax(lmn if ops.n else [np.inf] * 3, lmx if ops.n else [-np.inf] * 3)
    inside = bool((gmn >= lo).all() and (gmx <= hi).all())

    mark("bbox + local histogram")
    # (1) global histogram of level-k cells
    counts_k = comm.all_reduce_sum_u64(local_hist)
    k2 = usable_prefix_levels(counts_k, k, root_edge, res, max_points_per_node)
    if k2 < k:
        counts_k = counts_k.reshape(8 ** k2, -1).sum(1).astype(np.uint64)
        local_hist = local_hist.reshape(8 ** k2, -1).sum(1).astype(np.uint64)
        k = k2
    levels = level_counts(counts_k, k)
    prefix_counts = concat_counts(levels)

    mark("histogram")
    # (2) cells -> ranks, (3) stable pack + one all-to-all
    c2r = assign_cells(counts_k, nranks)
    fused = hasattr(ops, "pack_exchange") and not os.environ.get("PCV_NO_FUSED_EXCHANGE")
    if fused:
        # one kernel ranks the points and stores them straight into the destination ranks' receive arrays over NVLink
        send_counts = np.array([int(local_hist[c2r == d].sum()) for d in range(nranks)], np.int64)
        recv = ops.pack_exchange(k, c2r, nranks, index_base, comm, send_counts)
        mark("pack+exchange")
        local = ops.build_sharded_soa(recv, k, prefix_counts)
        r_idx = recv.idx
        mark("local build")
    else:
        local, r_idx = _staged_exchange_and_build(ops, comm, k, c2r, nranks, index_base, prefix_counts, mark)
    stats = local.ctx.last_build_stats() if hasattr(local, "ctx") and hasattr(local.ctx, "last_build_stats") else {}
    return _finish_sharded(ops, comm, local, r_idx, k, c2r, nranks, rank, prefix_counts, stats, inside, marks, mark)


def _build_sharded_records(ops, comm, index_base, k, max_points_per_node, root_edge, marks, mark):
    """GPU path: ingest locally, exchange the records once over peer memory, build from the received records."""
    nranks, rank = comm.world, comm.rank
    local_hist = np.asarray(ops.ingest(k), np.uint64)
    mark("ingest + histogram")
    counts_k = comm.all_reduce_sum_u64(local_hist)
    k2 = usable_prefix_levels(counts_k, k, root_edge, ops.res, max_points_per_node)
    if k2 < k:
        counts_k = counts_k.reshape(8 ** k2, -1).sum(1).astype(np.uint64)
        local_hist = local_hist.reshape(8 ** k2, -1).sum(1).astype(np.uint64)
        k = k2
    prefix_counts = concat_counts(level_counts(counts_k, k))
    c2r = assign_cells(counts_k, nranks)
    send_counts = np.array([int(local_hist[c2r == d].sum()) for d in range(nranks)], np.int64)
    mark("all-reduce + plan")
    slab, n_recv, M = ops.exchange_records(k, c2r, nranks, comm, send_counts)
    mark("exchange")
    local = ops.build_from_records(slab, n_recv, k, prefix_counts)
    mark("local build")
    stats = local.ctx.last_build_stats()
    r_idx = LazyIndex(ops.ctx, ops.send, index_base, ops.n, M, comm)
    out = _finish_sharded(ops, comm, local, r_idx, k, c2r, nranks, rank, prefix_counts, stats, None, marks, mark)
    out.send_handle = (ops.ctx, ops.send)
    return out


def _staged_exchange_and_build(ops, comm, k, c2r, nranks, index_base, prefix_counts, mark):
    """Stable pack into send buffers + one NCCL / gloo all-to-all per attribute array (the path of the CPU tests, and of
    PCV_NO_FUSED_EXCHANGE=1)."""
    xyz, rgb, inten, idx, send_counts = ops.pack(k, c2r, nranks, index_base)
    mark("pack")
    recv_counts = comm.exchange_counts(send_counts)
    # one logical all-to-all, issued per attribute array; every send buffer is released as soon as it has been exchanged so
    # that the peak footprint stays at (input + largest send + receive) instead of (input + all sends + all receives)
    alloc = getattr(ops, "recv_buffer", None)
    a2a = (lambda t: comm.all_to_all(t, send_counts, recv_counts, alloc)) if alloc is not None else (lambda t: comm.all_to_all(t, send_counts, recv_counts))
    r_xyz = a2a(xyz)
    comm.done_with(xyz)
    del xyz
    r_rgb = a2a(rgb)
    r_idx = a2a(idx)
    r_int = a2a(inten) if inten is not None else None
    comm.done_with(rgb, idx, inten)
    del rgb, inten, idx

    mark("all_to_all")
    # (4) independent local build of this rank's sub-trees
    local = ops.build_sharded(r_xyz, r_rgb, r_int, k, prefix_counts)
    mark("local build")
    return local, r_idx


def _finish_sharded(ops, comm, local, r_idx, k, c2r, nranks, rank, prefix_counts, stats, inside, marks, mark):
    import os
    import time

    res = ops.res

    # (5) top of the tree: unit sizes, collectors' content -> rank 0
    unit_nsub = np.zeros(8 ** k, np.uint64)
    collectors = []  # (cell index at level k-1, node name or table position)
    if hasattr(local, "meta"):  # CUDA tree: vectorised over the node table
        meta, ns = local.meta, local.nsub_all()
        idx_mask = (1 << 60) - 1
        sel = np.nonzero(meta["level"] == k)[0]
        unit_nsub[(meta["id_low"][sel] & idx_mask).astype(np.int64)] = ns[sel]
        for i in np.nonzero((meta["level"] == k - 1) & (meta["num_points"] > 0))[0]:
            collectors.append((int(meta["id_low"][i] & idx_mask), int(i), int(meta["num_points"][i]), int(meta["enc"][i])))
        fetch = local.node_data_at
    else:
        for name, m in local.nodes.items():
            if m["level"] == k:
                unit_nsub[int(name[1:], 8)] = local.node_nsub(name)
            elif m["level"] == k - 1 and m["num_points"] > 0:
                collectors.append((int(name[1:], 8) if k > 1 else 0, name, m["num_points"], m["enc"]))
        fetch = local.node_data
    unit_nsub = comm.all_reduce_sum_u64(unit_nsub)
    pieces = {}
    lazy = isinstance(r_idx, LazyIndex)
    lazy_slots = {}
    for pidx, key, npts, enc in collectors:
        cx, cr, ci, cs = fetch(key)
        gsrc = np.asarray(cs, np.uint64) if lazy else _take(r_idx, cs)  # lazy: slots now, global indices on demand
        bpc = ENC_BYTES[enc]
        off = 0
        for c in range(8):
            cell = pidx * 8 + c
            if c2r[cell] != rank or unit_nsub[cell] == 0:
                continue
            cnt = (int(unit_nsub[cell]) + 7) // 8
            pieces[(pidx, c)] = (cx[off * 3 * bpc:(off + cnt) * 3 * bpc].copy(), cr[off * 3:(off + cnt) * 3].copy(), None if ci is None else ci[off:off + cnt].copy(),
                                 None if lazy else gsrc[off:off + cnt].copy())
            if lazy:
                lazy_slots[(pidx, c)] = gsrc[off:off + cnt].copy()
            off += cnt
        assert off == npts, (pidx, off, npts)
    top, top_index = None, None
    if hasattr(comm, "all_gather_bytes") and lazy:
        # Every rank can derive every rank's piece list (cell order) from the all-reduced unit sizes and the cell -> rank map, so
        # the collectors' content travels as ONE padded byte tensor per rank: [xyz of its pieces | rgb | intensity].
        has_int = getattr(ops, "intensity", None) is not None
        enc_all = comm.all_gather_counts([max([e for _, _, _, e in collectors], default=0)])
        bpc = ENC_BYTES[int(enc_all.max())] if int(enc_all.max()) else 1
        owned = [[] for _ in range(nranks)]  # per rank: (cell, count) in cell order
        for cell in range(8 ** k):
            if unit_nsub[cell]:
                owned[int(c2r[cell])].append((cell, (int(unit_nsub[cell]) + 7) // 8))
        per_pt = 3 * bpc + 3 + (4 if has_int else 0)
        nbytes = [sum(c for _, c in lst) * per_pt for lst in owned]
        mine = owned[rank]
        parts = [[], [], []]
        for cell, cnt in mine:
            px, pr, pi, _ = pieces[(cell // 8, cell % 8)]
            assert len(pr) == 3 * cnt, (cell, len(pr), cnt)
            parts[0].append(np.asarray(px, np.uint8))
            parts[1].append(np.asarray(pr, np.uint8))
            if has_int:
                parts[2].append(np.asarray(pi, np.float32).view(np.uint8))
        buf = np.concatenate([a for grp in parts for a in grp]) if mine else np.zeros(0, np.uint8)
        assert len(buf) == nbytes[rank]
        allb = comm.all_gather_bytes(buf, max(max(nbytes), 16))
        if rank == 0:
            xs, rs, its = {}, {}, {}
            for r in range(nranks):
                tot = sum(c for _, c in owned[r])
                row, ox, orr, oi = allb[r], 0, tot * 3 * bpc, tot * (3 * bpc + 3)
                for cell, cnt in owned[r]:
                    xs[cell] = row[ox:ox + cnt * 3 * bpc]
                    rs[cell] = row[orr:orr + cnt * 3]
                    ox += cnt * 3 * bpc
                    orr += cnt * 3
                    if has_int:
                        its[cell] = row[oi:oi + cnt * 4]
                        oi += cnt * 4
            cells = sorted(xs)
            t_xyz = np.concatenate([xs[c] for c in cells]) if cells else np.zeros(0, np.uint8)
            t_rgb = np.concatenate([rs[c] for c in cells]) if cells else np.zeros(0, np.uint8)
            t_int = np.concatenate([its[c] for c in cells]).view(np.float32) if (cells and has_int) else None
            top = ops.assemble_top(k, prefix_counts, unit_nsub, t_xyz, t_rgb, t_int)
    else:
        gathered = comm.all_gather_objects(pieces)
        if rank == 0:
            allp = {}
            for part in gathered:
                allp.update(part)
            keys = sorted(allp)
            cat = lambda i, dt: np.concatenate([np.asarray(allp[kk][i]) for kk in keys]).astype(dt) if keys else np.zeros(0, dt)
            t_xyz, t_rgb = cat(0, np.uint8), cat(1, np.uint8)
            top_index = None if lazy else cat(3, np.uint64)
            t_int = cat(2, np.float32) if (keys and allp[keys[0]][2] is not None) else None
            top = ops.assemble_top(k, prefix_counts, unit_nsub, t_xyz, t_rgb, t_int)
    if lazy:
        top_index = {"mine": lazy_slots}
    mark("top assembly")
    if os.environ.get("PCV_TIMING") and rank == 0:
        print("[pcv sharded] " + "  ".join("%s %.1f ms" % (marks[i][0], (marks[i][1] - marks[i - 1][1]) * 1e3) for i in range(1, len(marks))), file=sys.stderr, flush=True)
    out = ShardedOctree(local, top, k, r_idx, top_index, c2r, rank, stats)
    out.bbox_inside = inside
    out.recv_points = int(r_idx.numel()) if hasattr(r_idx, "numel") else len(r_idx)
    out.phases_ms = {marks[i][0]: (marks[i][1] - marks[i - 1][1]) * 1e3 for i in range(1, len(marks))}
    return out


def make_c_comm(comm):
    """pcv_comm over a TorchComm (or any object with all_reduce_sum_u64 / all_gather_bytes / barrier): the three collectives
    pcv_build_octree_sharded needs, as C callbacks over host buffers.  Keep the returned struct alive for the call."""
    import ctypes as C

    from . import _native as N

    def allreduce(_user, ptr, count):
        try:
            a = np.ctypeslib.as_array(ptr, shape=(int(count),))
            a[:] = comm.all_reduce_sum_u64(a.copy())
            return 0
        except Exception:  # noqa: BLE001 - an exception must not unwind through the C frame
            import traceback

            traceback.print_exc()
            return 1

    def allgather(_user, send, nbytes, recv):
        try:
            nbytes = int(nbytes)
            src = np.frombuffer((C.c_uint8 * nbytes).from_address(send), np.uint8)
            out = comm.all_gather_bytes(src, nbytes)
            C.memmove(recv, out.ctypes.data, comm.world * nbytes)
            return 0
        except Exception:  # noqa: BLE001
            import traceback

            traceback.print_exc()
            return 1

    def barrier(_user):
        try:
            comm.barrier()
            return 0
        except Exception:  # noqa: BLE001
            import traceback

            traceback.print_exc()
            return 1

    cs = N.Comm(None, comm.rank, comm.world, N.ALLREDUCE_FN(allreduce), N.ALLGATHER_FN(allgather), N.BARRIER_FN(barrier))
    return cs


def build_octree_sharded_native(ctx, x, y, z, rgb, intensity, index_base, resolution, bbox_min, bbox_max, prefix_levels=2, comm=None):
    """Same result as build_octree_sharded, but the whole orchestration runs inside the C library (pcv_build_octree_sharded):
    Python only lends it torch.distributed's collectives.  This is the call a non-Python host makes with its own NCCL / MPI."""
    comm = comm or TorchComm(x.device)
    cs = make_c_comm(comm)
    n = int(x.numel())
    local, top, k, c2r, unit_nsub, n_recv, send = ctx.build_octree_sharded(cs, x.data_ptr(), y.data_ptr(), z.data_ptr(), 1, rgb.data_ptr(),
                                                                           intensity.data_ptr() if intensity is not None else None, n, resolution, bbox_min,
                                                                           bbox_max, prefix_levels)
    stats = ctx.last_build_stats()
    # provenance, all on demand: slots of the received points from the senders' per-point bytes, slots of the top pieces from
    # the local tree
    import torch

    if ctx.shard_send_cells(send) is not None:  # the fused exchange pass ran
        r_idx = LazyCellIndex(ctx, send, index_base, n, c2r, n_recv, comm)
    else:
        r_idx = LazyIndex(ctx, send, index_base, n, None, comm, n_recv)  # the count matrix is derived on first use
    lazy_slots = {}
    meta = local.meta
    idx_mask = (1 << 60) - 1
    for i in np.nonzero((meta["level"] == k - 1) & (meta["num_points"] > 0))[0]:
        pidx = int(meta["id_low"][i] & idx_mask) if k > 1 else 0
        cs_ = np.asarray(local.node_data_at(int(i))[3], np.uint64)
        off = 0
        for c in range(8):
            cell = pidx * 8 + c
            if c2r[cell] != comm.rank or unit_nsub[cell] == 0:
                continue
            cnt = (int(unit_nsub[cell]) + 7) // 8
            lazy_slots[(pidx, c)] = cs_[off:off + cnt].copy()
            off += cnt
    out = ShardedOctree(local, top, k, r_idx, {"mine": lazy_slots}, c2r, comm.rank, stats)
    out.send_handle = (ctx, send)
    out.recv_points = r_idx.numel()
    out.phases_ms = ctx.sharded_phases()
    out.c_comm = cs  # keeps the callbacks alive as long as the tree (pcv_sharded_release takes the same struct)
    return out


def build_octree_sharded(ctx, x, y, z, rgb, intensity, index_base, resolution, bbox_min, bbox_max, prefix_levels=2, max_points_per_node=100000,
                         consume_input=False):
    """GPU entry point used by bench.py: torch cuda tensors in, ShardedOctree out (torch.distributed must be initialised).
    consume_input=True releases pool-backed (Context.device_buffer) input tensors right after the pack, which is what lets
    1e9 points per GPU fit: input 27 GB -> send 35 GB -> receive 35 GB -> build working set ~80 GB, never all at once."""
    ops = CudaOps(ctx, x, y, z, rgb, intensity, resolution, bbox_min, bbox_max, consume_input=consume_input)
    comm = TorchComm(x.device)
    return build_sharded(ops, comm, index_base, prefix_levels, max_points_per_node)
