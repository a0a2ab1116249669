"""Many-sensor frames sharded across GPUs (SURVEY.md section 8(e)): one process per GPU, replicated grid,
each rank fuses its own sensors' clouds, and the per-cell partial results are all-reduced over
NCCL / NVLink between the phases of the frame:

    begin (index + error count)  -> exchange 1: counts (int32 SUM), drift statistics (int64 SUM)
    phase 1 (drift, Kalman)      -> exchange 2: sum new_h / new_v (int64 SUM, 2^-32 fixed point), counts
                                                (int32 SUM), last-writer keys (int64 MAX)
    phase 2 (ray-cast)           -> exchange 3: validity decrements (int64 SUM), counts (int32 SUM),
                                                upper-bound keys (int32 MIN)
    phase 3 (finalise + dilation + traversability + normals), identical on every rank.

Semantic channels of the kinds that reduce as sums (average, class_average, color, class_bayesian, bayesian_inference)
are summed by each rank in phase 1, reduced with exchange 2 (int64 / int32 SUM) and written to every replica's layers in
phase 3; class_max is refused.  Depth cameras shard like clouds: a rank's rows are its cameras' pixels, offset by the
pixels of the lower ranks' cameras.

Every reduction is over integers, so the replicas stay bit-identical and the result equals the
single-GPU `input_sensors` of the concatenated clouds bit for bit (which tests/ check against the oracle).
The reference has no multi-GPU path (SURVEY 2.1); sensors there are fused sequentially.
"""
import ctypes as C

import numpy as np

from . import _lib

# emap_exchange.kind -> (torch dtype name, reduce op name)
KIND = {0: ("int64", "SUM"), 1: ("int64", "MAX"), 2: ("int32", "MIN"), 3: ("int32", "SUM")}
_TYPESTR = {"int64": "<i8", "int32": "<i4"}


class _Buf:
    def __init__(self, ptr, count, typestr, owner):
        self.__cuda_array_interface__ = {"shape": (int(count),), "typestr": typestr, "data": (int(ptr), False),
                                         "version": 3, "strides": None}
        self._owner = owner


def reduce_plan(exchanges):
    """[(ptr, count, kind)] -> [(ptr, count, dtype_name, op_name)] (pure host logic, unit-tested on CPU)."""
    return [(p, n, *KIND[k]) for (p, n, k) in exchanges]


def all_reduce_buffers(tensors_and_ops, group=None):
    """In-place all-reduce of each (tensor, op_name); works for NCCL (CUDA tensors) and gloo (CPU)."""
    import torch.distributed as dist
    ops = {"SUM": dist.ReduceOp.SUM, "MAX": dist.ReduceOp.MAX, "MIN": dist.ReduceOp.MIN}
    for t, op in tensors_and_ops:
        dist.all_reduce(t, op=ops[op], group=group)


def split_exchange2(todo):
    """Exchange 2's arrays as (critical, deferred): only the fused counts, listed second, gate the ray-cast of phase 2;
    the height sums, last-writer keys and semantic sums are read in phase 3 (pure host logic, unit-tested on CPU)."""
    return todo[1:2], todo[:1] + todo[2:]


def depth_frame_offsets(pixels, first_z, group=None, static_offsets=None, overlap_z=None):
    """(row offset, overlap z) of this rank's cameras in a sharded depth frame: the pixels (height * width summed) of the
    lower ranks' cameras, or static_offsets[0]; `overlap_z`, or rank 0's first camera's t[2].  One all_gather of
    (pixels, first_z) when either has to be found."""
    if static_offsets is not None and overlap_z is not None:
        return int(static_offsets[0]), float(overlap_z)
    import torch
    import torch.distributed as dist
    ws, rk = dist.get_world_size(group), dist.get_rank(group)
    dev = "cuda" if dist.get_backend(group) == "nccl" else "cpu"
    mine = torch.tensor([float(pixels), float(first_z)], dtype=torch.float64, device=dev)     # exact below 2^53 pixels
    allv = [torch.zeros_like(mine) for _ in range(ws)]
    dist.all_gather(allv, mine, group=group)
    rows = [v.tolist() for v in allv]
    off = int(static_offsets[0]) if static_offsets is not None else int(sum(r[0] for r in rows[:rk]))
    return off, float(overlap_z) if overlap_z is not None else rows[0][1]


def global_point_offsets(local_count, group=None):
    """Rank-ordered exclusive prefix of the per-rank point counts: (my_offset, total)."""
    import torch
    import torch.distributed as dist
    ws, rk = dist.get_world_size(group), dist.get_rank(group)
    dev = "cuda" if dist.get_backend(group) == "nccl" else "cpu"
    mine = torch.tensor([int(local_count)], dtype=torch.int64, device=dev)
    allc = [torch.zeros_like(mine) for _ in range(ws)]
    dist.all_gather(allc, mine, group=group)
    counts = [int(c.item()) for c in allc]
    return sum(counts[:rk]), sum(counts)


class ShardedElevationMap:
    """Wraps one ElevationMap replica per rank; `input_sensors` is collective over `group`."""

    def __init__(self, elevation_map, group=None, static_offsets=None, mode="auto"):
        """mode: "multicast" (NVLink multicast reductions fused into the kernels), "nccl" (three integer
        all-reduces per frame) or "auto" (multicast when the fabric offers a multicast pointer)."""
        import torch
        self.em = elevation_map
        self.group = group
        self.torch = torch
        self.static_offsets = static_offsets      # (my_offset, total) when every rank's count is fixed
        em = self.em
        # run the library on one explicit torch stream so that kernels and NCCL collectives are stream-ordered
        # (the legacy default stream, handle 0, cannot be named through the C ABI)
        cur = torch.cuda.current_stream()
        self.stream = cur if cur.cuda_stream != 0 else torch.cuda.Stream()
        em._check(em._L.emap_set_stream(em._h, C.c_void_p(self.stream.cuda_stream)))
        self.side = torch.cuda.Stream()
        self._cache = {}
        self.mode = "nccl"
        self._symm = None
        if mode in ("auto", "multicast"):
            ok = self._attach_multicast()
            if not ok and mode == "multicast":
                raise RuntimeError("NVLink multicast is not available on this fabric")

    def _attach_multicast(self, required=False):
        """Attaches a symmetric block of emap_shard_scratch_bytes() (collective).  Without multicast support: False, or
        an error when `required` (a re-attach of a handle that was attached)."""
        import torch.distributed as dist
        torch = self.torch
        em = self.em
        try:
            import torch.distributed._symmetric_memory as symm_mem
            nbytes = int(em._L.emap_shard_scratch_bytes(em._h))
            buf = symm_mem.empty(nbytes, dtype=torch.uint8, device=f"cuda:{em.device}")
            grp = self.group if self.group is not None else dist.group.WORLD
            hdl = symm_mem.rendezvous(buf, grp.group_name)
            mc = int(hdl.multicast_ptr)
        except Exception as e:          # no symmetric-memory support in this build / fabric
            if required:
                raise
            print(f"[sharded] multicast unavailable ({type(e).__name__}: {e}); using NCCL all-reduces")
            return False
        if mc == 0:
            if required:
                raise RuntimeError("NVLink multicast is not available for the re-attached block")
            return False
        torch.cuda.synchronize()
        em._check(em._L.emap_shard_attach(em._h, C.c_void_p(buf.data_ptr()), C.c_void_p(mc), nbytes))
        hdl.barrier()
        torch.cuda.synchronize()
        self._symm = (buf, hdl, nbytes)        # the block it replaces is released here, after the attach
        self.mode = "multicast"
        return True

    def _fit_block(self):
        """Multicast mode: a new block when the semantic configuration outgrew the attached one.  Collective, like the
        configuration itself: every rank configures the same channels in the same call."""
        em = self.em
        if self.mode == "multicast" and int(em._L.emap_shard_scratch_bytes(em._h)) > self._symm[2]:
            self._attach_multicast(required=True)

    def _plan(self, phase):
        em = self.em
        arr = (_lib.EmapExchange * _lib.EMAP_SHARD_MAX_EXCHANGES)()
        n = C.c_int32(_lib.EMAP_SHARD_MAX_EXCHANGES)
        em._check(em._L.emap_shard_exchange(em._h, phase, arr, C.byref(n)))
        plan = reduce_plan([(arr[i].ptr, arr[i].count, arr[i].kind) for i in range(n.value)])
        todo = []
        for ptr, count, dt, op in plan:
            key = (ptr, count, dt)
            t = self._cache.get(key)
            if t is None:
                t = self.torch.as_tensor(_Buf(ptr, count, _TYPESTR[dt], em), device=f"cuda:{em.device}")
                self._cache[key] = t
            todo.append((t, op))
        return todo

    def _exchange(self, phase):
        all_reduce_buffers(self._plan(phase), self.group)

    def _exchange2_overlapped(self):
        """Exchange 2: only the counts (cnt_fused | n_out) gate the ray-cast; the fixed-point sums, the last-writer keys
        and the semantic sums are consumed in phase 3, so their all-reduces run on a side stream under the ray-cast.
        Returns the pending work handles."""
        import torch.distributed as dist
        ops = {"SUM": dist.ReduceOp.SUM, "MAX": dist.ReduceOp.MAX, "MIN": dist.ReduceOp.MIN}
        critical, deferred = split_exchange2(self._plan(2))
        all_reduce_buffers(critical, self.group)
        self.side.wait_stream(self.stream)
        works = []
        with self.torch.cuda.stream(self.side):
            for t, op in deferred:
                works.append(dist.all_reduce(t, op=ops[op], group=self.group, async_op=True))
        return works

    def input_sensors(self, clouds, Rs, ts, position_noise, orientation_noise, device_ptrs=False, overlap_z=None,
                      channels=None):
        """`overlap_z`: absolute z of the frame's first sensor (rank 0's), the same value on every rank.  `channels`:
        the clouds' channel names as ElevationMap.input_pointcloud takes them, the same on every rank."""
        em = self.em
        from .elevation_mapping import _clouds, _to_host
        em._configure_cloud_channels(channels)
        ptrs, counts, stride, dt, _keep = _clouds(clouds, device_ptrs)
        ns = len(counts)
        total_local = sum(int(c) for c in counts)
        off, _total = self.static_offsets if self.static_offsets else global_point_offsets(total_local, self.group)
        Rm = np.ascontiguousarray(np.stack([np.asarray(_to_host(r), np.float32).reshape(9) for r in Rs]))
        tm = np.ascontiguousarray(np.stack([np.asarray(_to_host(t), np.float32).reshape(3) for t in ts]))
        L, h = em._L, em._h
        self.stream.wait_stream(self.torch.cuda.current_stream())
        with self.torch.cuda.stream(self.stream):
            self._frame(lambda: L.emap_shard_begin(h, ns, ptrs, counts, stride, dt, int(bool(device_ptrs)), Rm.ctypes.data,
                                                   tm.ctypes.data, off, float(position_noise), float(orientation_noise)),
                        overlap_z)
        self.torch.cuda.current_stream().wait_stream(self.stream)

    def input_depth_images(self, cameras, position_noise, orientation_noise, channels=(), confidence_threshold=10.0,
                           max_depth=8.0, overlap_z=None):
        """This rank's depth cameras of one sharded frame, collective over `group`: cameras and channels as
        ElevationMap.input_depth_images (the same channels on every rank).  The frame's rows are the pixels of every
        rank's cameras in rank order (static_offsets, if given, count pixels); `overlap_z` defaults to rank 0's first
        camera's t[2]."""
        em = self.em
        depth = em._depth_frame(cameras, channels)
        off, z = depth_frame_offsets(depth.pixels, depth.first_z, self.group, self.static_offsets, overlap_z)
        L, h = em._L, em._h
        self.stream.wait_stream(self.torch.cuda.current_stream())
        with self.torch.cuda.stream(self.stream):
            self._frame(lambda: L.emap_shard_begin_depth_images(h, *depth.args, float(confidence_threshold),
                                                                float(max_depth), off, float(position_noise),
                                                                float(orientation_noise)), z)
        # the converted images in depth.keep are freed on return: their stream's later work follows the frame's
        self.torch.cuda.current_stream().wait_stream(self.stream)

    def _frame(self, begin, overlap_z):
        """One sharded frame after `begin()` (an emap_shard_begin* call) on the library's stream."""
        em = self.em
        L, h = em._L, em._h
        self._fit_block()
        em._check(begin())
        if overlap_z is not None:
            em._check(L.emap_shard_set_overlap_z(h, float(overlap_z)))
        if self.mode == "multicast":
            # every accumulation of the frame kernels is a multimem.red applied to all replicas by the switch;
            # only stream-ordered cross-rank barriers separate the phases (no NCCL, no host sync)
            bar = self._symm[1].barrier
            bar()                                   # all ranks have reset their frame scalars / finished the last frame
            em._check(L.emap_shard_phase(h, 0)); bar()
            em._check(L.emap_shard_phase(h, 1)); bar()
            em._check(L.emap_shard_phase(h, 2)); bar()
            em._check(L.emap_shard_phase(h, 3))
            return
        self._exchange(1)
        em._check(L.emap_shard_phase(h, 1))
        works = self._exchange2_overlapped()
        em._check(L.emap_shard_phase(h, 2))
        self._exchange(3)
        with self.torch.cuda.stream(self.side):
            for w in works:
                w.wait()
        self.stream.wait_stream(self.side)
        em._check(L.emap_shard_phase(h, 3))
