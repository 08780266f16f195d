"""Host-side mirror of cartographer::mapping::constraints::ConstraintBuilder2D
(cartographer/mapping/internal/constraints/constraint_builder_2d.{h,cc}) for the
fast-correlative-scan-matching part of the queue.

Same public surface and gating as the reference —
  MaybeAddConstraint / MaybeAddGlobalConstraint / NotifyEndOfNode / WhenDone /
  GetNumFinishedNodes / DeleteScanMatcher
— but instead of one thread-pool task per (submap, node) pair the queued pairs are
drained as ONE batched device call (csm_match2d_batch) when WhenDone is invoked.
With torch.distributed initialised the queue is sharded submap-major across ranks
(rank r owns the submaps whose first-use order index % world == r; stacks are
only built on their owner) and the fixed-size constraint records are exchanged
with a single all_gather; every rank then reports the same Result in queue order.

By default constraints are the fast matcher's: `pose` is ComputeSubmapPose(submap)^-1 *
pose_estimate (constraint_builder_2d.cc:251-258), which is what the bit-exact parity
tests pin.  With ConstraintBuilderOptions.ceres_scan_matcher_options set, every found
match is first refined as constraint_builder_2d.cc:245-249 does — all of a drain's
matches in one csm_ceres_match2d_batch launch (scan_matching.CeresScanMatcher2D; Ceres
itself is not linked, see DESIGN.md).
"""
import math
from dataclasses import dataclass, field

import numpy as np

RECORD_DTYPE = np.dtype([("submap_trajectory", "<i4"), ("submap_index", "<i4"),
                         ("node_trajectory", "<i4"), ("node_index", "<i4"),
                         ("found", "<u4"), ("score", "<f4"), ("pose", "<f8", (3,)),
                         ("pad", "<u4", (4,))], align=True)
assert RECORD_DTYPE.itemsize == 64


@dataclass
class ConstraintBuilderOptions:
    """constraints/proto/constraint_builder_options.proto (the fields on the path);
    defaults from configuration_files/pose_graph.lua:18-36."""
    sampling_ratio: float = 0.3
    max_constraint_distance: float = 15.0
    min_score: float = 0.55
    global_localization_min_score: float = 0.6
    loop_closure_translation_weight: float = 1.1e4
    loop_closure_rotation_weight: float = 1e5
    linear_search_window: float = 7.0
    angular_search_window: float = math.radians(30.0)
    branch_and_bound_depth: int = 7
    # scan_matching.CeresScanMatcherOptions2D, or None to leave matches unrefined
    ceres_scan_matcher_options: object = None


@dataclass
class Submap2D:
    """What the builder needs of a Submap2D: its grid and local pose (x, y, yaw).

    The grid is either a host record (.cells, .resolution, .max_x, .max_y, .min_cost,
    .max_cost) or, for a finished submap kept on the device as
    ProbabilityGridRangeDataInserter2D fills it and RealTimeGrid2D.ComputeCroppedGrid crops it,
    a ProbabilityGrid scan_matching.RealTimeGrid2D on the builder's device.  A device submap's
    stack and refinement read its grid where it is; the caller keeps it alive until WhenDone
    has run its callback, and DeleteScanMatcher never closes it."""
    grid: object
    local_pose: tuple = (0.0, 0.0, 0.0)


def _is_device_grid(grid, device):
    """True for a Submap2D grid that is a RealTimeGrid2D, False for a host record; ValueError
    for a TSDF handle (it has no precomputation stack) or one on another device than
    `device`.  Reads only the handle's attributes: nothing reaches the library."""
    from .scan_matching import RealTimeGrid2D
    if not isinstance(grid, RealTimeGrid2D):
        return False
    if grid.is_tsdf:
        raise ValueError("Submap2D: a TSDF RealTimeGrid2D cannot close loops")
    if grid.device != device:
        raise ValueError("Submap2D: the grid lives on device %d, the builder on device %d"
                         % (grid.device, device))
    return True


@dataclass
class Constraint:
    """PoseGraphInterface::Constraint (mapping/pose_graph_interface.h:36-53)."""
    submap_id: tuple
    node_id: tuple
    zbar_ij: tuple            # (x, y, yaw) of submap i <- node j
    translation_weight: float
    rotation_weight: float
    tag: str = "INTER_SUBMAP"
    score: float = 0.0


class FixedRatioSampler:
    """common/fixed_ratio_sampler.cc:23-39."""

    def __init__(self, ratio):
        if not 0.0 <= ratio <= 1.0:
            raise ValueError("ratio must be in [0, 1]")
        self.ratio = ratio
        self.num_pulses = 0
        self.num_samples = 0

    def Pulse(self):
        self.num_pulses += 1
        if self.num_samples / self.num_pulses < self.ratio:
            self.num_samples += 1
            return True
        return False


def _compose(a, b):
    """transform::Rigid2d operator* (transform/rigid_transform.h:93-99)."""
    c, s = math.cos(a[2]), math.sin(a[2])
    return (c * b[0] - s * b[1] + a[0], s * b[0] + c * b[1] + a[1], a[2] + b[2])


def _inverse(a):
    """Rigid2::inverse (transform/rigid_transform.h:76-80)."""
    c, s = math.cos(-a[2]), math.sin(-a[2])
    return (-(c * a[0] - s * a[1]), -(s * a[0] + c * a[1]), -a[2])


@dataclass
class _Job:
    submap_id: tuple
    node_id: tuple
    cloud_key: int
    initial_pose: tuple
    full: bool
    min_score: float


class CudaExecutor:
    """Drains a list of jobs through csm_match2d_batch on one device.  Keeps one
    device stack per submap (DispatchScanMatcherConstruction,
    constraint_builder_2d.cc:165-186) and one device cloud per node scan.  A device
    submap's stack is built from its RealTimeGrid2D without a host copy, and its
    refinement reads that grid directly."""

    def __init__(self, options, device=0):
        from . import scan_matching as sm
        self.sm = sm
        self.options = options
        self.device = device
        self.matchers = {}
        # submap id -> RealTimeGrid2D uploaded for the Ceres refinement (host submaps only)
        self.grids = {}
        self.clouds = {}
        self.stats = {"candidates_scored": 0, "device_ms": 0.0, "searched": 0, "refined": 0,
                      "refine_device_ms": 0.0}

    def ensure_matcher(self, submap_id, grid):
        if submap_id not in self.matchers:
            o = self.options
            fo = self.sm.FastCorrelativeScanMatcherOptions2D(
                o.linear_search_window, o.angular_search_window, o.branch_and_bound_depth)
            if _is_device_grid(grid, self.device):
                m = self.sm.FastCorrelativeScanMatcher2D.from_device_grid(grid, fo)
            else:
                m = self.sm.FastCorrelativeScanMatcher2D(grid, fo, device=self.device)
            self.matchers[submap_id] = m

    def delete_matcher(self, submap_id):
        m = self.matchers.pop(submap_id, None)
        if m is not None:
            m.close()
        g = self.grids.pop(submap_id, None)
        if g is not None:
            g.close()

    def refine(self, jobs, submaps, clouds, out):
        """constraint_builder_2d.cc:245-249 for every found match of the drain, one launch."""
        sm = self.sm
        idx = [i for i, r in enumerate(out) if r[0]]
        if not idx:
            return out
        grids = []
        for i in idx:
            sid = jobs[i].submap_id
            grid = submaps[sid].grid
            if not _is_device_grid(grid, self.device):
                if sid not in self.grids:
                    self.grids[sid] = sm.RealTimeGrid2D(grid, device=self.device)
                grid = self.grids[sid]
            grids.append(grid)
        matcher = sm.CeresScanMatcher2D(self.options.ceres_scan_matcher_options)
        poses, _ = matcher.MatchBatch([out[i][2][:2] for i in idx], [out[i][2] for i in idx],
                                      [clouds[jobs[i].cloud_key] for i in idx], grids)
        self.stats["refined"] += len(idx)
        self.stats["refine_device_ms"] += matcher.last_stats["device_ms"]
        out = list(out)
        for i, p in zip(idx, poses):
            out[i] = (True, out[i][1], (float(p[0]), float(p[1]), float(p[2])))
        return out

    def run(self, jobs, submaps, clouds):
        """-> list of (found, score, pose_estimate) in job order."""
        if not jobs:
            return []
        sm = self.sm
        sub_ids = sorted({j.submap_id for j in jobs})
        for sid in sub_ids:
            self.ensure_matcher(sid, submaps[sid].grid)
        cloud_keys = sorted({j.cloud_key for j in jobs})
        for k in cloud_keys:
            if k not in self.clouds:
                self.clouds[k] = sm.DeviceCloud(clouds[k], device=self.device)
        sidx = {s: i for i, s in enumerate(sub_ids)}
        cidx = {k: i for i, k in enumerate(cloud_keys)}
        arr = np.zeros(len(jobs), sm.JOB2D_DTYPE)
        for i, j in enumerate(jobs):
            arr[i]["stack_index"] = sidx[j.submap_id]
            arr[i]["cloud_index"] = cidx[j.cloud_key]
            arr[i]["full_submap"] = int(j.full)
            arr[i]["initial_pose"] = j.initial_pose
            arr[i]["min_score"] = j.min_score
        res, st = sm.match_batch([self.matchers[s] for s in sub_ids],
                                 [self.clouds[k] for k in cloud_keys], arr,
                                 self.options.linear_search_window,
                                 self.options.angular_search_window)
        self.stats["candidates_scored"] += st["candidates_scored"]
        self.stats["device_ms"] += st["device_ms"]
        self.stats["searched"] += len(jobs)
        out = [(bool(r["found"]), float(r["score"]), tuple(r["pose_estimate"])) for r in res]
        if self.options.ceres_scan_matcher_options is not None:
            out = self.refine(jobs, submaps, clouds, out)
        return out

    def release_clouds(self):
        for c in self.clouds.values():
            c.close()
        self.clouds = {}


class _ConstraintQueue:
    """What ConstraintBuilder2D and ConstraintBuilder3D share: the queue of (submap, node)
    pairs, the per-submap FixedRatioSamplers, the node counters and the WhenDone drain.

    With a `process_group` (torch.distributed) or a `context` (scan_matching.MultiGpuContext)
    the queue is sharded submap-major: rank r runs the pairs of the submaps whose first-use
    order % world == r, and one all-gather of fixed-size records (RECORD) gives every rank the
    whole Result in queue order.  A dimension supplies its record dtype, `_fill` (one executor
    result -> one record), `_is_device` and its MaybeAdd*Constraint gates."""

    RECORD = None

    def __init__(self, options, executor, process_group, device, context=None):
        self.options = options
        self.executor = executor
        self.pg = process_group
        self.ctx = context
        self.device = device
        self._jobs = []
        self._submaps = {}
        self._constant_data = {}   # id(constant_data) -> the node's cloud / data
        self._submap_order = {}
        self._samplers = {}
        self._when_done = None
        self.num_started_nodes = 0
        self.num_finished_nodes = 0
        self.last_records = None

    def _world(self):
        if self.ctx is not None:
            return self.ctx.rank, self.ctx.world_size
        if self.pg is None:
            return 0, 1
        import torch.distributed as dist
        return dist.get_rank(self.pg), dist.get_world_size(self.pg)

    # -- queue --------------------------------------------------------------------
    def _check_submap(self, submap):
        """Refuses, before any gate, a device submap the builder cannot use (see `_is_device`),
        or any device submap when the queue is sharded over several ranks (a device submap
        stays on the GPU that inserted it)."""
        if self._is_device(submap) and self._world()[1] > 1:
            raise ValueError("device-resident submaps are not sharded over several ranks")

    def _pulse(self, submap_id):
        """The per-submap FixedRatioSampler of constraint_builder_2d.cc:85-90."""
        sampler = self._samplers.setdefault(submap_id,
                                            FixedRatioSampler(self.options.sampling_ratio))
        return sampler.Pulse()

    def _register(self, submap_id, submap, constant_data):
        self._submaps[submap_id] = submap
        self._submap_order.setdefault(submap_id, len(self._submap_order))
        key = id(constant_data)
        self._constant_data[key] = constant_data
        return key

    def NotifyEndOfNode(self):
        """constraint_builder_2d.cc:139-151 (the node finishes when WhenDone drains)."""
        self.num_started_nodes += 1

    def GetNumFinishedNodes(self):
        return self.num_finished_nodes

    def DeleteScanMatcher(self, submap_id):
        """constraint_builder_2d.cc:307-316."""
        if hasattr(self.executor, "delete_matcher"):
            self.executor.delete_matcher(submap_id)
        self._samplers.pop(submap_id, None)

    # -- drain ---------------------------------------------------------------------
    def WhenDone(self, callback):
        """constraint_builder_2d.cc:153-163 + RunWhenDoneCallback :279-300: runs the
        queue, then calls callback(Result) with the found constraints in queue order."""
        if self._when_done is not None:
            raise RuntimeError("WhenDone called twice")  # CHECK(when_done_ == nullptr)
        self._when_done = callback
        rank, world = self._world()
        jobs = self._jobs
        owner = [self._submap_order[j.submap_id] % world for j in jobs]
        mine = [i for i, o in enumerate(owner) if o == rank]
        out = self.executor.run([jobs[i] for i in mine], self._submaps, self._constant_data)
        local = np.zeros(len(mine), self.RECORD)
        for rec, i, r in zip(local, mine, out):
            j = jobs[i]
            rec["submap_trajectory"], rec["submap_index"] = j.submap_id
            rec["node_trajectory"], rec["node_index"] = j.node_id
            self._fill(rec, j, r)
        records = self._exchange(local, owner, world)
        self.last_records = records
        result = [Constraint((int(r["submap_trajectory"]), int(r["submap_index"])),
                             (int(r["node_trajectory"]), int(r["node_index"])),
                             tuple(float(v) for v in r["pose"]),
                             self.options.loop_closure_translation_weight,
                             self.options.loop_closure_rotation_weight, "INTER_SUBMAP",
                             float(r["score"])) for r in records if r["found"]]
        self._jobs = []
        self._constant_data = {}
        if hasattr(self.executor, "release_clouds"):
            self.executor.release_clouds()
        self.num_finished_nodes = self.num_started_nodes
        cb, self._when_done = self._when_done, None
        cb(result)
        return result

    def _exchange(self, local, owner, world):
        """The queue's single collective: every rank's records, padded to the largest shard,
        gathered to every rank (ncclAllGather inside the library with a `context`, else
        all_gather_into_tensor on the process group) and put back in queue order."""
        if world == 1:
            return local
        cap = max(1, max(owner.count(r) for r in range(world)))
        send = np.zeros(cap, local.dtype)
        send[:len(local)] = local
        if self.ctx is not None:
            raw = b"".join(self.ctx.allgather(send.tobytes()))
        else:
            import torch
            import torch.distributed as dist
            dev = (torch.device("cuda", self.device) if dist.get_backend(self.pg) == "nccl"
                   else torch.device("cpu"))
            t_send = torch.from_numpy(send.view(np.uint8).reshape(-1).copy()).to(dev)
            t_recv = torch.empty(world * send.nbytes, dtype=torch.uint8, device=dev)
            dist.all_gather_into_tensor(t_recv, t_send, group=self.pg)
            raw = t_recv.cpu().numpy().tobytes()
        allrec = np.frombuffer(raw, dtype=local.dtype).reshape(world, cap)
        out = np.zeros(len(owner), local.dtype)
        cursor = [0] * world
        for i, r in enumerate(owner):
            out[i] = allrec[r, cursor[r]]
            cursor[r] += 1
        return out


class ConstraintBuilder2D(_ConstraintQueue):
    """constraint_builder_2d.h:60-107.  `executor.run(jobs, submaps, clouds)` does the
    matching (CudaExecutor in production); `process_group` (torch.distributed) turns
    on submap-major sharding + the single all_gather of constraint records."""

    RECORD = RECORD_DTYPE

    def __init__(self, options, executor=None, process_group=None, device=0, context=None):
        """`context` (scan_matching.MultiGpuContext): the library's own NCCL communicator;
        when given, the single all-gather runs inside libcsm_b200.so (csm_ctx_allgather ->
        ncclAllGather) and no torch.distributed group is needed."""
        super().__init__(options,
                         executor if executor is not None else CudaExecutor(options, device),
                         process_group, device, context)

    def _is_device(self, submap):
        """_is_device_grid against the executor's device: ValueError for a TSDF handle or one
        on another device."""
        return _is_device_grid(submap.grid, getattr(self.executor, "device", self.device))

    def MaybeAddConstraint(self, submap_id, submap, node_id, constant_data,
                           initial_relative_pose):
        """constraint_builder_2d.cc:77-112.  constant_data is the node's
        filtered_gravity_aligned_point_cloud (N x 3 float32)."""
        self._check_submap(submap)
        if math.hypot(initial_relative_pose[0], initial_relative_pose[1]) > \
                self.options.max_constraint_distance:
            return
        if not self._pulse(submap_id):
            return
        key = self._register(submap_id, submap, constant_data)
        initial_pose = _compose(tuple(submap.local_pose), tuple(initial_relative_pose))  # :196-197
        self._jobs.append(_Job(submap_id, node_id, key, initial_pose, False,
                               self.options.min_score))

    def MaybeAddGlobalConstraint(self, submap_id, submap, node_id, constant_data):
        """constraint_builder_2d.cc:114-137."""
        self._check_submap(submap)
        key = self._register(submap_id, submap, constant_data)
        self._jobs.append(_Job(submap_id, node_id, key, (0.0, 0.0, 0.0), True,
                               self.options.global_localization_min_score))

    def _fill(self, rec, job, result):
        found, score, pose = result
        rec["found"] = int(found)
        if found:
            rec["score"] = score
            # constraint_transform = ComputeSubmapPose(submap)^-1 * pose_estimate (:251-252)
            rec["pose"] = _compose(_inverse(tuple(self._submaps[job.submap_id].local_pose)), pose)


# ===========================================================================
# ConstraintBuilder3D (mapping/internal/constraints/constraint_builder_3d.{h,cc})
# ===========================================================================
RECORD3D_DTYPE = np.dtype([("submap_trajectory", "<i4"), ("submap_index", "<i4"),
                           ("node_trajectory", "<i4"), ("node_index", "<i4"),
                           ("found", "<u4"), ("score", "<f4"), ("pose", "<f8", (7,)),
                           ("rotational_score", "<f4"), ("low_resolution_score", "<f4"),
                           ("pad", "<u4", (2,))], align=True)
assert RECORD3D_DTYPE.itemsize == 96


@dataclass
class ConstraintBuilderOptions3D:
    """constraint_builder_options.proto + fast_correlative_scan_matcher_options_3d;
    defaults from configuration_files/pose_graph.lua:18-48."""
    sampling_ratio: float = 0.3
    max_constraint_distance: float = 15.0
    min_score: float = 0.55
    global_localization_min_score: float = 0.6
    loop_closure_translation_weight: float = 1.1e4
    loop_closure_rotation_weight: float = 1e5
    branch_and_bound_depth: int = 8
    full_resolution_depth: int = 3
    min_rotational_score: float = 0.77
    min_low_resolution_score: float = 0.55
    linear_xy_search_window: float = 5.0
    linear_z_search_window: float = 1.0
    angular_search_window: float = math.radians(15.0)
    # scan_matching.CeresScanMatcherOptions3D, or None to leave matches unrefined
    ceres_scan_matcher_options_3d: object = None


@dataclass
class Submap3D:
    """What the builder needs of a Submap3D (constraint_builder_3d.cc:172-198):
    high / low resolution hybrid grids and the rotational scan matcher histogram.

    The two grids are either host records (.resolution, .indices, .values) or, for a submap
    kept on the device as RangeDataInserter3D fills it, two scan_matching.DeviceHybridGrids.
    A device submap's matcher and refinement read its grids where they are; the caller keeps
    them alive until WhenDone has run its callback."""
    high_resolution_hybrid_grid: object
    low_resolution_hybrid_grid: object
    rotational_scan_matcher_histogram: object
    grid_size_in_voxels: int = 0


def _is_device_submap(submap):
    """True for a Submap3D whose two grids are DeviceHybridGrids, False for host grids;
    ValueError for one of each."""
    from .scan_matching import DeviceHybridGrid
    on_device = [isinstance(g, DeviceHybridGrid)
                 for g in (submap.high_resolution_hybrid_grid, submap.low_resolution_hybrid_grid)]
    if on_device[0] != on_device[1]:
        raise ValueError("Submap3D: both grids must be DeviceHybridGrids, or neither")
    return on_device[0]


@dataclass
class _Job3:
    submap_id: tuple
    node_id: tuple
    node_key: int
    node_pose: tuple
    submap_pose: tuple
    full: bool
    min_score: float


class CudaExecutor3D:
    """One csm_matcher3d per submap (DispatchScanMatcherConstruction,
    constraint_builder_3d.cc:172-198); jobs run through csm_match3d_batch.  A device
    submap's matcher is built from its DeviceHybridGrids without a host copy, and its
    refinement reads them directly."""

    def __init__(self, options, device=0, threads=8):
        from . import scan_matching as sm
        self.sm = sm
        self.options = options
        self.device = device
        self.threads = threads
        self.matchers = {}
        # submap id -> (high, low) DeviceHybridGrid uploaded for the refinement (host submaps)
        self.grids = {}
        self.stats = {"candidates_scored": 0, "device_ms": 0.0, "searched": 0, "refined": 0,
                      "refine_device_ms": 0.0}

    def delete_matcher(self, submap_id):
        m = self.matchers.pop(submap_id, None)
        if m is not None:
            m.close()
        for g in self.grids.pop(submap_id, ()):
            g.close()

    def refine(self, jobs, submaps, nodes, out):
        """constraint_builder_3d.cc:265-275 for every found match of the drain, one launch."""
        sm = self.sm
        idx = [i for i, r in enumerate(out) if r is not None]
        if not idx:
            return out
        pairs = []
        for i in idx:
            sid = jobs[i].submap_id
            sub = submaps[sid]
            if _is_device_submap(sub):
                hi, lo = sub.high_resolution_hybrid_grid, sub.low_resolution_hybrid_grid
            else:
                if sid not in self.grids:
                    self.grids[sid] = (
                        sm.DeviceHybridGrid(sub.high_resolution_hybrid_grid, self.device),
                        sm.DeviceHybridGrid(sub.low_resolution_hybrid_grid, self.device))
                hi, lo = self.grids[sid]
            node = nodes[jobs[i].node_key]
            pairs.append([(node.high_resolution_point_cloud, hi),
                          (node.low_resolution_point_cloud, lo)])
        matcher = sm.CeresScanMatcher3D(self.options.ceres_scan_matcher_options_3d)
        poses, _ = matcher.MatchBatch([out[i]["pose_estimate"][:3] for i in idx],
                                      [out[i]["pose_estimate"] for i in idx], pairs)
        self.stats["refined"] += len(idx)
        self.stats["refine_device_ms"] += matcher.last_stats["device_ms"]
        out = list(out)
        for i, p in zip(idx, poses):
            out[i] = dict(out[i], pose_estimate=np.array(p, np.float64))
        return out

    def run(self, jobs, submaps, nodes):
        """Matchers are built first (one per submap, like the reference's creation
        tasks); the whole queue then goes to the library in one call."""
        sm, o = self.sm, self.options
        for j in jobs:
            if j.submap_id not in self.matchers:
                sub = submaps[j.submap_id]
                fo = sm.FastCorrelativeScanMatcherOptions3D(
                    o.branch_and_bound_depth, o.full_resolution_depth, o.min_rotational_score,
                    o.min_low_resolution_score, o.linear_xy_search_window,
                    o.linear_z_search_window, o.angular_search_window)
                if _is_device_submap(sub):
                    m = sm.FastCorrelativeScanMatcher3D.from_device_grids(
                        sub.high_resolution_hybrid_grid, sub.low_resolution_hybrid_grid,
                        sub.rotational_scan_matcher_histogram, fo,
                        grid_size_in_voxels=sub.grid_size_in_voxels)
                else:
                    m = sm.FastCorrelativeScanMatcher3D(
                        sub.high_resolution_hybrid_grid, sub.low_resolution_hybrid_grid,
                        sub.rotational_scan_matcher_histogram, fo, device=self.device,
                        grid_size_in_voxels=sub.grid_size_in_voxels)
                self.matchers[j.submap_id] = m

        # one csm_match3d_batch call: the library keeps `threads` matches in flight on
        # separate CUDA streams (the reference's pool threads call Match concurrently
        # too, constraint_builder_3d.cc:104-113)
        sub_ids = sorted({j.submap_id for j in jobs})
        node_keys = sorted({j.node_key for j in jobs})
        sub_index = {k: i for i, k in enumerate(sub_ids)}
        node_index = {k: i for i, k in enumerate(node_keys)}
        out, st = sm.match_batch3d(
            [self.matchers[k] for k in sub_ids], [nodes[k] for k in node_keys],
            [(sub_index[j.submap_id], node_index[j.node_key], j.full, j.node_pose,
              j.submap_pose, j.min_score) for j in jobs],
            max_concurrency=self.threads)
        self.stats["candidates_scored"] += st["candidates_scored"]
        self.stats["device_ms"] += st["device_ms"]
        self.stats["searched"] += len(jobs)
        if self.options.ceres_scan_matcher_options_3d is not None:
            out = self.refine(jobs, submaps, nodes, out)
        return out


class ConstraintBuilder3D(_ConstraintQueue):
    """constraint_builder_3d.h:59-114 over the 3D engine; same sharding / single
    all_gather scheme as ConstraintBuilder2D.  Constraint poses are the fast
    matcher's pose_estimate (submap <- node); with
    ConstraintBuilderOptions3D.ceres_scan_matcher_options_3d set they are first refined as
    constraint_builder_3d.cc:265-275 does (one csm_ceres_match3d_batch launch per drain)."""

    RECORD = RECORD3D_DTYPE

    def __init__(self, options, executor=None, process_group=None, device=0):
        super().__init__(options,
                         executor if executor is not None else CudaExecutor3D(options, device),
                         process_group, device)

    def _is_device(self, submap):
        return _is_device_submap(submap)

    def MaybeAddConstraint(self, submap_id, submap, node_id, constant_data, global_node_pose,
                           global_submap_pose):
        """constraint_builder_3d.cc:79-114; poses are [tx,ty,tz,qw,qx,qy,qz]."""
        self._check_submap(submap)
        d = np.asarray(global_node_pose[:3], float) - np.asarray(global_submap_pose[:3], float)
        if float(np.sqrt((d * d).sum())) > self.options.max_constraint_distance:
            return
        if not self._pulse(submap_id):
            return
        key = self._register(submap_id, submap, constant_data)
        self._jobs.append(_Job3(submap_id, node_id, key, tuple(global_node_pose),
                                tuple(global_submap_pose), False, self.options.min_score))

    def MaybeAddGlobalConstraint(self, submap_id, submap, node_id, constant_data,
                                 global_node_rotation, global_submap_rotation):
        """constraint_builder_3d.cc:116-142; rotations are [qw,qx,qy,qz]."""
        self._check_submap(submap)
        key = self._register(submap_id, submap, constant_data)
        self._jobs.append(_Job3(submap_id, node_id, key, (0, 0, 0) + tuple(global_node_rotation),
                                (0, 0, 0) + tuple(global_submap_rotation), True,
                                self.options.global_localization_min_score))

    def _fill(self, rec, job, result):
        if result is not None:
            rec["found"] = 1
            rec["score"] = result["score"]
            rec["pose"] = result["pose_estimate"]
            rec["rotational_score"] = result["rotational_score"]
            rec["low_resolution_score"] = result["low_resolution_score"]
