"""The queue both Python ConstraintBuilders share, on CPU with world_size 2 over gloo: the 3D
builder refuses device submaps on a sharded queue before any gate, as the 2D builder does
(tests/test_cb2d_device_submaps_cpu.py), and the `context` transport of the single exchange
(a MultiGpuContext's allgather, here a stand-in over the gloo group) ends with the same Result
and the same records as the process_group transport."""
import os
import socket

import numpy as np
import torch.distributed as dist
import torch.multiprocessing as mp

from cartographer_b200 import constraint_builder as cb
from tests.test_constraint_builder_cpu import OracleExecutor, _fill, _small_queue


def _no_library(*args, **kwargs):
    raise AssertionError("the library was called")


def _run_world2(worker, *args):
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    ret = ctx.Manager().dict()
    procs = [ctx.Process(target=worker, args=(r, 2, port, ret) + args) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(300)
        assert p.exitcode == 0
    return ret


def _init(rank, world, port):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)


def _refusal_worker(rank, world, port, ret):
    _init(rank, world, port)
    from cartographer_b200 import _lib, scan_matching as sm
    _lib.lib = sm.lib = _no_library
    grid = object.__new__(sm.DeviceHybridGrid)
    submap = cb.Submap3D(grid, grid, np.zeros(10, np.float32))
    b = cb.ConstraintBuilder3D(cb.ConstraintBuilderOptions3D(sampling_ratio=1.0,
                                                             max_constraint_distance=10.0),
                               process_group=dist.group.WORLD)
    ident = [0, 0, 0, 1, 0, 0, 0]
    refused = 0
    # a pair the distance gate passes, one it would drop, and a global one
    for node_pose in (ident, [100, 0, 0, 1, 0, 0, 0]):
        try:
            b.MaybeAddConstraint((0, rank), submap, (0, 0), object(), node_pose, ident)
        except ValueError:
            refused += 1
    try:
        b.MaybeAddGlobalConstraint((0, rank), submap, (0, 0), object(), [1, 0, 0, 0],
                                   [1, 0, 0, 0])
    except ValueError:
        refused += 1
    ret[rank] = (refused, len(b._jobs), len(b._submaps), len(b._samplers))
    dist.destroy_process_group()


def test_3d_world2_gloo_refuses_device_submaps_before_gating():
    ret = _run_world2(_refusal_worker)
    # every call refused; nothing queued, and no sampler pulsed
    assert ret[0] == (3, 0, 0, 0) and ret[1] == (3, 0, 0, 0)


class _GlooContext:
    """What the builder reads of a MultiGpuContext: rank, world_size and allgather(bytes) ->
    one byte string per rank, here over the default gloo group."""

    def __init__(self):
        self.rank, self.world_size = dist.get_rank(), dist.get_world_size()

    def allgather(self, payload):
        parts = [None] * self.world_size
        dist.all_gather_object(parts, payload)
        return parts


def _transport_worker(rank, world, port, ret):
    _init(rank, world, port)
    got = {}
    for name, kw in (("context", dict(context=_GlooContext())),
                     ("process_group", dict(process_group=dist.group.WORLD))):
        opts, submaps, clouds, poses = _small_queue()
        ex = OracleExecutor(opts)
        b = cb.ConstraintBuilder2D(opts, executor=ex, **kw)
        _fill(b, submaps, clouds, poses)
        res = b.WhenDone(lambda r: None)
        got[name] = ([(c.submap_id, c.node_id, c.zbar_ij, c.score) for c in res],
                     sorted(ex.touched), b.last_records.tobytes())
    ret[rank] = got
    dist.destroy_process_group()


def test_2d_context_transport_world2_gloo():
    opts, submaps, clouds, poses = _small_queue()
    single = cb.ConstraintBuilder2D(opts, executor=OracleExecutor(opts))
    _fill(single, submaps, clouds, poses)
    want = [(c.submap_id, c.node_id, c.zbar_ij, c.score) for c in single.WhenDone(lambda r: None)]
    assert len(want) > 0
    ret = _run_world2(_transport_worker)
    ctx0, ctx1 = ret[0]["context"], ret[1]["context"]
    assert ctx0[0] == want and ctx1[0] == want          # the single-process Result on both ranks
    assert ctx0[2] == ctx1[2]                           # byte-identical gathered records
    assert ctx0[2] == ret[0]["process_group"][2]        # the same records as the torch transport
    assert set(ctx0[1]).isdisjoint(ctx1[1])             # a stack only on its owner
    assert sorted(ctx0[1] + ctx1[1]) == sorted(submaps.keys())
