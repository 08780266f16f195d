"""ConstraintBuilder2D's refusals of device submaps it cannot use, without a device: a TSDF
handle, a handle on another device, and a device submap on a builder sharded over two ranks
(gloo, or a MultiGpuContext).  Each raises ValueError before anything is queued, and nothing
reaches the library.  The device side is tests/test_gpu_cb2d_device_submaps.py."""
import os
import socket

import numpy as np
import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

from cartographer_b200 import constraint_builder as cb


def _no_library(*args, **kwargs):
    raise AssertionError("the library was called")


@pytest.fixture
def sm(monkeypatch):
    from cartographer_b200 import _lib, scan_matching
    monkeypatch.setattr(_lib, "lib", _no_library)
    monkeypatch.setattr(scan_matching, "lib", _no_library)
    return scan_matching


def _handle(sm, device=0, is_tsdf=False):
    """A RealTimeGrid2D as a device submap's grid looks to the builder, without a device."""
    grid = object.__new__(sm.RealTimeGrid2D)
    grid.device, grid.is_tsdf = device, is_tsdf
    return grid


def _options():
    return cb.ConstraintBuilderOptions(sampling_ratio=1.0, max_constraint_distance=10.0)


CLOUD = np.array([[0.1, 0.2, 0.0]], np.float32)


def _assert_refused(builder, submap):
    with pytest.raises(ValueError):
        builder.MaybeAddConstraint((0, 0), submap, (0, 0), CLOUD, (0.0, 0.0, 0.0))
    with pytest.raises(ValueError):
        builder.MaybeAddGlobalConstraint((0, 0), submap, (0, 0), CLOUD)
    # nothing was queued and the sampler did not pulse
    assert builder._jobs == [] and builder._submaps == {} and builder._samplers == {}


@pytest.mark.parametrize("device,is_tsdf", [(0, True), (1, False), (1, True)])
def test_refused_handles(sm, device, is_tsdf):
    b = cb.ConstraintBuilder2D(_options(), device=0)
    _assert_refused(b, cb.Submap2D(_handle(sm, device, is_tsdf)))
    b.NotifyEndOfNode()
    assert b.WhenDone(lambda r: None) == []
    # the executor refuses them on its own too
    with pytest.raises(ValueError):
        b.executor.ensure_matcher((0, 0), _handle(sm, device, is_tsdf))
    assert b.executor.matchers == {}


def test_device_of_the_executor_decides(sm):
    """A builder handed an executor checks the handle against the executor's device."""
    b = cb.ConstraintBuilder2D(_options(), executor=cb.CudaExecutor(_options(), device=1))
    _assert_refused(b, cb.Submap2D(_handle(sm, device=0)))
    b = cb.ConstraintBuilder2D(_options(), executor=cb.CudaExecutor(_options(), device=1))
    b.MaybeAddConstraint((0, 0), cb.Submap2D(_handle(sm, device=1)), (0, 0), CLOUD,
                         (0.0, 0.0, 0.0))
    assert len(b._jobs) == 1   # queued; nothing ran


def test_accepted_handle_is_queued_without_a_device_call(sm):
    b = cb.ConstraintBuilder2D(_options())
    sub = cb.Submap2D(_handle(sm), (0.5, -0.2, 0.1))
    b.MaybeAddConstraint((0, 0), sub, (0, 0), CLOUD, (0.1, 0.0, 0.0))
    b.MaybeAddGlobalConstraint((0, 0), sub, (0, 1), CLOUD)
    assert len(b._jobs) == 2
    assert b._jobs[0].initial_pose == cb._compose((0.5, -0.2, 0.1), (0.1, 0.0, 0.0))
    b._jobs = []   # drop the queue: draining it would need the device


def test_multi_gpu_context_refuses_device_submaps(sm):
    ctx = object.__new__(sm.MultiGpuContext)
    ctx.world_size, ctx.rank, ctx.device = 2, 0, 0
    b = cb.ConstraintBuilder2D(_options(), context=ctx)
    _assert_refused(b, cb.Submap2D(_handle(sm)))


def _worker(rank, world, port, ret):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from cartographer_b200 import _lib, scan_matching as sm
    _lib.lib = sm.lib = _no_library
    b = cb.ConstraintBuilder2D(_options(), process_group=dist.group.WORLD)
    refused = 0
    try:
        b.MaybeAddConstraint((0, rank), cb.Submap2D(_handle(sm)), (0, 0), CLOUD,
                             (0.0, 0.0, 0.0))
    except ValueError:
        refused += 1
    try:
        b.MaybeAddGlobalConstraint((0, rank), cb.Submap2D(_handle(sm)), (0, 0), CLOUD)
    except ValueError:
        refused += 1
    ret[rank] = (refused, len(b._jobs))
    dist.destroy_process_group()


def test_world2_gloo_refuses_device_submaps():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    ret = ctx.Manager().dict()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, ret)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(300)
        assert p.exitcode == 0
    assert ret[0] == (2, 0) and ret[1] == (2, 0)
