"""CPU-side checks of the 2D and 3D sweep-limit hooks (csm_sweep_limits2d,
csm_match2d_batch_limits, csm_dives2d; csm_sweep_limits3d, csm_match3d_batch_limits,
csm_top_queue3d): exported, laid out as the C compiler lays them out, defaulting to the
engines' constants, and refusing every out-of-range limit and null pointer with
CSM_E_INVALID before any device is needed."""
import ctypes as C
import math
import os
import subprocess
import tempfile

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INT32_MAX = 2 ** 31 - 1


@pytest.fixture(scope="module")
def csm():
    from cartographer_b200 import _lib
    if not os.path.exists(_lib.SO_PATH):
        _lib.build()
    return _lib


@pytest.fixture(scope="module")
def sm(csm):
    from cartographer_b200 import scan_matching
    return scan_matching


def test_symbols_exported(csm):
    lib = csm.lib()
    for name in ("csm_sweep_limits2d_default", "csm_match2d_batch_limits", "csm_dives2d"):
        assert hasattr(lib, name), name


def _c_layout(fields, struct="csm_sweep_limits2d"):
    src = ('#include <stdio.h>\n#include <stddef.h>\n#include "include/csm_abi.h"\nint main(){'
           'printf("%%zu\\n", sizeof(%s));' % struct +
           "".join('printf("%%zu\\n", offsetof(%s, %s));' % (struct, f) for f in fields) + "}")
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "lim.c"), "w").write(src)
        subprocess.check_call(["gcc", "-I", ROOT, os.path.join(d, "lim.c"), "-o",
                               os.path.join(d, "lim")])
        return [int(v) for v in subprocess.check_output([os.path.join(d, "lim")]).split()]


def test_struct_layout(sm):
    fields = [f for f, _ in sm.SweepLimits2D._fields_]
    assert fields == ["chunk", "leaf_cap", "inline_best", "lattice_min", "unroll", "dive_ratio",
                      "max_points"]
    got = _c_layout(fields)
    assert got[0] == C.sizeof(sm.SweepLimits2D) == 32
    assert got[1:] == [getattr(sm.SweepLimits2D, f).offset for f in fields]


def test_defaults_are_the_engine_constants(sm, monkeypatch):
    d = sm.SweepLimits2D.default()
    assert d.chunk == 1 << 23
    assert d.leaf_cap == 1 << 22
    assert d.inline_best == 4096
    # CSM_NO_LATTICE / CSM_LAT_UNROLL are read once per process
    assert d.lattice_min == (INT32_MAX if os.environ.get("CSM_NO_LATTICE") else 16384)
    if not os.environ.get("CSM_LAT_UNROLL"):
        assert d.unroll == 8
    assert d.dive_ratio == np.float32(0.97)
    assert d.max_points == 1 << 30


def _batch_args(limits, results=True, stacks=True, stack_index=0):
    # handles are never dereferenced: validation fails first
    hs = (C.c_void_p * 1)(C.c_void_p(0x10))
    cs = (C.c_void_p * 1)(C.c_void_p(0x20))
    from cartographer_b200._lib import JOB2D_DTYPE, RESULT2D_DTYPE
    jobs = np.zeros(1, JOB2D_DTYPE)
    jobs["stack_index"] = stack_index
    res = np.zeros(1, RESULT2D_DTYPE)
    keep = (hs, cs, jobs, res)
    args = (hs if stacks else None, C.c_int32(1), cs, C.c_int32(1),
            jobs.ctypes.data_as(C.c_void_p), C.c_int32(1), C.c_double(1.0), C.c_double(0.3),
            C.byref(limits) if limits is not None else None,
            res.ctypes.data_as(C.c_void_p) if results else None, None, None)
    return args, keep


BAD_LIMITS = [("chunk", 0), ("chunk", (1 << 23) + 1), ("chunk", -5),
              ("leaf_cap", 1), ("leaf_cap", (1 << 22) + 1),
              ("inline_best", -1), ("inline_best", 4097),
              ("lattice_min", 0), ("lattice_min", -1),
              ("unroll", 2), ("unroll", 12), ("unroll", 32),
              ("dive_ratio", -0.5), ("dive_ratio", math.inf), ("dive_ratio", math.nan),
              ("max_points", 0), ("max_points", -1)]


@pytest.mark.parametrize("field,value", BAD_LIMITS)
def test_out_of_range_limit_is_refused(csm, sm, field, value):
    lim = sm.SweepLimits2D.default()
    setattr(lim, field, value)
    args, keep = _batch_args(lim)
    assert csm.lib().csm_match2d_batch_limits(*args) == 1
    assert field.encode() in csm.lib().csm_last_error_string()


@pytest.mark.parametrize("field,value", [("chunk", 1), ("chunk", 1 << 23), ("leaf_cap", 2),
                                         ("inline_best", 0), ("inline_best", 4096),
                                         ("lattice_min", INT32_MAX), ("unroll", 16),
                                         ("dive_ratio", 0.0), ("max_points", 1)])
def test_limits_at_their_ends_pass_validation(csm, sm, field, value):
    """A limit at the end of its range gets past the limit checks, which come before the
    jobs' checks: the call then fails on the job's stack index, not on the limit."""
    lim = sm.SweepLimits2D.default()
    setattr(lim, field, value)
    args, keep = _batch_args(lim, stack_index=5)
    assert csm.lib().csm_match2d_batch_limits(*args) == 1
    assert b"invalid argument: stack index (" in csm.lib().csm_last_error_string()


def test_null_pointers_are_refused(csm, sm):
    lib = csm.lib()
    lim = sm.SweepLimits2D.default()
    for kw in ({"results": False}, {"stacks": False}):
        args, keep = _batch_args(lim, **kw)
        assert lib.csm_match2d_batch_limits(*args) == 1
        assert b"null" in lib.csm_last_error_string()
    # csm_dives2d: every output pointer, and a queue without storage
    xyz = np.zeros((4, 3), np.float32)
    pose = np.zeros(3, np.float64)
    jb, cnt = C.c_int32(), C.c_int32()
    bounds = np.zeros(2, np.float32)
    ctr = np.zeros(2, np.int64)
    q = np.zeros(4, sm.NODE2D_DTYPE)

    def dives(job_best=True, b=True, c=True, queue=True, cap=4, count=True, ratio=0.97,
              initial=True, full=0):
        return lib.csm_dives2d(
            C.c_void_p(0x10), xyz.ctypes.data_as(C.POINTER(C.c_float)), C.c_int32(4),
            pose.ctypes.data_as(C.POINTER(C.c_double)) if initial else None, C.c_int32(full),
            C.c_double(1.0), C.c_double(0.3), C.c_float(0.1), C.c_float(ratio),
            C.byref(jb) if job_best else None,
            bounds.ctypes.data_as(C.POINTER(C.c_float)) if b else None,
            ctr.ctypes.data_as(C.POINTER(C.c_int64)) if c else None,
            q.ctypes.data_as(C.c_void_p) if queue else None, C.c_int32(cap),
            C.byref(cnt) if count else None)

    for kw in ({"job_best": False}, {"b": False}, {"c": False}, {"count": False},
               {"queue": False}, {"cap": -1}, {"ratio": -1.0}, {"ratio": math.nan},
               {"ratio": math.inf}, {"initial": False}):
        assert dives(**kw) == 1, kw
        assert lib.csm_last_error_string(), kw
    # a null stack, with every output present
    st = lib.csm_dives2d(None, xyz.ctypes.data_as(C.POINTER(C.c_float)), C.c_int32(4),
                         pose.ctypes.data_as(C.POINTER(C.c_double)), C.c_int32(0),
                         C.c_double(1.0), C.c_double(0.3), C.c_float(0.1), C.c_float(0.97),
                         C.byref(jb), bounds.ctypes.data_as(C.POINTER(C.c_float)),
                         ctr.ctypes.data_as(C.POINTER(C.c_int64)), None, C.c_int32(0),
                         C.byref(cnt))
    assert st == 1


# ---- 3D: csm_sweep_limits3d, csm_match3d_batch_limits, csm_top_queue3d --------------------
def test_symbols_exported_3d(csm):
    lib = csm.lib()
    for name in ("csm_sweep_limits3d_default", "csm_match3d_batch_limits", "csm_top_queue3d"):
        assert hasattr(lib, name), name


def test_struct_layout_3d(sm):
    fields = [f for f, _ in sm.SweepLimits3D._fields_]
    assert fields == ["chunk", "leaf_cap", "inline_best", "dive_ratio"]
    got = _c_layout(fields, "csm_sweep_limits3d")
    assert got[0] == C.sizeof(sm.SweepLimits3D) == 16
    assert got[1:] == [getattr(sm.SweepLimits3D, f).offset for f in fields]


def test_defaults_are_the_engine_constants_3d(sm):
    d = sm.SweepLimits3D.default()
    assert (d.chunk, d.leaf_cap, d.inline_best) == (1 << 16, 1 << 20, 256)
    assert d.dive_ratio == np.float32(0.97)


def _batch3d_args(sm, limits, matchers=True, nodes=True, jobs=True, results=True,
                  matcher_index=0, num_jobs=1):
    # the matcher handle is never dereferenced: validation fails first
    hs = (C.c_void_p * 1)(C.c_void_p(0x10))
    cloud = np.zeros((4, 3), np.float32)
    nd = (sm.CsmNode3D * 1)()
    nd[0].high_resolution_point_cloud = cloud.ctypes.data_as(C.POINTER(C.c_float))
    nd[0].num_high = 4
    js = (sm.CsmJob3D * 1)()
    js[0].matcher_index = matcher_index
    res = (sm.CsmResult3D * 1)()
    trace = np.zeros(3, np.int32)
    keep = (hs, cloud, nd, js, res, trace)
    args = (hs if matchers else None, C.c_int32(1), nd if nodes else None, C.c_int32(1),
            js if jobs else None, C.c_int32(num_jobs), C.c_int32(0),
            C.byref(limits) if limits is not None else None, res if results else None, None,
            trace.ctypes.data_as(C.POINTER(C.c_int32)))
    return args, keep


BAD_LIMITS_3D = [("chunk", 0), ("chunk", (1 << 16) + 1), ("chunk", -5),
                 ("leaf_cap", 0), ("leaf_cap", (1 << 20) + 1), ("leaf_cap", -1),
                 ("inline_best", -1), ("inline_best", 257),
                 ("dive_ratio", -0.5), ("dive_ratio", math.inf), ("dive_ratio", math.nan)]


@pytest.mark.parametrize("field,value", BAD_LIMITS_3D)
def test_out_of_range_limit_is_refused_3d(csm, sm, field, value):
    """Refused before anything else, even for an empty batch."""
    lim = sm.SweepLimits3D.default()
    setattr(lim, field, value)
    for n in (1, 0):
        args, keep = _batch3d_args(sm, lim, num_jobs=n)
        assert csm.lib().csm_match3d_batch_limits(*args) == 1
        assert field.encode() in csm.lib().csm_last_error_string()


@pytest.mark.parametrize("field,value", [("chunk", 1), ("chunk", 1 << 16), ("leaf_cap", 1),
                                         ("leaf_cap", 1 << 20), ("inline_best", 0),
                                         ("inline_best", 256), ("dive_ratio", 0.0),
                                         ("dive_ratio", 1e30)])
def test_limits_at_their_ends_pass_validation_3d(csm, sm, field, value):
    """A limit at the end of its range gets past the limit checks, which come before the
    jobs' checks: the call then fails on the job's matcher index, not on the limit.  An
    empty batch under the same limits succeeds and leaves a zero trace."""
    lim = sm.SweepLimits3D.default()
    setattr(lim, field, value)
    args, keep = _batch3d_args(sm, lim, matcher_index=5)
    assert csm.lib().csm_match3d_batch_limits(*args) == 1
    assert b"matcher_index out of range" in csm.lib().csm_last_error_string()
    args, keep = _batch3d_args(sm, lim, num_jobs=0)
    keep[-1][:] = 7
    assert csm.lib().csm_match3d_batch_limits(*args) == 0
    assert list(keep[-1]) == [0, 0, 0]


def test_null_pointers_are_refused_3d(csm, sm):
    lib = csm.lib()
    lim = sm.SweepLimits3D.default()
    for kw in ({"matchers": False}, {"nodes": False}, {"jobs": False}, {"results": False}):
        args, keep = _batch3d_args(sm, lim, **kw)
        assert lib.csm_match3d_batch_limits(*args) == 1, kw
        assert b"null" in lib.csm_last_error_string(), kw
    # csm_top_queue3d: every output pointer, a queue without storage and the dive ratio are
    # checked before the handle is used
    cloud = np.zeros((4, 3), np.float32)
    nd = sm.CsmNode3D()
    nd.high_resolution_point_cloud = cloud.ctypes.data_as(C.POINTER(C.c_float))
    nd.num_high = 4
    pose = np.array([0, 0, 0, 1, 0, 0, 0], np.float64)
    bound, cnt = C.c_float(), C.c_int32()
    q = np.zeros(4, sm.BNB_NODE3D_DTYPE)

    def top_queue(matcher=True, node=True, npose=True, spose=True, b=True, queue=True, cap=4,
                  count=True, ratio=0.97):
        pp = pose.ctypes.data_as(C.POINTER(C.c_double))
        return lib.csm_top_queue3d(
            C.c_void_p(0x10) if matcher else None, C.byref(nd) if node else None,
            pp if npose else None, pp if spose else None, C.c_int32(0), C.c_float(0.1),
            C.c_float(ratio), C.byref(bound) if b else None,
            q.ctypes.data_as(C.c_void_p) if queue else None, C.c_int32(cap),
            C.byref(cnt) if count else None)

    for kw in ({"b": False}, {"count": False}, {"queue": False}, {"cap": -1}, {"ratio": -1.0},
               {"ratio": math.nan}, {"ratio": math.inf}):
        assert top_queue(**kw) == 1, kw
        assert lib.csm_last_error_string(), kw
    # with every output valid, the null inputs (the fake handle is never reached)
    for kw in ({"matcher": False}, {"node": False}, {"npose": False}, {"spose": False}):
        assert top_queue(**kw) == 1, kw
        assert b"null" in lib.csm_last_error_string(), kw
