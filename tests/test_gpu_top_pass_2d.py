"""The lowest-resolution pass of the 2D fast matcher (csm_score_top2d) in every form.

The host picks the form from a-priori sizes of the batch (RunBatch2D):
  small   if small_lanes = ceil(cap_x / 4) * cap_y <= 32,
  gather  else if max_cap = cap_x * cap_y < 128,
  tile<K> else if tile_words = dec_jd * dec_ids / 4 + 1 <= 128 (K = ceil(tile_words / 32))
          and lat_ints = ceil(cap_x / 4) * 4 * cap_y ints per warp fit 96 KB,
  dense   otherwise.
With a linear window wider than the map, the a-priori lattice per axis is
cap = (cells - 1 + 2 e) // 2^(depth-1) + 1 with e = ceil(max_norm / resolution) + 4, so
the grid size and one far point of the cloud place a case on either side of each
threshold.  Every case compares every lowest-resolution sum of every scan, bit for bit,
with the oracle's ScoreCandidates at depth - 1, for the auto choice and every forced form
that can serve the shape (the others must return CSM_E_INVALID), and checks through
csm_profile_read that the intended kernel ran.
"""
import math
import os
import subprocess
import sys

import numpy as np
import pytest

from benchmarks import synthetic

pytestmark = pytest.mark.gpu

RES = 0.05
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KERNEL = {"small": "k_score_top_small", "gather": "k_score_top_gather",
          "tile": "k_score_top_tile", "dense": "k_score_top_dense"}


@pytest.fixture(scope="module")
def sm():
    from cartographer_b200 import scan_matching
    return scan_matching


def selection(nx, ny, depth, e, lin_cells=10 ** 9, c=(0, 0)):
    """The host's a-priori sizes and its choice (RunBatch2D's lowest-resolution pass);
    c = cell of the sensor origin (index x, index y)."""
    s = 1 << (depth - 1)

    def span(cells, c):
        return min(lin_cells, max(0, cells - 1 - (c - e))) + min(lin_cells, max(0, c + e))

    cx, cy = (span(nx, c[0]) + s) // s, (span(ny, c[1]) + s) // s
    dec_id, dec_jd = -(-(nx + s - 1) // s), -(-(ny + s - 1) // s)
    tile_words = dec_jd * ((dec_id + 6) // 4) + 1
    small_lanes = -(-cx // 4) * cy
    lat_ints = -(-cx // 4) * 4 * cy
    tile_ok = cx * cy >= 128 and tile_words <= 128 and lat_ints * 4 * 4 <= 96 * 1024
    auto = ("small" if small_lanes <= 32 else "gather" if cx * cy < 128 else
            "tile" if tile_ok else "dense")
    return dict(cap=(cx, cy), small_lanes=small_lanes, max_cap=cx * cy, tile_words=tile_words,
                lat_ints=lat_ints, auto=auto, small_ok=small_lanes <= 32, tile_ok=tile_ok,
                tile_k=min(4, -(-tile_words // 32)))


def cloud(rng, n, radius_cells, far_cells=None):
    """n points within +-radius cells; with far_cells, the last point lies at (far - 0.5)
    cells so that e = far + 4."""
    xy = rng.uniform(-radius_cells, radius_cells, (n, 2)) * RES
    if far_cells is not None:
        xy[-1] = ((far_cells - 0.5) * RES * 0.6, (far_cells - 0.5) * RES * 0.8)
    out = np.concatenate([xy, np.zeros((n, 1))], axis=1).astype(np.float32)
    return out


def e_of(xyz):
    norm = np.sqrt(xyz[:, 0] * xyz[:, 0] + xyz[:, 1] * xyz[:, 1]).astype(np.float32).max()
    return int(math.ceil(float(norm) / RES)) + 4


def profiled(sm, fn):
    from cartographer_b200 import _lib
    import ctypes as C
    lib = _lib.lib()
    lib.csm_profile_enable(1)
    try:
        out = fn()
        buf = C.create_string_buffer(8192)
        lib.csm_profile_read(buf, 8192)
    finally:
        lib.csm_profile_enable(0)
    return out, {ln.split()[0] for ln in buf.value.decode().splitlines() if ln.strip()}


def check_top(oracle, sm, grid, depth, xyz, pose=(0.0, 0.0, 0.0), full=False, lin=None, ang=0.3,
              expect=None, all_scans=True, tile_k=None):
    """Runs auto and every form; compares every sum with the oracle and checks the form
    that ran (and tile_k, the K of k_score_top_tile<K> the case is built for, if given).
    Returns the sums."""
    from cartographer_b200 import _lib
    lin = lin if lin is not None else 4.0 * max(grid.num_x, grid.num_y) * RES + 50.0
    m = sm.FastCorrelativeScanMatcher2D(grid, sm.FastCorrelativeScanMatcherOptions2D(lin, ang, depth))
    og = oracle.Grid2D(grid.cells, grid.resolution, grid.max_x, grid.max_y)
    om = oracle.FastCorrelativeScanMatcher2D(og, lin, ang, depth)
    fe = oracle.frontend2d(og, xyz, pose, full=full, lin=lin, ang=ang)
    ds, bounds = fe["discrete_scans"], fe["bounds"]
    step = 1 << (depth - 1)
    if expect is None:
        if full:
            lin_cells, px, py = 10 ** 9, grid.max_x - 0.5 * RES * grid.num_y, \
                grid.max_y - 0.5 * RES * grid.num_x
        else:
            lin_cells, px, py = math.ceil(lin / RES), pose[0], pose[1]
        c = (math.floor((grid.max_y - py) / RES - 0.5), math.floor((grid.max_x - px) / RES - 0.5))
        expect = selection(grid.num_x, grid.num_y, depth, e_of(xyz), lin_cells, c)
    S = ds.shape[0]
    scans = range(S) if all_scans else sorted(set(np.linspace(0, S - 1, 48).astype(int)))
    want = {}
    for k in scans:
        mnx, mxx, mny, mxy = bounds[k]
        cand = [(k, x, y) for x in range(mnx, mxx + 1, step) for y in range(mny, mxy + 1, step)]
        want[k] = om.score_candidates(depth - 1, ds, np.array(cand, np.int32))[1]
    sel = expect
    results = {}
    try:
        for form in ("auto", "small", "gather", "tile", "dense"):
            ok = {"auto": True, "small": sel["small_ok"], "gather": True,
                  "tile": sel["tile_ok"], "dense": True}[form]
            if not ok:
                with pytest.raises(_lib.CsmError) as err:
                    m.score_top(xyz, pose, full, form)
                assert err.value.status == 1, form
                continue
            (sums, lat, kernel), ran = profiled(sm, lambda: m.score_top(xyz, pose, full, form))
            form_ran = sel["auto"] if form == "auto" else form
            assert KERNEL[form_ran] in ran, (form, ran, sel)
            k = (tile_k or sel["tile_k"]) if form_ran == "tile" else 0
            assert kernel == (form_ran, k), (form, kernel, sel)
            np.testing.assert_array_equal(lat[:, :4], bounds)
            assert (lat[:, 4] == (bounds[:, 1] - bounds[:, 0] + step) // step).all()
            assert (lat[:, 5] == (bounds[:, 3] - bounds[:, 2] + step) // step).all()
            for k in scans:
                np.testing.assert_array_equal(sums[k], want[k], err_msg="%s scan %d" % (form, k))
            results[form] = sums
    finally:
        m.close()
    return results


def centred(cells):
    ny, nx = cells.shape
    return synthetic.GridSpec(cells, RES, 0.5 * ny * RES, 0.5 * nx * RES)


def random_cells(rng, ny, nx, zero=0.2):
    cells = rng.randint(1, 32768, size=(ny, nx)).astype(np.uint16)
    cells[rng.uniform(size=cells.shape) < zero] = 0
    return cells


# (name, nx, ny, depth, far point in cells or None, expected auto form, K of the tile
# form where it can run).  The form and K are the ones the engine must report, so a
# change of the host's selection that moves a case off its threshold fails here.
SHAPES = [
    ("small_lanes_32", 4, 116, 3, None, "small", 2),
    ("small_lanes_33", 4, 120, 3, None, "tile", 2),
    ("max_cap_127", 6, 2010, 5, None, "gather", None),
    ("max_cap_128", 6, 2030, 5, None, "dense", None),
    ("tile_words_32", 1, 121, 3, 36, "tile", 1),
    ("tile_words_33", 8, 61, 3, 36, "tile", 2),
    ("tile_words_64", 25, 81, 3, 36, "tile", 2),
    ("tile_words_65", 8, 125, 3, 36, "tile", 3),
    ("tile_words_96", 57, 73, 3, 36, "tile", 3),
    ("tile_words_97", 25, 125, 3, 36, "tile", 4),
    ("tile_words_128", 1, 505, 3, 36, "tile", 4),
    ("tile_words_129", 8, 253, 3, 36, "dense", None),
    ("lat_ints_6144", 8, 520, 5, 500, "tile", 3),
    ("lat_ints_6208", 8, 536, 5, 500, "dense", None),
]


@pytest.mark.parametrize("name,nx,ny,depth,far,auto,tile_k", SHAPES, ids=[s[0] for s in SHAPES])
def test_selection_thresholds(oracle, sm, name, nx, ny, depth, far, auto, tile_k):
    rng = np.random.RandomState(len(name) * 100 + nx + ny)
    xyz = cloud(rng, 300, 0.45, far)
    e = e_of(xyz)
    sel = selection(nx, ny, depth, e)
    assert sel["auto"] == auto, (name, sel)
    value = {"small_lanes": sel["small_lanes"], "max_cap": sel["max_cap"],
             "tile_words": sel["tile_words"], "lat_ints": sel["lat_ints"]}
    key, _, target = name.rpartition("_")
    assert value[key] == int(target), (name, sel)
    assert sel["tile_ok"] == (tile_k is not None), (name, sel)
    check_top(oracle, sm, centred(random_cells(rng, ny, nx)), depth, xyz,
              ang=0.004 if far == 500 else 0.5, expect=sel, tile_k=tile_k)


def test_config2_full_submap_tile3(oracle, sm):
    """Config 2: 1000 x 1000 @ 5 cm, depth 7, a 1081-beam scan, MatchFullSubmap (tile<3>).
    All forms agree on every scan; the oracle checks every slot of 48 scans."""
    grid, occ = synthetic.make_grid2d(0, 1000)
    rng = np.random.RandomState(1)
    pose = synthetic.random_free_pose(occ, grid, rng)
    scan = synthetic.cast_scan(occ, grid, pose, seed=1)
    sel = selection(1000, 1000, 7, e_of(scan))
    assert sel["auto"] == "tile" and sel["tile_k"] == 3, sel
    res = check_top(oracle, sm, grid, 7, scan, full=True, expect=sel, all_scans=False, tile_k=3)
    for form in ("gather", "dense", "auto"):
        for a, b in zip(res["tile"], res[form]):
            np.testing.assert_array_equal(a, b)


@pytest.mark.parametrize("where", ["partly", "wholly"])
def test_scans_outside_the_map(oracle, sm, where):
    rng = np.random.RandomState(7)
    grid = centred(random_cells(rng, 70, 50))
    xyz = cloud(rng, 500, 60)
    pose = (0.0, 0.0, 0.0) if where == "partly" else (40.0, -35.0, 0.3)
    check_top(oracle, sm, grid, 4, xyz, pose=pose, lin=1.5, ang=0.2)
    check_top(oracle, sm, grid, 4, xyz, pose=pose, full=True)


@pytest.mark.parametrize("n", [257, 1081])
def test_saturated_grid(oracle, sm, n):
    """Every cell at the highest probability, and every point in one coarse cell: the
    packed u16 sums of every form reach 255 per point for runs longer than 256 points."""
    cells = np.ones((150, 140), np.uint16)
    assert (oracle.precompute_grid2d(cells, synthetic.K_MIN_COST, synthetic.K_MAX_COST, 1) == 255).all()
    rng = np.random.RandomState(n)
    grid = centred(cells)
    for xyz in (cloud(rng, n, 6), np.tile(cloud(rng, 1, 0.2), (n, 1))):
        check_top(oracle, sm, grid, 4, xyz, lin=1.0, ang=0.2)
        check_top(oracle, sm, grid, 3, xyz, full=True)


@pytest.mark.parametrize("depth", [1, 2])
def test_shallow_stacks(oracle, sm, depth):
    rng = np.random.RandomState(depth)
    grid = centred(random_cells(rng, 40, 45))
    xyz = cloud(rng, 150, 15)
    check_top(oracle, sm, grid, depth, xyz, lin=0.5, ang=0.3)
    check_top(oracle, sm, grid, depth, xyz, lin=3.0, ang=0.3)


# Runs pytest in-process with the per-kernel profile on and prints the kernels that ran.
_PROFILED_PYTEST = r"""
import ctypes, sys, pytest
from cartographer_b200 import _lib
lib = _lib.lib()
lib.csm_profile_enable(1)
rc = pytest.main(sys.argv[1:])
buf = ctypes.create_string_buffer(1 << 16)
lib.csm_profile_read(buf, 1 << 16)
print("KERNELS_RAN", " ".join(sorted({ln.split()[0] for ln in buf.value.decode().splitlines()
                                      if ln.strip()})))
sys.exit(rc)
"""


@pytest.mark.parametrize("env", ["CSM_NO_LATTICE=1", "CSM_LAT_UNROLL=4", "CSM_LAT_UNROLL=16"])
def test_parity_cases_under_switches(env):
    """The end-to-end 2D parity cases (8 local-window seeds, 4 full-submap seeds, the
    reference's sparse-cloud ties) with a debug switch set; the switches are read once
    per process, hence the subprocess.  Those cases stay below the lattice kernel's
    frontier threshold (16384 nodes per level chunk), so the config-2 full-submap case
    runs too: it is the one whose frontiers reach k_expand_lattice, and the profile shows
    that the lattice kernel ran under CSM_LAT_UNROLL and not under CSM_NO_LATTICE."""
    k, v = env.split("=")
    cmd = [sys.executable, "-c", _PROFILED_PYTEST, "-q", "-p", "no:cacheprovider",
           os.path.join(ROOT, "tests", "test_gpu_parity_2d.py"),
           os.path.join(ROOT, "tests", "test_gpu_baseline_sizes.py"),
           "-k", "local_window_parity or full_submap_parity or correct_pose_test_on_device or "
                 "test_full_submap_1000x1000_depth7_vs_oracle"]
    out = subprocess.run(cmd, cwd=ROOT, env=dict(os.environ, **{k: v}), capture_output=True,
                         text=True, timeout=1800)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
    assert "14 passed" in out.stdout, out.stdout[-2000:]
    ran = out.stdout.split("KERNELS_RAN", 1)[1].split()
    assert "k_expand" in ran, ran
    assert ("k_expand_lattice" in ran) == (k != "CSM_NO_LATTICE"), ran
