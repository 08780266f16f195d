"""CPU checks of the submap textures (csm_rt_grid2d_to_texture, csm_grid3d_to_texture):
declarations and exports, refusals that need no device, the step table of
ProbabilityToLogOddsInteger over every float it is used on, the restatement against hand-derived
cases for each branch, the gzip member and the message framing."""
import ctypes as C
import gzip
import os
import re
import struct
import zlib

import numpy as np
import pytest

from tests import protowire as pw
from tests import submap_texture_oracle as T

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENTRIES = {
    "csm_rt_grid2d_to_texture":
        r"csm_status csm_rt_grid2d_to_texture\(const csm_rt_grid2d\* grid, const double local_pose\[7\],",
    "csm_grid3d_to_texture":
        r"csm_status csm_grid3d_to_texture\(const csm_grid3d\* grid, const double global_submap_pose\[7\],",
}
IDENTITY = (0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0)
F32 = np.float32


def test_declared_and_exported():
    with open(os.path.join(ROOT, "include", "csm_abi.h")) as f:
        header = f.read()
    from cartographer_b200._lib import lib
    for name, pattern in ENTRIES.items():
        assert re.search(pattern, header), name
        assert hasattr(lib(), name), name


def test_null_arguments_are_refused_without_a_device():
    from cartographer_b200._lib import lib
    pose = np.array(IDENTITY, np.float64)
    pp = pose.ctypes.data_as(C.c_void_p)
    n = C.c_int64(-7)
    for fn in (lib().csm_rt_grid2d_to_texture, lib().csm_grid3d_to_texture):
        assert fn(None, pp, None, C.c_int64(0), C.byref(n)) == 1
        assert fn(None, None, None, C.c_int64(0), C.byref(n)) == 1
        assert n.value == -7


# ---- ProbabilityToLogOddsInteger as a step table ----
def test_step_table_equals_the_direct_function_on_every_float():
    checked, bad, first = T.log_odds_exhaustive()
    lo, hi = (struct.unpack("<I", struct.pack("<f", v))[0] for v in (F32(0.1), F32(0.9)))
    assert checked == hi - lo + 1 > 20_000_000
    assert bad == 0, first


def test_step_table_shape():
    s = T.steps()
    assert (np.diff(s) > 0).all()
    assert s[0] > F32(0.1) and s[-1] <= F32(0.9)
    assert T.log_odds_integer(F32(0.1)) == 1 and T.log_odds_integer(F32(0.9)) == 255
    for k, t in enumerate(s):   # each step is the first float of its value
        below = np.nextafter(t, F32(0))
        assert T.log_odds_integer(t) >= k + 2 > T.log_odds_integer(below)
        assert T.log_odds_from_steps(t) == T.log_odds_integer(t)
        assert T.log_odds_from_steps(below) == T.log_odds_integer(below)


# ---- 3D by hand ----
SCALE = (F32(0.9) - F32(0.1)) / F32(32766)
BIAS = F32(0.1) - SCALE


def prob(v):
    return F32(F32(v) * SCALE + BIAS)


def first_value_at_limit():
    v = 1
    while prob(v) < F32(0.501):
        v += 1
    return v


def pixel_bytes(count, zdiff, psum, pmax):
    """ComputePixelValues for one pixel, in float32 by hand."""
    if F32(zdiff) < F32(3):
        return b"\0\0"
    fs = max(F32(F32(zdiff) - F32(count)), F32(0))
    fsw = F32(F32(0.15) * fs)
    tw = F32(F32(count) + fsw)
    avg = F32(F32(psum + F32(F32(F32(1) - pmax) * fsw)) / tw)
    avg = min(max(avg, F32(0.1)), F32(0.9))
    delta = 128 - T.log_odds_integer(avg)
    alpha = 0 if delta > 0 else -delta
    value = delta if delta > 0 else 0
    return bytes([value, alpha if (value or alpha) else 1])


def column(zs, values, res=0.1):
    idx = np.array([[0, 0, z] for z in zs], np.int32)
    return T.texture3d(idx, values, res, IDENTITY)


@pytest.mark.parametrize("zdiff", [2, 3, 4])
def test_z_difference(zdiff):
    v = 30000
    t = column([0, zdiff], [v, v])
    assert (t["width"], t["height"]) == (1, 1)
    p = prob(v)
    assert t["cells"] == pixel_bytes(2, zdiff, F32(p + p), p)
    assert (t["cells"] == b"\0\0") == (zdiff < 3)


def test_free_space_clamped_at_zero():
    # 5 voxels over z 0..3 in one pixel (two columns merged by rounding would do the same):
    # z_difference 3 - count 4 < 0 gives no free space
    vals = [20000, 25000, 30000, 32000]
    t = column([0, 1, 2, 3], vals)
    ps = [prob(v) for v in vals]
    s = F32(0)
    for p in ps:
        s = F32(s + p)
    assert t["cells"] == pixel_bytes(4, 3, s, max(ps))
    # free space pulls the average down: a sparse column of high values
    t = column([0, 40], [32767, 32767])
    p = prob(32767)
    assert t["cells"] == pixel_bytes(2, 40, F32(p + p), p)


def test_delta_signs_and_the_alpha_one_byte():
    # delta > 0: low average (free space dominates); delta < 0: high average; delta = 0: the
    # value whose pixel average lands on log-odds integer 128, written (0, 1)
    lo = column([0, 200], [16500, 16500])["cells"]
    assert lo[0] > 0 and lo[1] == 0
    hi = column([0, 1, 2, 3], [32767] * 4)["cells"]
    assert hi[0] == 0 and hi[1] > 0
    found = False
    for v in range(first_value_at_limit(), 32768, 7):
        p = prob(v)
        if T.log_odds_integer(F32(F32(F32(p + p) + p) + p) / F32(4)) == 128:
            assert column([0, 1, 2, 3], [v] * 4)["cells"] == b"\0\x01"
            found = True
            break
    assert found


def test_probability_limit_and_its_neighbours():
    v = first_value_at_limit()
    assert prob(v - 1) < F32(0.501) <= prob(v)
    kept = T.texture3d(np.array([[0, 0, 0]], np.int32), [v], 0.1, IDENTITY)
    assert (kept["width"], kept["height"]) == (1, 1)
    dropped = T.texture3d(np.array([[0, 0, 0]], np.int32), [v - 1], 0.1, IDENTITY)
    assert (dropped["width"], dropped["height"], dropped["cells"]) == (2, 2, bytes(8))
    # the empty box's slice pose: INT_MIN * resolution in float, z from the pose
    want = float(F32(-2147483648.0) * F32(0.1))
    assert dropped["slice_pose"][:3] == (want, want, 0.0)


@pytest.mark.parametrize("x,pixel", [(0, 1), (-1, -1), (1, 2), (-2, -2)])
def test_rounding_ties_after_the_transform(x, pixel):
    # resolution 0.5 and a translation of 0.25: the centre x * 0.5 + 0.25 is pixel + 0.5 or
    # pixel - 0.5 exactly, and RoundToInt rounds half away from zero
    pose = (0.25, 0.25, 0.0, 1.0, 0.0, 0.0, 0.0)
    t = T.texture3d(np.array([[x, x, 0]], np.int32), [30000], 0.5, pose)
    assert (t["width"], t["height"]) == (1, 1)
    # slice = pose^-1 * Translation(max * res): max * 0.5 - 0.25
    assert t["slice_pose"][:2] == (pixel * 0.5 - 0.25, pixel * 0.5 - 0.25)
    assert t["slice_pose"][3:] == (1.0, -0.0, -0.0, -0.0)


def test_pixel_layout():
    # pixel (max_x - x) * width + (max_y - y): x runs down the rows, y along them, both reversed
    idx = np.array([[0, 0, 0], [0, 0, 3], [1, 0, 0], [1, 0, 3], [0, 2, 0], [0, 2, 3]], np.int32)
    vals = [30000, 30000, 20000, 20000, 25000, 25000]
    t = T.texture3d(idx, vals, 0.1, IDENTITY)
    assert (t["width"], t["height"]) == (3, 2)
    cells = np.frombuffer(t["cells"], np.uint8).reshape(2, 3, 2)
    px = {v: pixel_bytes(2, 3, F32(prob(v) + prob(v)), prob(v)) for v in (20000, 25000, 30000)}
    assert cells[0, 2].tobytes() == px[20000]   # x = 1 (max), y = 0
    assert cells[1, 2].tobytes() == px[30000]   # x = 0, y = 0
    assert cells[1, 0].tobytes() == px[25000]   # x = 0, y = 2 (max)
    assert cells[0, 0].tobytes() == cells[0, 1].tobytes() == b"\0\0"


# ---- 2D by hand ----
def test_probability_grid_2d_cells_and_crop():
    cost_scale = (F32(0.9) - F32(0.1)) / F32(32766)
    cells = np.zeros((4, 5), np.uint16)
    cells[1, 2], cells[2, 3], cells[3, 2] = 1, 32767, 16384
    t = T.texture2d(cells, 0.05, 1.0, 2.0, (2, 1, 3, 3), IDENTITY)
    assert (t["width"], t["height"]) == (2, 3)
    c = np.frombuffer(t["cells"], np.uint8).reshape(3, 2, 2)

    def want(v):
        p = F32(F32(1) - F32(F32(v) * cost_scale + F32(F32(0.1) - cost_scale)))
        d = 128 - T.log_odds_integer(p)
        return bytes([max(d, 0), 0 if d > 0 else -d]) if d else b"\0\x01"
    assert c[0, 0].tobytes() == want(1) and c[0, 0, 1] > 0        # low cost: dark
    assert c[1, 1].tobytes() == want(32767) and c[1, 1, 0] > 0    # high cost: light
    assert c[2, 0].tobytes() == want(16384)
    assert c[0, 1].tobytes() == b"\0\0"                           # unknown
    # max_x - res * offset.y, max_y - res * offset.x under the identity
    assert t["slice_pose"][:3] == (1.0 - 0.05 * 1, 2.0 - 0.05 * 2, 0.0)
    empty = T.texture2d(np.zeros((3, 3), np.uint16), 0.05, 1.0, 2.0, None, IDENTITY)
    assert (empty["width"], empty["height"], empty["cells"]) == (1, 1, b"\0\0")
    assert empty["slice_pose"][:2] == (1.0, 2.0)


def test_tsdf_2d_cells():
    trunc, max_w = F32(0.3), F32(10.0)
    tsd = np.array([[16384, 1, 32767, 0]], np.uint16)     # ~0, -trunc, +trunc, unknown
    wgt = np.array([[32767, 32767, 16384, 5]], np.uint16)
    t = T.texture2d(tsd, 0.05, 0.0, 0.0, (0, 0, 2, 0), IDENTITY, wgt, trunc, max_w)
    c = np.frombuffer(t["cells"], np.uint8).reshape(3, 2)
    # |tsd| = trunc, full weight: round(1 * (255 - 128)) = 127 -> value 127
    assert tuple(c[1]) == (127, 0)
    assert c[0, 1] > 100 and c[0, 0] == 0                  # near the surface: -128 * w -> alpha
    assert c[2, 0] > 0 and c[2, 1] == 0


# ---- gzip and framing ----
def test_gzip_member():
    rng = np.random.RandomState(1)
    for data in (b"", b"\0\0", bytes(rng.randint(0, 3, 100000, dtype=np.uint8)),
                 bytes(rng.randint(0, 256, 5000, dtype=np.uint8))):
        z = T.library_gzip(data)
        assert z[:10] == T.GZIP_HEADER            # magic, deflate, no flags, mtime 0, XFL 4, OS 255
        assert struct.unpack("<I", z[-8:-4])[0] == zlib.crc32(data) & 0xFFFFFFFF
        assert struct.unpack("<I", z[-4:])[0] == len(data)
        assert gzip.decompress(z) == data
        assert zlib.decompress(z[10:-8], -15) == data
        if T.zlib_version() == zlib.ZLIB_RUNTIME_VERSION:
            assert z == T.gzip_member(data)       # level 1, window 15, memLevel 8, one stream


def test_message_framing_by_hand():
    t = dict(cells=b"\x05\x00\x00\x07", width=2, height=1, resolution=0.05,
             slice_pose=(1.5, 0.0, -0.0, 1.0, 0.0, 0.0, 0.0))
    z = T.gzip_member(t["cells"])
    want = (b"\x0a" + pw.varint(len(z)) + z + b"\x10\x02" + b"\x18\x01" +
            b"\x21" + struct.pack("<d", 0.05) +
            b"\x2a" + pw.varint(2 + 9 + 9 + 2 + 9) +
            b"\x0a\x12" + b"\x09" + struct.pack("<d", 1.5) + b"\x19" + struct.pack("<d", -0.0) +
            b"\x12\x09" + b"\x21" + struct.pack("<d", 1.0))
    assert T.message(t) == want
    back = T.parse(want)
    assert back["cells"] == t["cells"] and back["width"] == 2 and back["height"] == 1
    assert T.same_bits(back["slice_pose"], t["slice_pose"])
    # zero width / height and an all-zero pose: the sub-messages stay, empty
    t0 = dict(t, width=0, height=0, resolution=0.0, slice_pose=(0.0,) * 7)
    assert T.message(t0).endswith(b"\x2a\x04\x0a\x00\x12\x00")
