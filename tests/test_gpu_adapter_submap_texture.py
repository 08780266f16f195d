"""The C++ adapter's DeviceHybridGrid::AddToTextureProto and DeviceGrid2D::DrawToSubmapTexture as
Submap3D / Submap2D::ToResponseProto compose them (adapter_selftest.cc, `texture_response*`
RESULT lines), against the CPU restatement applied to the grids the self-test prints beside
them."""
import os
import subprocess

import numpy as np
import pytest

from tests import grid_proto_ref as R
from tests import submap_texture_oracle as T

ADAPTER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                       "cartographer_b200", "adapter")
POSE3D = (0.5, -0.25, 0.125, 0.96592582628906831, 0.0, 0.0, 0.25881904510252074)
POSE2D = (0.5, -0.25, 0.0, 0.96592582628906831, 0.0, 0.0, 0.25881904510252074)


def _assert_texture(msg, want):
    got = T.parse(msg)
    assert got["cells"] == want["cells"]
    assert (got["width"], got["height"]) == (want["width"], want["height"])
    assert T.same_bits(got["slice_pose"], want["slice_pose"])
    assert msg == T.message(want, gzipped=got["gzipped"])


def _texture2d(fields, pose):
    res, max_x, max_y = (float(v) for v in fields[:3])
    nx, ny, empty, mn_x, mn_y, mx_x, mx_y = (int(v) for v in fields[3:10])
    cells = np.array([int(v) for v in fields[10:]], np.uint16)[:nx * ny].reshape(ny, nx)
    box = None if empty else (mn_x, mn_y, mx_x, mx_y)
    return T.texture2d(cells, res, max_x, max_y, box, pose)


@pytest.mark.gpu
def test_adapter_textures_match_the_restatement():
    exe = os.path.join(ADAPTER, "adapter_selftest")
    subprocess.check_call(["make", "-C", ADAPTER, "-s"])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    lines = [ln.split() for ln in out.stdout.splitlines() if ln.startswith("RESULT ")]
    res = {ln[1]: ln[2:] for ln in lines}
    # the response's order: version, high-resolution texture, low-resolution texture
    names = [ln[1] for ln in lines]
    i = names.index("texture_response3d")
    assert names[i + 1:i + 3] == ["texture_response3d_high", "texture_response3d_low"]
    assert res["texture_response3d"] == ["2"]
    box = [int(v) for v in res["insert3d"]]
    lo, dims = np.array(box[:3]), box[3:6]
    vol = np.array(box[6:], np.uint16).reshape(dims[::-1])
    z, y, x = np.nonzero(vol)
    idx, val, _ = R.walk((np.stack([x, y, z], 1) + lo, vol[z, y, x]))
    _assert_texture(bytes.fromhex(res["texture_response3d_high"][0]),
                    T.texture3d(idx, val, 1.0, POSE3D))
    low = T.texture3d(np.zeros((0, 3), np.int32), np.zeros(0, np.uint16), 2.0, POSE3D)
    assert (low["width"], low["height"]) == (2, 2)
    _assert_texture(bytes.fromhex(res["texture_response3d_low"][0]), low)
    _assert_texture(bytes.fromhex(res["texture_response2d_insert"][0]),
                    _texture2d(res["insert2d"], POSE2D))
    _assert_texture(bytes.fromhex(res["texture_response2d_crop"][0]),
                    _texture2d(res["crop2d"], POSE2D))
