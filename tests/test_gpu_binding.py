"""The launch convention of the ctypes binding: every entry point that launches work is called through
_lib.launch, which holds each argument, temporaries made in the argument list included, until the call
returns."""
import os
import re

import pytest
import torch

from conftest import ROOT, load_golden


@pytest.mark.gpu
@pytest.mark.parametrize("tag", ["nocrop", "crop"])
def test_splat_boxes_float32_coordinates(tag):
    """float32 projections are converted to float64 in the argument list: the two copies must reach the
    kernel as two buffers, giving the boxes of the same values passed as float64."""
    from deepviewagg_b200.core.multimodal import visibility as V
    g = load_golden("zbuffer_" + tag)
    W, H = [int(v) for v in g["size"]]
    ct, cb = [int(v) for v in g["crop"]]
    x32, y32, d = g["x_proj"].float().cuda(), g["y_proj"].float().cuda(), g["dist"].cuda()
    got = V.splat_boxes(x32, y32, d, None, (W, H), ct, cb, voxel=0.05, k_swell=1.0, d_swell=1000)
    ref = V.splat_boxes(x32.double(), y32.double(), d, None, (W, H), ct, cb, voxel=0.05, k_swell=1.0, d_swell=1000)
    assert torch.equal(got, ref)


@pytest.mark.gpu
def test_fisheye_splat_boxes_float32_coordinates():
    from deepviewagg_b200.core.multimodal import visibility as V
    g = load_golden("camera_kitti360_fisheye")
    W, H = [int(v) for v in g["size"]]
    xyz = g["xyz"][g["proj_idx"]].cuda()
    x32, y32 = g["x_proj"].float().cuda(), g["y_proj"].float().cuda()
    got = V.fisheye_splat_boxes(x32, y32, xyz, g["ext"], g["fish"], (W, H), voxel=0.05)
    ref = V.fisheye_splat_boxes(x32.double(), y32.double(), xyz, g["ext"], g["fish"], (W, H), voxel=0.05)
    assert torch.equal(got, ref)


def test_launches_only_through_lib():
    """No module but _lib.py picks the device or the stream of a launch: a call site that does so passes
    bare pointers, which outlive the temporaries they point into."""
    pkg = os.path.join(ROOT, "deepviewagg_b200")
    found = []
    for dp, _, files in os.walk(pkg):
        for f in files:
            path = os.path.join(dp, f)
            if f.endswith(".py") and path != os.path.join(pkg, "_lib.py"):
                src = open(path).read()
                found += [f"{os.path.relpath(path, ROOT)}: {m.group(0)}"
                          for m in re.finditer(r"stream_ptr\(|torch\.cuda\.device\(", src)]
    assert not found, found
