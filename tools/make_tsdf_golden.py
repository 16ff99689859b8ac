#!/usr/bin/env python3
"""Write tests/golden/tsdf_rgbd_known.npz: the five 16-bit depth frames and camera poses of the reference's RGB-D test
data (examples/testdata/rgbd/{depth/0000[0-4].png, odometry.log}) and the values its UniformTSDFVolume test pins on them
(src/tests/integration/uniform_fsdfvolume.cpp, RealData).

    python tools/make_tsdf_golden.py REFERENCE_ROOT

The PNGs are decoded losslessly with PIL.  The colour JPEGs are not stored: every pinned value used here depends only
on the depth maps, and a JPEG decoder other than the reference's libjpeg would not reproduce its colours.  The poses are
parsed as float32 (the test's sscanf("%f")); the extrinsics are their inverses computed in float64 and rounded to float32.
"""
import os
import sys

import numpy as np
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def read_poses(path):
    rows = [ln.split() for ln in open(path) if ln.strip()]
    poses = []
    for i in range(0, len(rows) - 4, 5):  # one meta line, then four matrix rows
        poses.append(np.array([[float(x) for x in rows[i + 1 + r]] for r in range(4)], np.float32))
    return np.stack(poses)


def main(ref):
    data = os.path.join(ref, "examples", "testdata", "rgbd")
    depth = np.stack([np.asarray(Image.open(os.path.join(data, "depth", "%05d.png" % i)), np.uint16) for i in range(5)])
    poses = read_poses(os.path.join(data, "odometry.log"))[:5]
    extrinsics = np.stack([np.linalg.inv(p.astype(np.float64)).astype(np.float32) for p in poses])
    out = os.path.join(ROOT, "tests", "golden", "tsdf_rgbd_known.npz")
    np.savez_compressed(out, depth=depth, poses=poses, extrinsics=extrinsics,
                        # UniformTSDFVolume(8.0, 200, 0.04, RGB8); CreateFromColorAndDepth(color, depth, 1000, 4.0, false);
                        # PrimeSenseDefault intrinsic
                        setup=np.array([8.0, 200, 0.04, 1000.0, 4.0]),
                        points_count=np.int64(2227), normal_sum=np.array([-161.569098, -95.969433, -1783.167177]),
                        voxel_count=np.int64(4488), voxel_color_sum=np.array([2096.428416] * 3), tolerance=np.float64(0.1))
    print(out, os.path.getsize(out), "bytes")


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    main(sys.argv[1])
