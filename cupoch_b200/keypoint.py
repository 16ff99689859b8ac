"""cupoch.geometry.keypoint mirror (keypoint.h, pybind geometry/keypoint.cpp): ISS keypoint detection."""
import ctypes as C
import sys

import numpy as np

from . import _lib
from .geometry import NUM_MAX_NN, PointCloud
from .utility import DeviceArray

ISS_MAX_NEIGHBORS = 256  # the radius search's limit (csrc/search.cu CPHB_RADIUS_MAX_NN)


def compute_iss_keypoints(input, salient_radius=0.0, non_max_radius=0.0, gamma_21=0.975, gamma_32=0.975, min_neighbors=5,
                          max_neighbots=NUM_MAX_NN):
    """geometry::keypoint::ComputeISSKeypoints (iss_keypoints.cu:108-172; Yu Zhong, "Intrinsic Shape Signatures", 2009)
    -> (keypoint cloud, device bool mask [n]).  The keypoints are the masked rows in ascending order, with their normals
    and colours.  salient_radius == 0 or non_max_radius == 0 replaces both by 6 and 4 times the cloud's resolution (the
    root-mean-square nearest-neighbour distance); the radii used go to input.last_iss_radii.  The last keyword keeps the
    reference binding's spelling `max_neighbots` (keypoint.cpp:49) so that existing callers work; it must lie in [0, 256].
    An empty cloud, or an illegal max_neighbots, is logged and gives an empty cloud and an empty mask."""
    n, k = len(input), int(max_neighbots)
    if n == 0:
        print("[cupoch_b200][warning] [ComputeISSKeypoints] Input PointCloud is empty!", file=sys.stderr)
        return PointCloud(), DeviceArray((0,), np.bool_)
    if not 0 <= k <= ISS_MAX_NEIGHBORS:
        print("[cupoch_b200][error] [ComputeISSKeypoints] max_neighbors = %d must lie in [0, %d]." % (k, ISS_MAX_NEIGHBORS),
              file=sys.stderr)
        return PointCloud(), DeviceArray((0,), np.bool_)
    mask = DeviceArray((n,), np.bool_)
    d_idx = DeviceArray((n,), np.int32)
    m, radii = C.c_size_t(0), (C.c_float * 2)()
    _lib.check(_lib.lib().cphb_compute_iss_keypoints(
        input.points.ptr, n, float(salient_radius), float(non_max_radius), float(gamma_21), float(gamma_32),
        int(min_neighbors), k, mask.ptr, d_idx.ptr, C.byref(m), None, radii, None))
    input.last_iss_radii = (float(radii[0]), float(radii[1]))
    return input._filtered(d_idx, m.value)[0], mask
