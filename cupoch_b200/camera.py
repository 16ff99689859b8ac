"""cupoch.camera mirror: the pinhole camera model as plain data (pinhole_camera_intrinsic.h,
pinhole_camera_parameters.h; pybind camera/camera.cpp), what VoxelGrid.carve_depth_map / carve_silhouette project
through.  Nothing here touches the device."""
import enum

import numpy as np


class PinholeCameraIntrinsicParameters(enum.IntEnum):
    """camera::PinholeCameraIntrinsicParameters (pinhole_camera_intrinsic.h:33-40): the defaults an intrinsic can be
    built from.  Only PrimeSenseDefault (640 x 480, fx = fy = 525, cx = 319.5, cy = 239.5) is provided."""
    PrimeSenseDefault = 0


class PinholeCameraIntrinsic:
    """camera::PinholeCameraIntrinsic: width, height and the 3x3 intrinsic_matrix
    [[fx, 0, cx], [0, fy, cy], [0, 0, 1]] (float32)."""

    def __init__(self, width=-1, height=-1, fx=0.0, fy=0.0, cx=0.0, cy=0.0):
        if isinstance(width, PinholeCameraIntrinsicParameters):  # PrimeSenseDefault
            width, height, fx, fy, cx, cy = 640, 480, 525.0, 525.0, 319.5, 239.5
        self.set_intrinsics(width, height, fx, fy, cx, cy)

    @property
    def intrinsic_matrix(self):
        return self._k

    @intrinsic_matrix.setter
    def intrinsic_matrix(self, k):
        self._k = np.array(k, np.float32).reshape(3, 3)

    def set_intrinsics(self, width, height, fx, fy, cx, cy):
        self.width, self.height = int(width), int(height)
        self._k = np.array([[fx, 0.0, cx], [0.0, fy, cy], [0.0, 0.0, 1.0]], np.float32)

    def get_focal_length(self):
        return float(self._k[0, 0]), float(self._k[1, 1])

    def get_principal_point(self):
        return float(self._k[0, 2]), float(self._k[1, 2])

    def is_valid(self):
        return self.width > 0 and self.height > 0

    def __repr__(self):
        return "camera::PinholeCameraIntrinsic with width = %d and height = %d.\nAccess intrinsics with intrinsic_matrix." % (
            self.width, self.height)


class PinholeCameraParameters:
    """camera::PinholeCameraParameters: intrinsic and the 4x4 world-to-camera extrinsic (float32)."""

    def __init__(self, intrinsic=None, extrinsic=None):
        self.intrinsic = PinholeCameraIntrinsic() if intrinsic is None else intrinsic
        self.extrinsic = np.eye(4, dtype=np.float32) if extrinsic is None else extrinsic

    @property
    def extrinsic(self):
        return self._e

    @extrinsic.setter
    def extrinsic(self, e):
        self._e = np.array(e, np.float32).reshape(4, 4)

    def __repr__(self):
        return "camera::PinholeCameraParameters class.\nAccess its data via intrinsic and extrinsic."
