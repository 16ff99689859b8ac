"""cupoch.geometry mirror (hot-path subset): PointCloud, the bounding boxes, KDTreeFlann, KDTreeSearchParam*.

Names, argument meaning and error behaviour follow src/python/cupoch_pybind/geometry/
pointcloud.cpp and kdtree_flann.cpp; computation goes through the C ABI only.
"""
import ctypes as C
import enum
import sys

import numpy as np

from . import _lib
from .utility import DeviceArray, Matrix3fVector, Vector3fVector, as_f16

NUM_MAX_NN = 100  # kdtree_search_param.h:26


class KDTreeSearchParam:
    pass


class KDTreeSearchParamKNN(KDTreeSearchParam):
    def __init__(self, knn=30):
        self.knn = int(knn)

    def __repr__(self):
        return "geometry::KDTreeSearchParamKNN with knn = %d" % self.knn


class KDTreeSearchParamRadius(KDTreeSearchParam):
    def __init__(self, radius, max_nn):
        self.radius = float(radius)
        self.max_nn = int(max_nn)

    def __repr__(self):
        return "geometry::KDTreeSearchParamRadius with radius = %f, max_nn = %d" % (self.radius, self.max_nn)


class PointCloud:
    """geometry::PointCloud (pointcloud.h:43-263): points_/normals_/colors_/covariances_ on the device."""

    def __init__(self, points=None):
        self._points = self._normals = self._colors = self._covariances = None
        self._color_gradient = None  # PointCloudForColoredICP (colored_icp.cu:36-40)
        if points is not None:
            self.points = points

    points = property(lambda s: s._points, lambda s, v: setattr(s, "_points", Vector3fVector(v)))
    normals = property(lambda s: s._normals, lambda s, v: setattr(s, "_normals", Vector3fVector(v)))
    colors = property(lambda s: s._colors, lambda s, v: setattr(s, "_colors", Vector3fVector(v)))
    covariances = property(lambda s: s._covariances, lambda s, v: setattr(s, "_covariances", Matrix3fVector(v)))

    def __len__(self):
        return 0 if self._points is None else len(self._points)

    def is_empty(self):
        return len(self) == 0

    # pointcloud.h:82-94: "non-empty and same length as points"
    def has_points(self):
        return len(self) > 0

    def _has(self, a):
        return len(self) > 0 and a is not None and len(a) == len(self)

    def has_normals(self):
        return self._has(self._normals)

    def has_colors(self):
        return self._has(self._colors)

    def has_covariances(self):
        return self._has(self._covariances)

    def _cloud(self, with_attrs=True):
        c = _lib.Cloud()
        c.points = self._points.ptr if self._points is not None else None
        c.n = len(self)
        if with_attrs:
            c.normals = self._normals.ptr if self.has_normals() else None
            c.colors = self._colors.ptr if self.has_colors() else None
            c.covariances = self._covariances.ptr if self.has_covariances() else None
            c.color_gradient = self._color_gradient.ptr if self._has(self._color_gradient) else None
        c.cov_col_major = 0
        return c

    # -- DLPack exchange (pointcloud.cpp:82-105, utility/dl_converter.h:32-40; examples/python/basic/*torch_tensor.py) --
    def _to_dlpack(self, arr):
        import torch
        from torch.utils.dlpack import to_dlpack
        if arr is None:
            raise ValueError("attribute is empty")
        return to_dlpack(torch.as_tensor(arr, device="cuda"))   # zero-copy view of the device array

    def _from_dlpack(self, capsule):
        from torch.utils.dlpack import from_dlpack
        t = from_dlpack(capsule)
        if not t.is_cuda:
            t = t.cuda()
        return DeviceArray.borrow(t.contiguous().float())

    def to_points_dlpack(self):
        return self._to_dlpack(self._points)

    def to_normals_dlpack(self):
        return self._to_dlpack(self._normals)

    def to_colors_dlpack(self):
        return self._to_dlpack(self._colors)

    def from_points_dlpack(self, capsule):
        self._points = self._from_dlpack(capsule)

    def from_normals_dlpack(self, capsule):
        self._normals = self._from_dlpack(capsule)

    def from_colors_dlpack(self, capsule):
        self._colors = self._from_dlpack(capsule)

    def clone(self):
        """deep copy (the reference's copy constructor, pointcloud.cu:150-155: all attribute vectors are copied)"""
        out = PointCloud()
        for name in ("_points", "_normals", "_colors", "_covariances", "_color_gradient"):
            a = getattr(self, name)
            if a is None:
                continue
            b = DeviceArray(a.shape, a.dtype)
            if a.nbytes:
                _lib.check(_lib.lib().cphb_memcpy_d2d(b.ptr, a.ptr, a.nbytes, None))
            setattr(out, name, b)
        return out

    # -- geometry ops ---------------------------------------------------------
    def transform(self, transformation):
        """PointCloud::Transform (pointcloud.cu:293-299), in place."""
        if len(self):
            _lib.check(_lib.lib().cphb_transform(
                self._points.ptr, self._normals.ptr if self.has_normals() else None,
                self._covariances.ptr if self.has_covariances() else None, 0, len(self), as_f16(transformation), None))
        return self

    def get_min_bound(self):
        return self._bounds()[0]

    def get_max_bound(self):
        return self._bounds()[1]

    def _bounds(self):
        mn, mx = (C.c_float * 3)(), (C.c_float * 3)()
        if len(self):
            _lib.check(_lib.lib().cphb_min_max_bound(self._points.ptr, len(self), mn, mx, None))
        return np.array(mn, np.float32), np.array(mx, np.float32)

    def voxel_down_sample(self, voxel_size):
        """PointCloud::VoxelDownSample (down_sample.cu:170-273)."""
        out = PointCloud()
        n = len(self)
        if n == 0:
            return out
        hn, hc = self.has_normals(), self.has_colors()
        op = DeviceArray((n, 3), np.float32)
        on = DeviceArray((n, 3), np.float32) if hn else None
        oc = DeviceArray((n, 3), np.float32) if hc else None
        m = C.c_size_t(0)
        _lib.check(_lib.lib().cphb_voxel_down_sample(
            self._points.ptr, self._normals.ptr if hn else None, self._colors.ptr if hc else None, n,
            float(voxel_size), op.ptr, on.ptr if hn else None, oc.ptr if hc else None, C.byref(m), None))
        m = m.value

        def cut(a):
            return None if a is None else DeviceArray((m, 3), np.float32, ptr=a.ptr, base=a)
        out._points, out._normals, out._colors = cut(op), cut(on), cut(oc)
        return out

    def select_by_index(self, indices, invert=False):
        """PointCloud::SelectByIndex (down_sample.cu:110-127): rows named by `indices` (host or device int array),
        in the order given; invert=True selects the complement in ascending order (sort + set_difference there,
        a host-side mask here)."""
        out = PointCloud()
        n = len(self)
        idx = indices.cpu() if hasattr(indices, "cpu") else np.asarray(indices)
        idx = np.ascontiguousarray(idx, np.int64).reshape(-1)
        if invert:
            mask = np.ones(n, bool)
            mask[idx[(idx >= 0) & (idx < n)]] = False
            idx = np.flatnonzero(mask)
        m = len(idx)
        if m == 0 or n == 0:
            return out
        d_idx = DeviceArray.from_numpy(idx.astype(np.int32), np.int32)
        hn, hc = self.has_normals(), self.has_colors()
        op = DeviceArray((m, 3), np.float32)
        on = DeviceArray((m, 3), np.float32) if hn else None
        oc = DeviceArray((m, 3), np.float32) if hc else None
        _lib.check(_lib.lib().cphb_select_by_index(
            self._points.ptr, self._normals.ptr if hn else None, self._colors.ptr if hc else None, n, d_idx.ptr, m,
            op.ptr, on.ptr if hn else None, oc.ptr if hc else None, None))
        _lib.check(_lib.lib().cphb_stream_synchronize(None))
        out._points, out._normals, out._colors = op, on, oc
        return out

    def _filtered(self, d_idx, m):
        """(selected cloud, device index vector) from the first m entries of a device index buffer"""
        kept = DeviceArray((m,), np.int32, ptr=d_idx.ptr, base=d_idx)
        out = PointCloud()
        n = len(self)
        if m:
            hn, hc = self.has_normals(), self.has_colors()
            op = DeviceArray((m, 3), np.float32)
            on = DeviceArray((m, 3), np.float32) if hn else None
            oc = DeviceArray((m, 3), np.float32) if hc else None
            _lib.check(_lib.lib().cphb_select_by_index(
                self._points.ptr, self._normals.ptr if hn else None, self._colors.ptr if hc else None, n, kept.ptr, m,
                op.ptr, on.ptr if hn else None, oc.ptr if hc else None, None))
            _lib.check(_lib.lib().cphb_stream_synchronize(None))
            out._points, out._normals, out._colors = op, on, oc
        return out, kept

    def remove_radius_outlier(self, nb_points, radius):
        """PointCloud::RemoveRadiusOutliers (down_sample.cu:317-354; bound as remove_radius_outlier,
        pointcloud.cpp:190-203) -> (filtered cloud, kept indices on the device, ascending)."""
        n = len(self)
        if n == 0:
            return PointCloud(), DeviceArray((0,), np.int32)
        d_idx = DeviceArray((n,), np.int32)
        m = C.c_size_t(0)
        _lib.check(_lib.lib().cphb_remove_radius_outliers(self._points.ptr, n, int(nb_points), float(radius), d_idx.ptr,
                                                          C.byref(m), None))
        return self._filtered(d_idx, m.value)

    def remove_statistical_outlier(self, nb_neighbors, std_ratio):
        """PointCloud::RemoveStatisticalOutliers (down_sample.cu:356-438; bound as remove_statistical_outlier,
        pointcloud.cpp:204-217) -> (filtered cloud, kept indices on the device, ascending)."""
        n = len(self)
        if n == 0:
            return PointCloud(), DeviceArray((0,), np.int32)
        d_idx = DeviceArray((n,), np.int32)
        m = C.c_size_t(0)
        stats = (C.c_float * 3)()
        _lib.check(_lib.lib().cphb_remove_statistical_outliers(self._points.ptr, n, int(nb_neighbors), float(std_ratio),
                                                               d_idx.ptr, C.byref(m), stats, None))
        self.last_outlier_stats = tuple(float(x) for x in stats)  # (cloud mean, std, threshold): diagnostics
        return self._filtered(d_idx, m.value)

    def segment_plane(self, distance_threshold=0.01, ransac_n=3, num_iterations=100):
        """PointCloud::SegmentPlane (segmentation.cu:187-267; bound as segment_plane, pointcloud.cpp) ->
        (plane float32[4] = [a, b, c, d], inlier indices on the device, int32 ascending).  Iteration t's seed is drawn
        from libc rand() -- the process-global stream the reference draws from, so srand() makes a run repeatable.
        Diagnostics of the winning hypothesis go to last_ransac_stats = (best iteration or -1, fitness, inlier_rmse)."""
        n, ransac_n, num_iterations = len(self), int(ransac_n), int(num_iterations)
        plane = np.zeros(4, np.float32)
        if ransac_n < 3:
            print("[cupoch_b200][error] ransac_n should be set to higher than or equal to 3.", file=sys.stderr)
            return plane, DeviceArray((0,), np.int32)
        if n < ransac_n:
            print("[cupoch_b200][error] There must be at least 'ransac_n' points.", file=sys.stderr)
            return plane, DeviceArray((0,), np.int32)
        rand = C.CDLL(None).rand
        rand.restype = C.c_int
        seeds = (C.c_int32 * max(num_iterations, 1))(*[rand() for _ in range(num_iterations)])
        d_idx = DeviceArray((n,), np.int32)
        h_plane, m, best, fr = (C.c_float * 4)(), C.c_size_t(0), C.c_int32(-1), (C.c_float * 2)()
        _lib.check(_lib.lib().cphb_segment_plane(self._points.ptr, n, float(distance_threshold), ransac_n, num_iterations,
                                                 seeds, h_plane, d_idx.ptr, C.byref(m), C.byref(best), fr, None, None))
        self.last_ransac_stats = (int(best.value), float(fr[0]), float(fr[1]))
        return np.array(h_plane, np.float32), DeviceArray((m.value,), np.int32, ptr=d_idx.ptr, base=d_idx)

    def farthest_point_down_sample(self, num_samples):
        """PointCloud::FarthestPointDownSample (pointcloud.cu:301-338; Open3D's binding name) -> new cloud of the
        num_samples points picked by farthest-point sampling from index 0, in pick order, with their normals and
        colours.  0 gives an empty cloud and len(self) a copy of the whole cloud in its original order.  More samples
        than points is logged and the loop runs anyway, as in the reference: the output then repeats points."""
        n, k = len(self), int(num_samples)
        if k < 0:
            raise ValueError("num_samples must be >= 0")
        if k == 0:
            return PointCloud()
        if k == n:
            return self.clone()
        if k > n:
            print("[cupoch_b200][error] Illegal number of samples: %d, must <= point size: %d" % (k, n), file=sys.stderr)
            if n == 0:  # the reference would gather out of range here
                return PointCloud()
        d_idx = DeviceArray((k,), np.int32)
        _lib.check(_lib.lib().cphb_farthest_point_down_sample(self._points.ptr, n, k, d_idx.ptr, None, None))
        return self._filtered(d_idx, k)[0]

    def cluster_dbscan(self, eps, min_points, print_progress=False, max_edges=100):
        """PointCloud::ClusterDBSCAN (pointcloud_cluster.cu:84-179; bound as cluster_dbscan, pointcloud.cpp:228-245) ->
        device vector of n int32 labels, -1 = noise."""
        n = len(self)
        labels = DeviceArray((n,), np.int32)
        if n:
            k = C.c_int(0)
            _lib.check(_lib.lib().cphb_cluster_dbscan(self._points.ptr, n, float(eps), int(min_points), int(max_edges),
                                                      labels.ptr, C.byref(k), None))
            self.last_cluster_count = int(k.value)
        return labels

    def gaussian_filter(self, search_radius, sigma2, num_max_search_points=50):
        """PointCloud::GaussianFilter (pointcloud.cu:387-433) -> new cloud (empty for illegal parameters)"""
        out = PointCloud()
        n = len(self)
        if n == 0:
            return out
        hn, hc = self.has_normals(), self.has_colors()
        op = DeviceArray((n, 3), np.float32)
        on = DeviceArray((n, 3), np.float32) if hn else None
        oc = DeviceArray((n, 3), np.float32) if hc else None
        m = C.c_size_t(0)
        _lib.check(_lib.lib().cphb_gaussian_filter(
            self._points.ptr, self._normals.ptr if hn else None, self._colors.ptr if hc else None, n, float(search_radius),
            float(sigma2), int(num_max_search_points), op.ptr, on.ptr if hn else None, oc.ptr if hc else None, C.byref(m), None))
        if m.value:
            out._points, out._normals, out._colors = op, on, oc
        return out

    def estimate_normals(self, search_param=None):
        """PointCloud::EstimateNormals (estimate_normals.cu:82-127)."""
        search_param = search_param or KDTreeSearchParamKNN()
        n = len(self)
        if n == 0:
            return True
        out = DeviceArray((n, 3), np.float32)
        if isinstance(search_param, KDTreeSearchParamKNN):
            knn, radius, max_nn = search_param.knn, 0.0, 0
        else:
            knn, radius, max_nn = 0, search_param.radius, search_param.max_nn
        _lib.check(_lib.lib().cphb_estimate_normals(self._points.ptr, n, knn, radius, max_nn, out.ptr, None))
        self._normals = out
        return True

    # -- bounding boxes and cleanup (SURVEY 8f rank 10) ----------------------
    def get_axis_aligned_bounding_box(self):
        """GetAxisAlignedBoundingBox: the min / max bound box (the zero box for an empty cloud)"""
        return AxisAlignedBoundingBox(*self._bounds())

    def get_oriented_bounding_box(self):
        """GetOrientedBoundingBox (boundingvolume.cu:219-269): PCA box; see cphb_oriented_bounding_box"""
        return OrientedBoundingBox.create_from_points(self._points)

    def _select(self, fn, *args):
        """(cloud of the rows a cphb_*_point_indices call keeps, their count)"""
        n = len(self)
        if n == 0:
            return PointCloud(), 0
        d_idx = DeviceArray((n,), np.int32)
        m = C.c_size_t(0)
        _lib.check(fn(self._points.ptr, n, *args, d_idx.ptr, C.byref(m), None))
        return self._filtered(d_idx, m.value)[0], m.value

    def crop(self, bounding_box):
        """Crop(AxisAlignedBoundingBox | OrientedBoundingBox) (pointcloud.cu:340-356): the rows inside the box, with their
        normals and colours.  An empty box (volume <= 0) is logged and the crop still runs, as in the reference."""
        if not isinstance(bounding_box, (AxisAlignedBoundingBox, OrientedBoundingBox)):
            raise TypeError("crop() takes an AxisAlignedBoundingBox or an OrientedBoundingBox")
        if bounding_box.is_empty():
            print("[cupoch_b200][error] [CropPointCloud] AxisAlignedBoundingBox either has zeros size, or has wrong "
                  "bounds.", file=sys.stderr)
        if isinstance(bounding_box, AxisAlignedBoundingBox):
            lo, hi = bounding_box._f3s()
            return self._select(_lib.lib().cphb_aabb_point_indices, lo, hi)[0]
        return self._select(_lib.lib().cphb_obb_point_indices, bounding_box._box24())[0]

    def pass_through_filter(self, axis_no, min_bound, max_bound):
        """PassThroughFilter (pointcloud.cu:436-460): the rows with min_bound <= p[axis_no] <= max_bound (NaN kept).
        axis_no outside 0..2 is logged and gives an empty cloud.  Covariances survive only when no row is removed (the
        reference copies the whole cloud and compacts points, normals and colours)."""
        axis_no = int(axis_no)
        if not 0 <= axis_no < 3:
            print("[cupoch_b200][error] [PassThroughFilter] Illegal input parameters, axis_no must be 0, 1 or 2.",
                  file=sys.stderr)
            return PointCloud()
        lo, hi = [-np.inf] * 3, [np.inf] * 3
        lo[axis_no], hi[axis_no] = float(min_bound), float(max_bound)
        out, m = self._select(_lib.lib().cphb_aabb_point_indices, (C.c_float * 3)(*lo), (C.c_float * 3)(*hi))
        if m == len(self) and self.has_covariances():
            out._covariances = self.clone()._covariances
        return out

    def remove_none_finite_points(self, remove_nan=True, remove_infinite=True):
        """RemoveNoneFinitePoints (pointcloud.cu:359-385), in place: points, normals and colours are compacted; when rows
        are removed the covariances no longer match the points and are dropped (has_covariances() becomes false)."""
        n = len(self)
        out, m = self._select(_lib.lib().cphb_finite_point_indices, int(bool(remove_nan)), int(bool(remove_infinite)))
        if m != n:
            hn, hc = self.has_normals(), self.has_colors()
            self._points = out._points if m else DeviceArray((0, 3), np.float32)
            if hn:
                self._normals = out._normals if m else DeviceArray((0, 3), np.float32)
            if hc:
                self._colors = out._colors if m else DeviceArray((0, 3), np.float32)
            self._covariances = self._color_gradient = None
        return self

    def uniform_down_sample(self, every_k_points):
        """UniformDownSample (down_sample.cu:275-300): rows 0, k, 2k, ... -- n // k of them (the reference sizes its
        output so but copies one more row when k does not divide n).  k == 0 is logged and gives an empty cloud."""
        k = int(every_k_points)
        if k <= 0:
            print("[cupoch_b200][error] [UniformDownSample] Illegal sample rate.", file=sys.stderr)
            return PointCloud()
        out = PointCloud()
        n = len(self)
        m = n // k
        if m == 0:
            return out
        hn, hc = self.has_normals(), self.has_colors()
        op = DeviceArray((m, 3), np.float32)
        on = DeviceArray((m, 3), np.float32) if hn else None
        oc = DeviceArray((m, 3), np.float32) if hc else None
        got = C.c_size_t(0)
        _lib.check(_lib.lib().cphb_uniform_down_sample(
            self._points.ptr, self._normals.ptr if hn else None, self._colors.ptr if hc else None, n, k, op.ptr,
            on.ptr if hn else None, oc.ptr if hc else None, C.byref(got), None))
        _lib.check(_lib.lib().cphb_stream_synchronize(None))
        out._points, out._normals, out._colors = op, on, oc
        return out

    @staticmethod
    def create_from_occupancy_grid(occupancy_grid):
        """PointCloud::CreateFromOccupancyGrid (pointcloud_factory.cu:418-430): one point per occupied cell, at
        (cell + (-(resolution / 2) + 0.5)) * voxel_size + origin, colour (0, 0, 1), in ExtractOccupiedVoxels order"""
        occupancy_grid._sync_params()
        L, h, n = _lib.lib(), occupancy_grid._h, C.c_size_t(0)
        _lib.check(L.cphb_point_cloud_from_occgrid(h, None, None, 0, C.byref(n), None))
        out = PointCloud()
        m = n.value
        if m:
            pts, cols = DeviceArray((m, 3), np.float32), DeviceArray((m, 3), np.float32)
            _lib.check(L.cphb_point_cloud_from_occgrid(h, pts.ptr, cols.ptr, m, C.byref(n), None))
            out._points, out._colors = pts, cols
        return out

    @staticmethod
    def _from_depth(d_depth, d_color, intrinsic, extrinsic, depth_scale, depth_trunc, stride, depth_cutoff, compute_normals,
                    valid_only):
        """cphb_depth_to_points into width / stride x height / stride rows; the rows kept are views of the first m"""
        w, h, dch, dbytes = RGBDImage._info(d_depth)
        cw, chh, cch, cbytes = RGBDImage._info(d_color) if d_color is not None else (0, 0, 0, 0)
        stride = int(stride)
        n = (w // stride) * (h // stride) if stride >= 1 else 0
        outs = [DeviceArray((n, 3), np.float32) if n and want else None
                for want in (True, compute_normals, d_color is not None)]
        m = C.c_size_t(0)
        _lib.check(_lib.lib().cphb_depth_to_points(
            d_depth.ptr, w, h, dch, dbytes, float(depth_scale), float(depth_trunc), stride,
            d_color.ptr if d_color is not None else None, cw, chh, cch, cbytes, _floats(intrinsic.intrinsic_matrix, 9),
            _floats(extrinsic, 16), float(depth_cutoff), int(bool(compute_normals)), int(bool(valid_only)),
            *[o.ptr if o is not None else None for o in outs], n, C.byref(m), None))
        out = PointCloud()
        if m.value:
            out._points, out._normals, out._colors = [None if o is None else o if m.value == n else
                                                      DeviceArray((m.value, 3), np.float32, ptr=o.ptr, base=o) for o in outs]
        return out

    @staticmethod
    def create_from_depth_image(depth, intrinsic, extrinsic=np.eye(4), depth_scale=1000.0, depth_trunc=1000.0, stride=1):
        """PointCloud::CreateFromDepthImage (pointcloud_factory.cu:43-105, 329-350): the point of every stride-th pixel
        of every stride-th row whose depth is > 0, in pixel order, in the world frame of the world-to-camera extrinsic.
        depth: a 1-channel uint16 geometry.Image (raw / int(depth_scale), 0 where that is >= int(depth_trunc)) or
        float32 one (metres, as it is).  Another format, stride < 1 or a singular extrinsic raises."""
        if depth.num_of_channels != 1 or depth.bytes_per_channel not in (2, 4):
            raise ValueError("[PointCloud::CreateFromDepthImage] Unsupported image format.")
        d = DeviceArray.from_numpy(depth._data.reshape(depth.height, depth.width), depth._data.dtype)
        return PointCloud._from_depth(d, None, intrinsic, extrinsic, depth_scale, depth_trunc, stride, -1.0, False, True)

    @staticmethod
    def create_from_rgbd_image(image, intrinsic, extrinsic=np.eye(4), project_valid_depth_only=True, depth_cutoff=-1.0,
                               compute_normals=False):
        """PointCloud::CreateFromRGBDImage (pointcloud_factory.cu:107-200, 288-327, 352-373), from the device images the
        RGBDImage holds: a point and colour per pixel whose depth is > 0 (and < depth_cutoff when that is > 0).  The
        colour image is uint8 RGB (c / 255) or 1-channel float32 intensity (g -> (g, g, g)); another format raises.
        compute_normals: structured normals from the four neighbouring pixels (0 on the border rows and columns),
        turned towards the camera (z <= 0).  project_valid_depth_only=False: one row per pixel, NaN where there is no
        point."""
        d_color, d_depth = image._device()
        if RGBDImage._info(d_depth)[2:] != (1, 4):
            raise ValueError("[PointCloud::CreateFromRGBDImage] the depth image must be 1-channel float32")
        return PointCloud._from_depth(d_depth, d_color, intrinsic, extrinsic, 1000.0, 1000.0, 1, depth_cutoff, compute_normals,
                                      project_valid_depth_only)

    def normalize_normals(self):
        """NormalizeNormals (pointcloud.cu:282-285), in place: every non-zero normal divided by its length"""
        if self._normals is not None and len(self._normals):
            _lib.check(_lib.lib().cphb_normalize_normals(self._normals.ptr, len(self._normals), None))
            _lib.check(_lib.lib().cphb_stream_synchronize(None))
        return self

    def orient_normals_to_align_with_direction(self, orientation_reference=(0.0, 0.0, 1.0)):
        """OrientNormalsToAlignWithDirection (estimate_normals.cu:129-141), in place: a zero normal becomes the
        reference, a normal pointing away from it (n . ref < 0) is negated.  No normals: warns, returns False."""
        if not self.has_normals():
            print("[cupoch_b200][warning] [OrientNormalsToAlignWithDirection] No normals in the PointCloud. Call "
                  "EstimateNormals() first.", file=sys.stderr)
            return False
        ref = (C.c_float * 3)(*[float(x) for x in np.asarray(orientation_reference, np.float32).reshape(3)])
        _lib.check(_lib.lib().cphb_orient_normals(self._normals.ptr, len(self), ref, None))
        _lib.check(_lib.lib().cphb_stream_synchronize(None))
        return True


class FilterScope(enum.IntEnum):
    """MeshBase::FilterScope (meshbase.h:55): which vertex attributes a mesh filter changes"""
    All = 0
    Color = 1
    Normal = 2
    Vertex = 3


# cphb_mesh_filter's kinds and attribute mask bits (include/cupoch_b200.h)
_SHARPEN, _SIMPLE, _LAPLACIAN, _TAUBIN = 0, 1, 2, 3
_SCOPE_MASK = {FilterScope.All: 7, FilterScope.Vertex: 1, FilterScope.Normal: 2, FilterScope.Color: 4}


class TriangleMesh:
    """geometry::TriangleMesh (trianglemesh.h): vertices_, triangles_ (int32 vertex indices), vertex_colors_,
    vertex_normals_, triangle_normals_ and edge_list_ (int32 pairs) on the device.  The normal computations,
    ComputeEdgeList, the four vertex filters, GetSurfaceArea, SamplePointsUniformly and the bounds run here, and
    VoxelGrid.create_from_triangle_mesh[_within_bounds] turns a mesh into a grid.  The cleanup operations
    (remove_duplicated_vertices / _triangles, remove_unreferenced_vertices, remove_degenerate_triangles),
    get_self_intersecting_triangles and + / += run here too; mesh IO, primitives and textures are not provided."""

    def __init__(self, vertices=None, triangles=None):
        self._vertices = self._triangles = self._vertex_colors = self._vertex_normals = self._triangle_normals = None
        self._edge_list = None
        if vertices is not None:
            self.vertices = vertices
        if triangles is not None:
            self.triangles = triangles

    vertices = property(lambda s: s._vertices, lambda s, v: setattr(s, "_vertices", Vector3fVector(v)))
    triangles = property(lambda s: s._triangles, lambda s, v: setattr(s, "_triangles", _vector3i(v)))
    vertex_colors = property(lambda s: s._vertex_colors, lambda s, v: setattr(s, "_vertex_colors", Vector3fVector(v)))
    vertex_normals = property(lambda s: s._vertex_normals, lambda s, v: setattr(s, "_vertex_normals", Vector3fVector(v)))
    triangle_normals = property(lambda s: s._triangle_normals, lambda s, v: setattr(s, "_triangle_normals", Vector3fVector(v)))
    edge_list = property(lambda s: s._edge_list, lambda s, v: setattr(s, "_edge_list", _vector2i(v)))

    def __repr__(self):
        return "geometry::TriangleMesh with %d points and %d triangles." % (self._n(self._vertices), self._n(self._triangles))

    @staticmethod
    def _n(a):
        return 0 if a is None else len(a)

    def is_empty(self):
        return not self.has_vertices()

    # trianglemesh.h / meshbase.h: "non-empty and, for a per-vertex or per-triangle attribute, of matching length"
    def has_vertices(self):
        return self._n(self._vertices) > 0

    def has_triangles(self):
        return self.has_vertices() and self._n(self._triangles) > 0

    def has_vertex_colors(self):
        return self.has_vertices() and self._n(self._vertex_colors) == len(self._vertices)

    def has_vertex_normals(self):
        return self.has_vertices() and self._n(self._vertex_normals) == len(self._vertices)

    def has_triangle_normals(self):
        return self.has_triangles() and self._n(self._triangle_normals) == len(self._triangles)

    def has_edge_list(self):
        return self._n(self._edge_list) > 0

    def get_min_bound(self):
        """MeshBase::GetMinBound: the smallest coordinate of all vertices per axis, (0, 0, 0) without vertices"""
        return self._bounds()[0]

    def get_max_bound(self):
        """MeshBase::GetMaxBound: the largest coordinate of all vertices per axis, (0, 0, 0) without vertices"""
        return self._bounds()[1]

    def _bounds(self):
        mn, mx = (C.c_float * 3)(), (C.c_float * 3)()
        n = self._n(self._vertices)
        if n:
            _lib.check(_lib.lib().cphb_min_max_bound(self._vertices.ptr, n, mn, mx, None))
        return np.array(mn, np.float32), np.array(mx, np.float32)

    def compute_triangle_normals(self, normalized=True):
        """ComputeTriangleNormals (trianglemesh.cu:466-477): (v1 - v0) x (v2 - v0) per triangle, then normalised when
        asked.  A vertex index outside [0, len(vertices)) raises."""
        m = self._n(self._triangles)
        out = DeviceArray((m, 3), np.float32)
        if m:
            _lib.check(_lib.lib().cphb_mesh_triangle_normals(self._vertices.ptr if self._vertices is not None else None,
                                                             self._n(self._vertices), self._triangles.ptr, m, int(bool(normalized)),
                                                             out.ptr, None))
        self._triangle_normals = out
        return self

    def compute_vertex_normals(self, normalized=True):
        """ComputeVertexNormals (trianglemesh.cu:479-503): the unnormalised triangle normals first when the mesh has
        none; each vertex's normal is the sum of its triangles' normals in ascending triangle order, then normalised
        when asked.  A vertex in no triangle gets a zero normal (the reference drops it and misaligns the rest)."""
        if not self.has_triangle_normals():
            self.compute_triangle_normals(False)
        n, m = self._n(self._vertices), self._n(self._triangles)
        out = DeviceArray((n, 3), np.float32)
        if n or m:
            _lib.check(_lib.lib().cphb_mesh_vertex_normals(self._triangles.ptr if m else None, m,
                                                           self._triangle_normals.ptr if m else None, n, int(bool(normalized)),
                                                           out.ptr, None))
        self._vertex_normals = out
        return self

    def compute_edge_list(self):
        """ComputeEdgeList (trianglemesh.cu:505-519): the directed edges (a, b) and (b, a) of every triangle edge, sorted
        and unique, as an (n, 2) int32 device array.  A vertex index outside [0, len(vertices)) raises."""
        m = self._n(self._triangles)
        buf = DeviceArray((max(6 * m, 1), 2), np.int32)
        n = C.c_size_t(0)
        _lib.check(_lib.lib().cphb_mesh_edge_list(self._triangles.ptr if m else None, m, self._n(self._vertices), buf.ptr, 6 * m,
                                                  C.byref(n), None))
        self._edge_list = _rows(buf, n.value)
        return self

    def _filter(self, kind, number_of_iterations, c0, c1, filter_scope):
        """the four filters' common path: a new mesh with the triangles, the edge list (this mesh's own when it has one,
        checked for range and order) and every vertex attribute, filtered or copied"""
        mask = _SCOPE_MASK[FilterScope(filter_scope)]
        if not self.has_edge_list():
            self.compute_edge_list()
        n = self._n(self._vertices)
        out = TriangleMesh()
        out._triangles, out._edge_list = self._triangles, self._edge_list
        ins = [self._vertices if n else None, self._vertex_normals if self.has_vertex_normals() else None,
               self._vertex_colors if self.has_vertex_colors() else None]
        outs = [None if a is None else DeviceArray((n, 3), np.float32) for a in ins]
        _lib.check(_lib.lib().cphb_mesh_filter(kind, int(number_of_iterations), float(c0), float(c1), self._edge_list.ptr,
                                               self._n(self._edge_list), n, *[None if a is None else a.ptr for a in ins], mask,
                                               *[None if a is None else a.ptr for a in outs], None))
        out._vertices, out._vertex_normals, out._vertex_colors = outs
        if out._vertices is None:
            out._vertices = DeviceArray((0, 3), np.float32)
        return out

    def filter_sharpen(self, number_of_iterations=1, strength=1.0, filter_scope=FilterScope.All):
        """FilterSharpen (trianglemesh.cu:521-599) -> a new mesh: per iteration v + strength * (v * N - sum of the N
        neighbours).  A vertex without neighbours keeps its value; number_of_iterations <= 0 copies."""
        return self._filter(_SHARPEN, number_of_iterations, strength, 0.0, filter_scope)

    def filter_smooth_simple(self, number_of_iterations=1, filter_scope=FilterScope.All):
        """FilterSmoothSimple (trianglemesh.cu:601-679) -> a new mesh: per iteration (v + sum of the N neighbours) /
        (1 + N)."""
        return self._filter(_SIMPLE, number_of_iterations, 0.0, 0.0, filter_scope)

    def filter_smooth_laplacian(self, number_of_iterations=1, lambda_=0.5, filter_scope=FilterScope.All, **kw):
        """FilterSmoothLaplacian (trianglemesh.cu:681-735) -> a new mesh: per iteration v + lambda (sum w_nb v_nb /
        sum w_nb - v), w = 1 / (|v - v_nb| + 1e-12) from the input vertices.  The reference's keyword `lambda` is
        accepted as lambda_."""
        return self._filter(_LAPLACIAN, number_of_iterations, kw.pop("lambda", lambda_), 0.0, _no_more(filter_scope, kw))

    def filter_smooth_taubin(self, number_of_iterations=1, lambda_=0.5, mu=-0.53, filter_scope=FilterScope.All, **kw):
        """FilterSmoothTaubin (trianglemesh.cu:737-800) -> a new mesh: per iteration a Laplacian step with lambda, then
        one with mu, with the weights of the input vertices.  `lambda` is accepted as lambda_."""
        return self._filter(_TAUBIN, number_of_iterations, kw.pop("lambda", lambda_), mu, _no_more(filter_scope, kw))

    def get_surface_area(self):
        """GetSurfaceArea (trianglemesh.cu:802-813): the sum of 0.5 |(p0 - p1) x (p0 - p2)| over the triangles, in
        float64 in a fixed order, as float32"""
        return self._surface_area(None)

    def _surface_area(self, areas):
        m = self._n(self._triangles)
        a = C.c_float(0)
        if m:
            _lib.check(_lib.lib().cphb_mesh_surface_area(self._vertices.ptr if self.has_vertices() else None, self._n(self._vertices),
                                                         self._triangles.ptr, m, None if areas is None else areas.ptr, C.byref(a), None))
        return float(a.value)

    def sample_points_uniformly(self, number_of_points=100, use_triangle_normal=False):
        """SamplePointsUniformly (trianglemesh.cu:830-901) -> a device PointCloud of exactly number_of_points points,
        triangle i taking llrint(cdf_i n) - llrint(cdf_{i-1} n) of them.  Normals: the triangle's when
        use_triangle_normal (computed, normalised, and kept on this mesh when it has none), else the interpolated vertex
        normals when there are any; colours are interpolated.  number_of_points 0 or above 2^30 - 1, no triangles or a
        surface area that is not positive and finite raises."""
        n = int(number_of_points)
        if n <= 0:
            raise ValueError("[SamplePointsUniformly] number_of_points <= 0")
        if not self.has_triangles():
            raise ValueError("[SamplePointsUniformly] input mesh has no triangles")
        if use_triangle_normal and not self.has_triangle_normals():
            self.compute_triangle_normals(True)
        vn = self._vertex_normals if self.has_vertex_normals() else None
        tn = self._triangle_normals if use_triangle_normal else None
        vc = self._vertex_colors if self.has_vertex_colors() else None
        if n > _MAX_SAMPLES:
            raise ValueError("[SamplePointsUniformly] number_of_points exceeds 2^30 - 1")
        pts = DeviceArray((n, 3), np.float32)
        nrm = DeviceArray((n, 3), np.float32) if (vn is not None or tn is not None) else None
        col = DeviceArray((n, 3), np.float32) if vc is not None else None
        _lib.check(_lib.lib().cphb_mesh_sample_points_uniformly(
            self._vertices.ptr, len(self._vertices), self._triangles.ptr, len(self._triangles), None if vn is None else vn.ptr,
            None if tn is None else tn.ptr, None if vc is None else vc.ptr, n, pts.ptr, None if nrm is None else nrm.ptr,
            None if col is None else col.ptr, None))
        pc = PointCloud()
        pc._points, pc._normals, pc._colors = pts, nrm, col
        return pc

    # ------------------------------------------------------------------ cleanup (trianglemesh.cu:903-1141)
    def _vertex_attrs(self):
        return (self._vertex_normals if self.has_vertex_normals() else None,
                self._vertex_colors if self.has_vertex_colors() else None)

    def _vertex_pass(self, fn):
        """the common path of the two vertex removals -> whether vertices were removed"""
        n, m = self._n(self._vertices), self._n(self._triangles)
        vn, vc = self._vertex_attrs()
        ov = DeviceArray((n, 3), np.float32)
        on, oc = [None if a is None else DeviceArray((n, 3), np.float32) for a in (vn, vc)]
        ot = DeviceArray((m, 3), np.int32)
        k = C.c_size_t(0)
        _lib.check(fn(self._vertices.ptr if n else None, None if vn is None else vn.ptr, None if vc is None else vc.ptr, n,
                      self._triangles.ptr if m else None, m, ov.ptr, None if on is None else on.ptr, None if oc is None else oc.ptr,
                      ot.ptr, C.byref(k), None))
        k = k.value
        if n:
            self._vertices = _rows(ov, k)
            if on is not None:
                self._vertex_normals = _rows(on, k)
            if oc is not None:
                self._vertex_colors = _rows(oc, k)
        if m:
            self._triangles = ot
        return k < n

    def _triangle_pass(self, fn):
        """the common path of the two triangle removals -> whether triangles were removed"""
        m = self._n(self._triangles)
        if m == 0:
            return False
        tn = self._triangle_normals if self.has_triangle_normals() else None
        ot = DeviceArray((m, 3), np.int32)
        otn = None if tn is None else DeviceArray((m, 3), np.float32)
        k = C.c_size_t(0)
        _lib.check(fn(self._triangles.ptr, None if tn is None else tn.ptr, m, self._n(self._vertices), ot.ptr,
                      None if otn is None else otn.ptr, C.byref(k), None))
        k = k.value
        self._triangles = _rows(ot, k)
        if otn is not None:
            self._triangle_normals = _rows(otn, k)
        return k < m

    def remove_duplicated_vertices(self):
        """RemoveDuplicatedVertices (trianglemesh.cu:903-969): the distinct positions (IEEE ==, so -0 and +0 are one) in
        lexicographic (x, y, z) order, each keeping the normal and colour of its lowest original index; triangles are
        remapped.  A vertex with a NaN coordinate merges with nothing and goes last, in original order.  The edge list
        is recomputed when the mesh has one.  A vertex index outside [0, len(vertices)) raises and changes nothing."""
        self._vertex_pass(_lib.lib().cphb_mesh_remove_duplicated_vertices)
        if self.has_edge_list():
            self.compute_edge_list()
        return self

    def remove_duplicated_triangles(self):
        """RemoveDuplicatedTriangles (trianglemesh.cu:971-1009): every triangle rotated so its smallest index comes first
        (orientation kept: (a, b, c) and (a, c, b) differ), sorted, and the first of each run kept with its normal.  The
        mesh keeps the rotated triangles in sorted order.  The edge list is recomputed when triangles were removed."""
        if self._triangle_pass(_lib.lib().cphb_mesh_remove_duplicated_triangles) and self.has_edge_list():
            self.compute_edge_list()
        return self

    def remove_unreferenced_vertices(self):
        """RemoveUnreferencedVertices (trianglemesh.cu:1011-1080): keeps, in order, the vertices some triangle uses, with
        their normals and colours; triangles are remapped.  The edge list is recomputed when vertices were removed."""
        if self._vertex_pass(_lib.lib().cphb_mesh_remove_unreferenced_vertices) and self.has_edge_list():
            self.compute_edge_list()
        return self

    def remove_degenerate_triangles(self):
        """RemoveDegenerateTriangles (trianglemesh.cu:1082-1121): drops, keeping the order, the triangles with two equal
        indices (a zero-area triangle with three distinct indices stays).  The edge list is recomputed when triangles
        were removed."""
        if self._triangle_pass(_lib.lib().cphb_mesh_remove_degenerate_triangles) and self.has_edge_list():
            self.compute_edge_list()
        return self

    def get_self_intersecting_triangles(self):
        """GetSelfIntersectingTriangles (trianglemesh.cu:1123-1141) -> (n, 2) int32 device array of the pairs i < j, in
        ascending order, that share no vertex index, have only finite vertices, have overlapping closed boxes, and
        that the reference's TriangleTriangle3d says intersect.  Found by an exact grid search (DESIGN section 4 item
        26): memory grows with the triangles and the hits, not with their square."""
        return self._self_intersections()[0]

    def _self_intersections(self):
        """-> (pairs, the number of box-overlapping pairs the predicate was evaluated on)"""
        m, n = self._n(self._triangles), self._n(self._vertices)
        L = _lib.lib()
        args = (self._vertices.ptr if n else None, n, self._triangles.ptr if m else None, m)
        cnt, cand = C.c_size_t(0), C.c_size_t(0)
        _lib.check(L.cphb_mesh_self_intersecting_triangles(*args, None, 0, C.byref(cnt), C.byref(cand), None))
        out = DeviceArray((cnt.value, 2), np.int32)
        if cnt.value:
            _lib.check(L.cphb_mesh_self_intersecting_triangles(*args, out.ptr, cnt.value, C.byref(cnt), C.byref(cand), None))
        return out, cand.value

    # ------------------------------------------------------------------ + and += (trianglemesh.cu:411-452, meshbase.cu:124-151)
    def __iadd__(self, other):
        """appends other's vertices and its triangles shifted by the old vertex count.  Vertex normals, vertex colours
        and triangle normals survive when other has them and this mesh has them or has no vertices (triangles for
        triangle normals); the edge list is recomputed when this mesh had one.  An empty other changes nothing."""
        if not isinstance(other, TriangleMesh):
            return NotImplemented
        if other.is_empty():
            return self
        na, nb = self._n(self._vertices), len(other._vertices)
        ta, tb = self._n(self._triangles), other._n(other._triangles)
        tri = DeviceArray((ta + tb, 3), np.int32)
        _lib.check(_lib.lib().cphb_mesh_append_triangles(self._triangles.ptr if ta else None, ta, na,
                                                         other._triangles.ptr if tb else None, tb, nb, tri.ptr, None))
        # the reference asks HasTriangles() after appending the vertices, so this mesh's own triangle count decides
        keep_tn = (ta == 0 or self.has_triangle_normals()) and other.has_triangle_normals()
        vn = (na == 0 or self.has_vertex_normals()) and other.has_vertex_normals()
        vc = (na == 0 or self.has_vertex_colors()) and other.has_vertex_colors()
        self._vertex_normals = _cat(self._vertex_normals if na else None, na, other._vertex_normals, nb) if vn else None
        self._vertex_colors = _cat(self._vertex_colors if na else None, na, other._vertex_colors, nb) if vc else None
        self._triangle_normals = (_cat(self._triangle_normals if ta else None, ta, other._triangle_normals, tb) if keep_tn
                                  else None)
        self._vertices = _cat(self._vertices, na, other._vertices, nb)
        self._triangles = tri
        if self.has_edge_list():
            self.compute_edge_list()
        return self

    def __add__(self, other):
        if not isinstance(other, TriangleMesh):
            return NotImplemented
        out = TriangleMesh()
        out._vertices, out._triangles, out._vertex_colors = self._vertices, self._triangles, self._vertex_colors
        out._vertex_normals, out._triangle_normals, out._edge_list = self._vertex_normals, self._triangle_normals, self._edge_list
        out += other
        return out


def _cat(a, na, b, nb):
    """rows [0, na) of a, then rows [0, nb) of b, as a new (na + nb, 3) device array"""
    out = DeviceArray((na + nb,) + b.shape[1:], b.dtype)
    L = _lib.lib()
    row = out.nbytes // max(na + nb, 1)
    if na:
        _lib.check(L.cphb_memcpy_d2d(out.ptr, a.ptr, row * na, None))
    if nb:
        _lib.check(L.cphb_memcpy_d2d(out.ptr + row * na, b.ptr, row * nb, None))
    _lib.check(L.cphb_stream_synchronize(None))
    return out


_MAX_SAMPLES = 2 ** 30 - 1  # CPHB_MESH_MAX_SAMPLES: draw 2 n must stay inside minstd_rand's period 2^31 - 2


def _no_more(filter_scope, kw):
    if kw:
        raise TypeError("unexpected keyword argument(s): %s" % ", ".join(sorted(kw)))
    return filter_scope


def _rows(buf, n):
    """the first n rows of a device array, as an array of their own"""
    out = DeviceArray((n,) + buf.shape[1:], buf.dtype)
    if out.nbytes:
        _lib.check(_lib.lib().cphb_memcpy_d2d(out.ptr, buf.ptr, out.nbytes, None))
        _lib.check(_lib.lib().cphb_stream_synchronize(None))
    return out


def _vector2i(a):
    if a is None:
        return None
    d = DeviceArray.wrap(a, np.int32)
    if len(d.shape) != 2 or d.shape[1] != 2:
        raise ValueError("expected (n,2) int32")
    return d


def _floats(a, n):
    return (C.c_float * n)(*np.asarray(a, np.float32).reshape(n).tolist())


def _vector3i(a):
    if a is None:
        return None
    d = DeviceArray.wrap(a, np.int32)
    if len(d.shape) != 2 or d.shape[1] != 3:
        raise ValueError("expected (n,3) int32")
    return d


def _v3(v):
    return np.asarray(v, np.float32).reshape(3).copy()


class AxisAlignedBoundingBox:
    """geometry::AxisAlignedBoundingBox<3> (boundingvolume.h:141-232; pybind boundingvolume.cpp): min_bound, max_bound
    and color are plain float32[3] attributes."""

    def __init__(self, min_bound=(0.0, 0.0, 0.0), max_bound=(0.0, 0.0, 0.0)):
        self.min_bound, self.max_bound = _v3(min_bound), _v3(max_bound)
        self.color = np.zeros(3, np.float32)

    def __repr__(self):
        return "geometry::AxisAlignedBoundingBox with min: (%f, %f, %f), max: (%f, %f, %f)" % (
            *self.min_bound.tolist(), *self.max_bound.tolist())

    def get_min_bound(self):
        return self.min_bound.copy()

    def get_max_bound(self):
        return self.max_bound.copy()

    def get_center(self):
        return ((self.min_bound + self.max_bound) * np.float32(0.5)).astype(np.float32)

    def get_extent(self):
        return (self.max_bound - self.min_bound).astype(np.float32)

    def get_half_extent(self):
        return (self.get_extent() * np.float32(0.5)).astype(np.float32)

    def get_max_extent(self):
        return float(self.get_extent().max())

    def volume(self):
        e = self.get_extent()
        return float(e[0] * e[1] * e[2])

    def is_empty(self):
        return self.volume() <= 0

    def get_axis_aligned_bounding_box(self):
        return AxisAlignedBoundingBox(self.min_bound, self.max_bound)

    def get_oriented_bounding_box(self):
        return OrientedBoundingBox.create_from_axis_aligned_bounding_box(self)

    def get_box_points(self):
        """GetBoxPoints (boundingvolume.cu:388-401) -> float32 [8, 3]"""
        lo, hi, e = self.min_bound, self.max_bound, self.get_extent()
        z = np.float32(0)
        ex, ey, ez = np.array([e[0], z, z]), np.array([z, e[1], z]), np.array([z, z, e[2]])
        return np.stack([lo, lo + ex, lo + ey, lo + ez, hi, hi - ex, hi - ey, hi - ez]).astype(np.float32)

    def _f3s(self):
        return (C.c_float * 3)(*self.min_bound.tolist()), (C.c_float * 3)(*self.max_bound.tolist())

    def get_point_indices_within_bounding_box(self, points):
        """ascending int32 indices (device) of the points inside the box, bounds inclusive; NaN points are kept"""
        return _point_indices(points, _lib.lib().cphb_aabb_point_indices, *self._f3s())

    @staticmethod
    def create_from_points(points):
        """CreateFromPoints (boundingvolume.cu:378-395): the points' min / max bound, the zero box when empty"""
        return PointCloud(points).get_axis_aligned_bounding_box()


class OrientedBoundingBox:
    """geometry::OrientedBoundingBox (boundingvolume.h:40-139; pybind boundingvolume.cpp): center, R (3x3, columns are
    the box axes) and extent are plain float32 attributes; color is kept for the reference's interface."""

    def __init__(self, center=(0.0, 0.0, 0.0), R=np.eye(3), extent=(0.0, 0.0, 0.0)):
        self.center, self.extent = _v3(center), _v3(extent)
        self.R = np.asarray(R, np.float32).reshape(3, 3).copy()
        self.color = np.zeros(3, np.float32)

    def __repr__(self):
        return "geometry::OrientedBoundingBox: center: (%f, %f, %f), extent: %f, %f, %f)" % (
            *self.center.tolist(), *self.extent.tolist())

    def get_center(self):
        return self.center.copy()

    def _size(self):
        return np.abs(self.R.astype(np.float32) @ self.extent.astype(np.float32)).astype(np.float32)

    def get_min_bound(self):
        return (self.center - np.float32(0.5) * self._size()).astype(np.float32)

    def get_max_bound(self):
        return (self.center + np.float32(0.5) * self._size()).astype(np.float32)

    def volume(self):
        return float(self.extent[0] * self.extent[1] * self.extent[2])

    def is_empty(self):
        return self.volume() <= 0

    def get_axis_aligned_bounding_box(self):
        return AxisAlignedBoundingBox(self.get_min_bound(), self.get_max_bound())

    def get_box_points(self):
        """GetBoxPoints (boundingvolume.cu:180-194) in float32: axis k = R[:, k] * (extent[k] / 2), the corners
        center -+ x -+ y -+ z evaluated left to right -> [8, 3]"""
        c, h = self.center, (self.extent / np.float32(2)).astype(np.float32)
        x, y, z = self.R[:, 0] * h[0], self.R[:, 1] * h[1], self.R[:, 2] * h[2]
        return np.stack([c - x - y - z, c + x - y - z, c - x + y - z, c - x - y + z,
                         c + x + y + z, c - x + y + z, c + x - y + z, c + x + y - z]).astype(np.float32)

    def _box24(self):
        return (C.c_float * 24)(*self.get_box_points().reshape(-1).tolist())

    def get_point_indices_within_bounding_box(self, points):
        """ascending int32 indices (device) of the points the six plane tests keep (boundingvolume.cu:38-79,228-244)"""
        return _point_indices(points, _lib.lib().cphb_obb_point_indices, self._box24())

    @staticmethod
    def create_from_axis_aligned_bounding_box(aabox):
        return OrientedBoundingBox(aabox.get_center(), np.eye(3), aabox.get_extent())

    @staticmethod
    def create_from_points(points):
        """CreateFromPoints (boundingvolume.cu:219-269): see cphb_oriented_bounding_box.  Empty input: the zero box."""
        pts = points if isinstance(points, DeviceArray) else Vector3fVector(points)
        n = 0 if pts is None else len(pts)
        c, R, e = (C.c_float * 3)(), (C.c_float * 9)(), (C.c_float * 3)()
        _lib.check(_lib.lib().cphb_oriented_bounding_box(pts.ptr if n else None, n, c, R, e, None))
        return OrientedBoundingBox(np.array(c, np.float32), np.array(R, np.float32).reshape(3, 3), np.array(e, np.float32))


def _point_indices(points, fn, *args):
    pts = points if isinstance(points, DeviceArray) else Vector3fVector(points)
    n = 0 if pts is None else len(pts)
    d_idx = DeviceArray((n,), np.int32)
    m = C.c_size_t(0)
    if n:
        _lib.check(fn(pts.ptr, n, *args, d_idx.ptr, C.byref(m), None))
    return DeviceArray((m.value,), np.int32, ptr=d_idx.ptr, base=d_idx)


class VoxelGrid:
    """geometry::VoxelGrid (voxelgrid.h:84-210; pybind voxelgrid.cpp:96-157).  voxels_keys / voxels_colors are device
    arrays ([m, 3] int32 grid indices, [m, 3] float32 colours).  The factories, +=, add_voxels and carving leave the
    keys in lexicographic order and unique; select_by_index and direct assignment may leave them in any order, with
    repeats, and every lookup accepts that."""

    def __init__(self):
        self.voxel_size = 0.0
        self.origin = np.zeros(3, np.float32)
        self.voxels_keys = None
        self.voxels_colors = None

    def __len__(self):
        return 0 if self.voxels_keys is None else self.voxels_keys.shape[0]

    def has_voxels(self):
        return len(self) > 0

    def has_colors(self):
        return True  # voxelgrid.h:112-114: by default the colours are (1, 1, 1)

    def get_voxels(self):
        """-> (keys [m,3] int32, colors [m,3] float32) on the host (VoxelGrid::GetVoxels)"""
        if not len(self):
            return np.zeros((0, 3), np.int32), np.zeros((0, 3), np.float32)
        return self.voxels_keys.cpu(), self.voxels_colors.cpu()

    def get_voxel(self, point):
        """VoxelGrid::GetVoxel (voxelgrid.cu:338-341): floor((point - origin) / voxel_size)"""
        p = np.asarray(point, np.float32)
        return np.floor((p - self.origin) / np.float32(self.voxel_size)).astype(np.int32)

    def get_min_bound(self):
        """voxelgrid.cu:161-172: min grid index * voxel_size + origin (origin when empty)"""
        if not len(self):
            return self.origin.copy()
        k = self.voxels_keys.cpu().min(0).astype(np.float32)
        return k * np.float32(self.voxel_size) + self.origin

    def get_max_bound(self):
        """voxelgrid.cu:174-187: (max grid index + 1) * voxel_size + origin"""
        if not len(self):
            return self.origin.copy()
        k = self.voxels_keys.cpu().max(0).astype(np.float32)
        return (k + np.float32(1)) * np.float32(self.voxel_size) + self.origin

    @staticmethod
    def create_from_point_cloud_within_bounds(input, voxel_size, min_bound, max_bound):
        """VoxelGrid::CreateFromPointCloudWithinBounds (voxelgrid_factory.cu:164-219)"""
        out = VoxelGrid()
        out.voxel_size = float(voxel_size)
        out.origin = np.asarray(min_bound, np.float32).reshape(3).copy()
        n = len(input)
        if n == 0:
            return out
        mn = (C.c_float * 3)(*[float(x) for x in out.origin])
        mx = (C.c_float * 3)(*[float(x) for x in np.asarray(max_bound, np.float32).reshape(3)])
        keys = DeviceArray((n, 3), np.int32)
        cols = DeviceArray((n, 3), np.float32)
        m = C.c_size_t(0)
        _lib.check(_lib.lib().cphb_voxel_grid_from_point_cloud(
            input._points.ptr, input._colors.ptr if input.has_colors() else None, n, float(voxel_size), mn, mx,
            keys.ptr, cols.ptr, C.byref(m), None))
        m = m.value
        if m:
            out.voxels_keys = DeviceArray((m, 3), np.int32, ptr=keys.ptr, base=keys)
            out.voxels_colors = DeviceArray((m, 3), np.float32, ptr=cols.ptr, base=cols)
        return out

    @staticmethod
    def create_from_point_cloud(input, voxel_size):
        """VoxelGrid::CreateFromPointCloud (voxelgrid_factory.cu:221-228): bounds widened by half a voxel"""
        if len(input) == 0:
            out = VoxelGrid()
            out.voxel_size = float(voxel_size)
            return out
        v = np.float32(voxel_size)
        mn, mx = input._bounds()
        return VoxelGrid.create_from_point_cloud_within_bounds(input, voxel_size, mn - v * np.float32(0.5),
                                                               mx + v * np.float32(0.5))

    # -- the rest of the reference's VoxelGrid (voxelgrid.cu:235-475) ------------------------------------------------
    def _like(self, keys=None, colors=None, m=0):
        """a grid with this one's geometry holding the first m rows of keys / colors; when that is fewer rows than the
        buffers hold (carving, merging) the rows are copied out, so the result does not keep the larger buffers alive"""
        out = VoxelGrid()
        out.voxel_size, out.origin = self.voxel_size, self.origin.copy()
        if m and m == keys.shape[0]:
            out.voxels_keys, out.voxels_colors = keys, colors
        elif m:
            out.voxels_keys, out.voxels_colors = DeviceArray((m, 3), np.int32), DeviceArray((m, 3), np.float32)
            L = _lib.lib()
            _lib.check(L.cphb_memcpy_d2d(out.voxels_keys.ptr, keys.ptr, 12 * m, None))
            _lib.check(L.cphb_memcpy_d2d(out.voxels_colors.ptr, colors.ptr, 12 * m, None))
            _lib.check(L.cphb_stream_synchronize(None))
        return out

    def _set(self, other):
        self.voxels_keys, self.voxels_colors = other.voxels_keys, other.voxels_colors
        return self

    def _f3(self, v=None):
        return (C.c_float * 3)(*np.asarray(self.origin if v is None else v, np.float32).reshape(3).tolist())

    def _device(self):
        """voxels_keys / voxels_colors as device arrays (assigned host keys are uploaded, missing colours are (1, 1, 1))"""
        if len(self):
            if not isinstance(self.voxels_keys, DeviceArray):
                self.voxels_keys = DeviceArray.wrap(self.voxels_keys, np.int32)
            if self.voxels_colors is None:
                self.voxels_colors = DeviceArray.from_numpy(np.ones((len(self), 3), np.float32), np.float32)
            elif not isinstance(self.voxels_colors, DeviceArray):
                self.voxels_colors = DeviceArray.wrap(self.voxels_colors, np.float32)
        return self

    def _keys_ptr(self):
        return self._device().voxels_keys.ptr if len(self) else None

    def _colors_ptr(self):
        return self._device().voxels_colors.ptr if len(self) else None

    @staticmethod
    def create_dense(origin, voxel_size, width, height, depth):
        """VoxelGrid::CreateDense (voxelgrid_factory.cu:134-162): int(round(extent / voxel_size)) voxels per axis, keys in
        lexicographic order, colours (1, 1, 1).  A bad voxel size, a negative count or an overflowing total raise."""
        out = VoxelGrid()
        out.voxel_size = float(np.float32(voxel_size))
        out.origin = np.asarray(origin, np.float32).reshape(3).copy()
        args = [float(np.float32(x)) for x in (voxel_size, width, height, depth)]
        n = C.c_size_t(0)
        _lib.check(_lib.lib().cphb_voxel_grid_create_dense(*args, None, None, 0, C.byref(n), None))
        m = n.value
        if m:
            keys, cols = DeviceArray((m, 3), np.int32), DeviceArray((m, 3), np.float32)
            _lib.check(_lib.lib().cphb_voxel_grid_create_dense(*args, keys.ptr, cols.ptr, m, C.byref(n), None))
            out.voxels_keys, out.voxels_colors = keys, cols
        return out

    @staticmethod
    def create_from_triangle_mesh_within_bounds(input, voxel_size, min_bound, max_bound):
        """VoxelGrid::CreateFromTriangleMeshWithinBounds (voxelgrid_factory.cu:229-272): origin = min_bound,
        int(round(extent / voxel_size)) cells per axis; a cell is a voxel when Akenine-Moeller's triangle/box test says
        some triangle meets it.  The cell tested for key k is centred at (k + 0.5) * voxel_size + origin, the cell
        get_voxel gives (the reference tests the box centred on the voxel's lower corner).  Keys unique and in
        lexicographic order, colours (1, 1, 1).  A triangle with a non-finite vertex meets no cell.  A bad vertex
        index, a voxel size that is not positive and finite, non-finite bounds, or a count that is negative or >= 2^21
        on an axis raise."""
        out = VoxelGrid()
        out.voxel_size = float(np.float32(voxel_size))
        out.origin = np.asarray(min_bound, np.float32).reshape(3).copy()
        nv, nt = TriangleMesh._n(input._vertices), TriangleMesh._n(input._triangles)
        mn, mx = out._f3(), out._f3(max_bound)
        args = (input._vertices.ptr if nv else None, nv, input._triangles.ptr if nt else None, nt, out.voxel_size, mn, mx)
        L, n = _lib.lib(), C.c_size_t(0)
        _lib.check(L.cphb_voxel_grid_from_triangle_mesh(*args, None, None, 0, C.byref(n), None))
        m = n.value
        if m:
            keys, cols = DeviceArray((m, 3), np.int32), DeviceArray((m, 3), np.float32)
            _lib.check(L.cphb_voxel_grid_from_triangle_mesh(*args, keys.ptr, cols.ptr, m, C.byref(n), None))
            out.voxels_keys, out.voxels_colors = keys, cols
        return out

    @staticmethod
    def create_from_triangle_mesh(input, voxel_size):
        """VoxelGrid::CreateFromTriangleMesh (voxelgrid_factory.cu:274-281): the bounds of all vertices widened by half a
        voxel"""
        v = np.float32(voxel_size)
        mn, mx = input._bounds()
        return VoxelGrid.create_from_triangle_mesh_within_bounds(input, voxel_size, mn - v * np.float32(0.5),
                                                                  mx + v * np.float32(0.5))

    @staticmethod
    def create_from_occupancy_grid(occupancy_grid):
        """VoxelGrid::CreateFromOccupancyGrid (voxelgrid_factory.cu:283-305): one voxel per occupied cell, key = its grid
        index, colour (0, 0, 1).  origin = grid origin - (resolution / 2) * voxel_size (the reference keeps the grid's
        origin, which puts every voxel resolution / 2 cells away from its cell)."""
        occupancy_grid._sync_params()
        L, h = _lib.lib(), occupancy_grid._h
        n, o = C.c_size_t(0), (C.c_float * 3)()
        _lib.check(L.cphb_voxel_grid_from_occgrid(h, None, None, 0, C.byref(n), o, None))
        out = VoxelGrid()
        out.voxel_size, out.origin = float(np.float32(occupancy_grid.voxel_size)), np.array(o, np.float32)
        m = n.value
        if m:
            keys, cols = DeviceArray((m, 3), np.int32), DeviceArray((m, 3), np.float32)
            _lib.check(L.cphb_voxel_grid_from_occgrid(h, keys.ptr, cols.ptr, m, C.byref(n), o, None))
            out.voxels_keys, out.voxels_colors = keys, cols
        return out

    def check_if_included(self, queries):
        """CheckIfIncluded (voxelgrid.cu:365-376): host [n, 3] queries -> [n] bool, whether each query's GetVoxel cell is
        a voxel.  Non-finite queries and cells outside the int range are False."""
        q = np.ascontiguousarray(np.asarray(queries, np.float32).reshape(-1, 3))
        if len(q) == 0:
            return np.zeros(0, bool)
        d = DeviceArray.from_numpy(q, np.float32)
        out = DeviceArray((len(q),), np.uint8)
        _lib.check(_lib.lib().cphb_voxel_grid_check_if_included(self._keys_ptr(), len(self), float(self.voxel_size), self._f3(),
                                                                d.ptr, len(q), out.ptr, None))
        return out.cpu().astype(bool)

    def get_voxel_center_coordinate(self, idx):
        """GetVoxelCenterCoordinate (voxelgrid.cu:343-354): ((idx + 0.5) * voxel_size) + origin, or the zero vector when
        idx is not a voxel (the reference's answer)."""
        k = np.asarray(idx, np.int32).reshape(3)
        found = C.c_int(0)
        _lib.check(_lib.lib().cphb_voxel_grid_has_key(self._keys_ptr(), len(self), (C.c_int32 * 3)(*k.tolist()), C.byref(found), None))
        if not found.value:
            return np.zeros(3, np.float32)
        return ((k.astype(np.float32) + np.float32(0.5)) * np.float32(self.voxel_size) + self.origin).astype(np.float32)

    def get_voxel_bounding_points(self, idx):
        """GetVoxelBoundingPoints (voxelgrid.cu:356-363): the 8 corners around GetVoxelCenterCoordinate(idx), in the
        order carving projects them (bit 0: +z, bit 1: +x, bit 2: +y)"""
        x = self.get_voxel_center_coordinate(idx)
        r = np.float32(self.voxel_size) * np.float32(0.5)
        sgn = np.array([[(j >> 1) & 1, (j >> 2) & 1, j & 1] for j in range(8)], np.float32) * 2 - 1
        return (x[None, :] + sgn * r).astype(np.float32)

    def _carve(self, image, camera_params, keep_voxels_outside_image, what):
        intr = camera_params.intrinsic
        if image.height != intr.height or image.width != intr.width:
            raise ValueError("[VoxelGrid] provided %s dimensions are not compatible with the provided camera_parameters" % what)
        n = len(self)
        sampled = image.num_of_channels == 1 and image.bytes_per_channel == 4
        img = DeviceArray.from_numpy(image._data, image._data.dtype) if sampled else None
        K = (C.c_float * 9)(*np.asarray(intr.intrinsic_matrix, np.float32).reshape(9).tolist())
        E = (C.c_float * 16)(*np.asarray(camera_params.extrinsic, np.float32).reshape(16).tolist())
        keys, cols = (DeviceArray((n, 3), np.int32), DeviceArray((n, 3), np.float32)) if n else (None, None)
        m = C.c_size_t(0)
        _lib.check(_lib.lib().cphb_voxel_grid_carve(self._keys_ptr(), self._colors_ptr(), n, float(self.voxel_size), self._f3(),
                                                    img.ptr if img is not None else None, image.width, image.height,
                                                    image.num_of_channels, image.bytes_per_channel, K, E,
                                                    int(bool(keep_voxels_outside_image)), keys.ptr if n else None,
                                                    cols.ptr if n else None, C.byref(m), None))
        return self._set(self._like(keys, cols, m.value))

    def carve_depth_map(self, depth_map, camera_params, keep_voxels_outside_image=False):
        """CarveDepthMap (voxelgrid.cu:378-403): removes every voxel none of whose corners projects to a pixel with
        depth d > 0 and z >= d (or outside the image, with keep_voxels_outside_image).  Only a 1-channel float32 image
        is sampled; any other image is outside everywhere, as in the reference."""
        return self._carve(depth_map, camera_params, keep_voxels_outside_image, "depth_map")

    def carve_silhouette(self, silhouette_mask, camera_params, keep_voxels_outside_image=False):
        """CarveSilhouette (voxelgrid.cu:405-430): the reference's test is the depth map's (d > 0 and z >= d), so a uint8
        mask is outside everywhere: every voxel is removed, or with keep_voxels_outside_image every voxel is kept."""
        return self._carve(silhouette_mask, camera_params, keep_voxels_outside_image, "silhouette_mask")

    def _merge(self, other, average):
        if float(np.float32(self.voxel_size)) != float(np.float32(other.voxel_size)):
            raise ValueError("[VoxelGrid] Could not combine VoxelGrid because voxel_size differs (this=%f, other=%f)"
                             % (self.voxel_size, other.voxel_size))
        if not np.array_equal(np.asarray(self.origin, np.float32), np.asarray(other.origin, np.float32)):
            raise ValueError("[VoxelGrid] Could not combine VoxelGrid because origin differs")
        n = len(self) + len(other)
        keys, cols = (DeviceArray((n, 3), np.int32), DeviceArray((n, 3), np.float32)) if n else (None, None)
        m = C.c_size_t(0)
        _lib.check(_lib.lib().cphb_voxel_grid_merge(self._keys_ptr(), self._colors_ptr(), len(self), other._keys_ptr(),
                                                    other._colors_ptr(), len(other), int(average), keys.ptr if n else None,
                                                    cols.ptr if n else None, C.byref(m), None))
        return self._like(keys, cols, m.value)

    def __iadd__(self, other):
        """operator+= (voxelgrid.cu:235-281): both grids' voxels, one per key, colours averaged over equal keys (summed
        in this grid's order, then the other's).  Different voxel sizes or origins raise."""
        return self._set(self._merge(other, True))

    def __add__(self, other):
        return self._merge(other, True)

    def add_voxels(self, keys, colors=None):
        """AddVoxels (voxelgrid.cu:299-319): voxels [m, 3] int32 keys (and [m, 3] colours, (1, 1, 1) by default); a key
        already present keeps its voxel"""
        other = self._like()
        k = np.ascontiguousarray(np.asarray(keys, np.int32).reshape(-1, 3))
        if len(k):
            c = np.ones((len(k), 3), np.float32) if colors is None else np.asarray(colors, np.float32).reshape(-1, 3)
            other.voxels_keys, other.voxels_colors = DeviceArray.from_numpy(k, np.int32), DeviceArray.from_numpy(c, np.float32)
        return self._set(self._merge(other, False))

    def add_voxel(self, key, color=(1.0, 1.0, 1.0)):
        """AddVoxel (voxelgrid.cu:288-297)"""
        return self.add_voxels(np.asarray(key).reshape(1, 3), np.asarray(color).reshape(1, 3))

    @staticmethod
    def _indices(indices):
        if isinstance(indices, DeviceArray) or hasattr(indices, "is_cuda"):
            return DeviceArray.wrap(indices, np.int64)
        return DeviceArray.from_numpy(np.ascontiguousarray(np.asarray(indices, np.int64).reshape(-1)), np.int64)

    def paint_uniform_color(self, color):
        """PaintUniformColor (voxelgrid.cu:321-325)"""
        _lib.check(_lib.lib().cphb_voxel_grid_paint(self._colors_ptr(), len(self), None, 0, self._f3(color), None))
        _lib.check(_lib.lib().cphb_stream_synchronize(None))
        return self

    def paint_indexed_color(self, indices, color):
        """PaintIndexedColor (voxelgrid.cu:327-336); an index outside [0, len) raises and nothing is painted"""
        d = self._indices(indices)
        if len(d):
            _lib.check(_lib.lib().cphb_voxel_grid_paint(self._colors_ptr(), len(self), d.ptr, len(d), self._f3(color), None))
            _lib.check(_lib.lib().cphb_stream_synchronize(None))
        return self

    def select_by_index(self, indices, invert=False):
        """SelectByIndex (voxelgrid.cu:432-475): the voxels at indices, in index order, or with invert the others in
        ascending order (repeated indices allowed).  An index outside [0, len) raises."""
        d = self._indices(indices)
        rows = len(self) if invert else len(d)
        keys, cols = (DeviceArray((rows, 3), np.int32), DeviceArray((rows, 3), np.float32)) if rows else (None, None)
        m = C.c_size_t(0)
        _lib.check(_lib.lib().cphb_voxel_grid_select_by_index(self._keys_ptr(), self._colors_ptr(), len(self),
                                                              d.ptr if len(d) else None, len(d), int(bool(invert)),
                                                              keys.ptr if rows else None, cols.ptr if rows else None,
                                                              C.byref(m), None))
        return self._like(keys, cols, m.value)


class Image:
    """geometry::Image as a data holder (image.h; pybind image.cpp:80-100): a C-contiguous uint8, uint16 or float32
    buffer of shape (height, width) or (height, width, channels) with 1, 3 or 4 channels.  Filters, pyramids and IO
    are not part of this project."""

    def __init__(self, data=None):
        if data is None:
            data = np.zeros((0, 0), np.uint8)
        a = np.asarray(data)
        if a.dtype not in (np.uint8, np.uint16, np.float32):
            raise ValueError("Image can only be initialized from buffer of uint8, uint16, or float!")
        if a.ndim not in (2, 3) or (a.ndim == 3 and a.shape[2] not in (1, 3, 4)):
            raise ValueError("Image can only be initialized from a (height, width) or (height, width, 1 | 3 | 4) buffer")
        self._data = np.ascontiguousarray(a)

    height = property(lambda s: int(s._data.shape[0]))
    width = property(lambda s: int(s._data.shape[1]))
    num_of_channels = property(lambda s: 1 if s._data.ndim == 2 else int(s._data.shape[2]))
    bytes_per_channel = property(lambda s: int(s._data.dtype.itemsize))

    def is_empty(self):
        return self._data.size == 0

    def __array__(self, dtype=None, copy=None):
        return self._data if dtype is None else self._data.astype(dtype)

    def __repr__(self):
        return "geometry::Image of size %dx%d, with %d channels." % (self.width, self.height, self.num_of_channels)


class RGBDImage:
    """geometry::RGBDImage (rgbdimage.h): a colour and a depth image of the same size, built by the create_from_*
    factories.  The converted images live on the device, where UniformTSDFVolume.integrate reads them; `color` and
    `depth` download them as geometry.Image on first access.  RGBDImage(color, depth) wraps two host Images as they
    are (no conversion), as the reference's constructor does."""

    def __init__(self, color=None, depth=None):
        self._color, self._depth = (Image() if color is None else color), (Image() if depth is None else depth)
        self._d_color = self._d_depth = None

    @staticmethod
    def _from_device(d_color, d_depth):
        out = RGBDImage()
        out._color = out._depth = None
        out._d_color, out._d_depth = d_color, d_depth
        return out

    @property
    def color(self):
        if self._color is None:
            self._color = Image(self._d_color.cpu())
        return self._color

    @property
    def depth(self):
        if self._depth is None:
            self._depth = Image(self._d_depth.cpu())
        return self._depth

    def _device(self):
        """(color, depth) as device arrays; host images are uploaded once"""
        if self._d_depth is None:
            self._d_depth = DeviceArray.from_numpy(self._depth._data, self._depth._data.dtype)
        if self._d_color is None:
            self._d_color = DeviceArray.from_numpy(self._color._data, self._color._data.dtype)
        return self._d_color, self._d_depth

    @staticmethod
    def _info(d):
        """(width, height, channels, bytes_per_channel) of a device image"""
        return (d.shape[1], d.shape[0], 1 if len(d.shape) == 2 else d.shape[2], d.dtype.itemsize)

    def _depth_info(self):
        return self._info(self._device()[1])

    def _color_info(self):
        return self._info(self._device()[0])

    def is_empty(self):
        return self.depth.is_empty()

    def __repr__(self):
        return "geometry::RGBDImage of size %dx%d." % (self.depth.width, self.depth.height)

    @staticmethod
    def _convert(image, to_depth, depth_scale=1000.0, depth_trunc=3.0):
        a = image._data
        src = DeviceArray.from_numpy(a, a.dtype)
        out = DeviceArray(a.shape[:2], np.float32)
        _lib.check(_lib.lib().cphb_rgbd_convert(src.ptr, image.width, image.height, image.num_of_channels, image.bytes_per_channel,
                                                int(to_depth), float(depth_scale), float(depth_trunc), out.ptr, None))
        _lib.check(_lib.lib().cphb_stream_synchronize(None))
        return out

    @staticmethod
    def create_from_color_and_depth(color, depth, depth_scale=1000.0, depth_trunc=3.0, convert_rgb_to_intensity=True):
        """RGBDImage::CreateFromColorAndDepth (rgbdimage_factory.cu:56-72): depth -> float32 metres, the raw value /
        int(depth_scale) and 0 where it is >= int(depth_trunc) (the reference converts both to int, so depth_trunc
        = 2.5 cuts at 2 m); colour -> float32 weighted intensity (/ 255 for 8-bit) when convert_rgb_to_intensity, else
        kept as it is.  Images of different sizes raise, as does a depth_scale below 1 (int 0 would divide by zero)."""
        if color.height != depth.height or color.width != depth.width:
            raise ValueError("[CreateFromColorAndDepth] Unsupported image format.")
        d = RGBDImage._convert(depth, True, depth_scale, depth_trunc)
        if convert_rgb_to_intensity:
            c = RGBDImage._convert(color, False)
        else:
            c = DeviceArray.from_numpy(color._data, color._data.dtype)
        return RGBDImage._from_device(c, d)

    @staticmethod
    def create_from_redwood_format(color, depth, convert_rgb_to_intensity=True):
        """CreateFromRedwoodFormat: depth_scale 1000, depth_trunc 4"""
        return RGBDImage.create_from_color_and_depth(color, depth, 1000.0, 4.0, convert_rgb_to_intensity)

    @staticmethod
    def create_from_tum_format(color, depth, convert_rgb_to_intensity=True):
        """CreateFromTUMFormat: depth_scale 5000, depth_trunc 4"""
        return RGBDImage.create_from_color_and_depth(color, depth, 5000.0, 4.0, convert_rgb_to_intensity)


class OccupancyVoxel:
    """geometry::OccupancyVoxel (occupancygrid.h:33-72): grid_index (3 uint16), prob_log, color (the default (0, 0, 1):
    nothing on this path ever changes it)."""

    def __init__(self, grid_index=(0, 0, 0), prob_log=float("nan"), color=(0.0, 0.0, 1.0)):
        self.grid_index = np.asarray(grid_index, np.uint16)
        self.prob_log = float(prob_log)
        self.color = np.asarray(color, np.float32)

    def __repr__(self):
        return "geometry::OccupancyVoxel with grid_index: (%d, %d, %d), prob_log: %f" % (*self.grid_index.tolist(), self.prob_log)


class OccupancyGrid:
    """geometry::OccupancyGrid (occupancygrid.h:74-147; pybind occupancygrid.cpp:77-126): dense log-odds grid on the device.
    `voxel_size`, `origin` and the five probability parameters are plain attributes as in the reference."""

    def __init__(self, voxel_size=0.05, resolution=512, origin=(0.0, 0.0, 0.0)):
        _lib.require_gpu()
        self._h = C.c_void_p()
        self._voxel_size, self._resolution = float(voxel_size), int(resolution)
        self._origin = np.asarray(origin, np.float32).reshape(3).copy()
        p = _lib.OccGridParams()
        _lib.lib().cphb_occgrid_default_params(C.byref(p))
        self.clamping_thres_min, self.clamping_thres_max = p.clamping_thres_min, p.clamping_thres_max
        self.prob_hit_log, self.prob_miss_log, self.occ_prob_thres_log = p.prob_hit_log, p.prob_miss_log, p.occ_prob_thres_log
        self.visualize_free_area = True
        _lib.check(_lib.lib().cphb_occgrid_create(self._voxel_size, self._resolution, self._f3(self._origin), None, C.byref(self._h)))

    @staticmethod
    def _f3(v):
        return (C.c_float * 3)(*np.asarray(v, np.float32).reshape(3).tolist())

    # voxel_size_ / origin_ are public members of the reference (its own tests assign them after construction)
    voxel_size = property(lambda s: s._voxel_size, lambda s, v: s._set_geometry(voxel_size=v))
    origin = property(lambda s: s._origin, lambda s, v: s._set_geometry(origin=v))
    resolution = property(lambda s: s._resolution)

    def _set_geometry(self, voxel_size=None, origin=None):
        if voxel_size is not None:
            self._voxel_size = float(voxel_size)
        if origin is not None:
            self._origin = np.asarray(origin, np.float32).reshape(3).copy()
        _lib.check(_lib.lib().cphb_occgrid_set_geometry(self._h, self._voxel_size, self._f3(self._origin)))

    def _sync_params(self):
        p = _lib.OccGridParams(self.clamping_thres_min, self.clamping_thres_max, self.prob_hit_log, self.prob_miss_log,
                               self.occ_prob_thres_log)
        _lib.check(_lib.lib().cphb_occgrid_set_params(self._h, C.byref(p)))

    def clear(self):
        _lib.check(_lib.lib().cphb_occgrid_clear(self._h, None))
        return self

    def insert(self, pointcloud, viewpoint, max_range=-1.0):
        """OccupancyGrid::Insert(pointcloud | points, viewpoint, max_range) (occupancygrid.cu:462-552)"""
        pts = pointcloud.points if isinstance(pointcloud, PointCloud) else Vector3fVector(pointcloud)
        self._sync_params()
        if pts is not None and len(pts):
            _lib.check(_lib.lib().cphb_occgrid_insert(self._h, pts.ptr, len(pts), self._f3(viewpoint), float(max_range), None))
        return self

    def add_voxel(self, voxel, occupied=False):
        self._sync_params()
        v = (C.c_int32 * 3)(*[int(x) for x in voxel])
        _lib.check(_lib.lib().cphb_occgrid_add_voxel(self._h, v, int(bool(occupied)), None))
        return self

    def add_voxels(self, voxels, occupied=False):
        self._sync_params()
        d = voxels if isinstance(voxels, DeviceArray) else DeviceArray.from_numpy(np.ascontiguousarray(voxels, np.int32).reshape(-1, 3), np.int32)
        if len(d):
            _lib.check(_lib.lib().cphb_occgrid_add_voxels(self._h, d.ptr, len(d), int(bool(occupied)), None))
        return self

    def set_free_area(self, min_bound, max_bound):
        self._sync_params()
        _lib.check(_lib.lib().cphb_occgrid_set_free_area(self._h, self._f3(min_bound), self._f3(max_bound), None))
        return self

    def _bounds(self):
        lo, hi = (C.c_int32 * 3)(), (C.c_int32 * 3)()
        _lib.check(_lib.lib().cphb_occgrid_bounds(self._h, lo, hi, None))
        return np.array(lo, np.int32), np.array(hi, np.int32)

    def get_min_bound(self):                  # occupancygrid.cu:317-322
        lo, _ = self._bounds()
        return ((lo - self._resolution // 2).astype(np.float32) * np.float32(self._voxel_size) + self._origin).astype(np.float32)

    def get_max_bound(self):                  # occupancygrid.cu:324-333
        _, hi = self._bounds()
        return ((hi - (self._resolution // 2 - 1)).astype(np.float32) * np.float32(self._voxel_size) + self._origin).astype(np.float32)

    def _extract(self, which):
        self._sync_params()
        cnt = C.c_size_t(0)
        _lib.check(_lib.lib().cphb_occgrid_extract(self._h, which, None, None, 0, C.byref(cnt), None))
        m = int(cnt.value)
        if m == 0:
            return np.zeros((0, 3), np.int32), np.zeros(0, np.float32)
        idx, pr = DeviceArray((m, 3), np.int32), DeviceArray((m,), np.float32)
        _lib.check(_lib.lib().cphb_occgrid_extract(self._h, which, idx.ptr, pr.ptr, m, C.byref(cnt), None))
        return idx.cpu(), pr.cpu()

    def extract_known_voxels(self):
        """-> (grid_index [m, 3] int32, prob_log [m] float32), bound-box order (ExtractKnownVoxels, occupancygrid.cu:380-388)"""
        return self._extract(0)

    def extract_free_voxels(self):
        return self._extract(1)

    def extract_occupied_voxels(self):
        return self._extract(2)

    @property
    def voxels(self):
        """the known voxels as OccupancyVoxel objects (pybind property, occupancygrid.cpp:98-101)"""
        idx, pr = self._extract(0)
        return [OccupancyVoxel(i, p) for i, p in zip(idx, pr)]

    def get_voxel(self, point):
        """-> (known, OccupancyVoxel)  (GetVoxel, occupancygrid.cu:351-356)"""
        k, p, gi = C.c_int(0), C.c_float(0), (C.c_int32 * 3)()
        _lib.check(_lib.lib().cphb_occgrid_get_voxel(self._h, self._f3(point), C.byref(k), C.byref(p), gi, None))
        return bool(k.value), OccupancyVoxel(list(gi), p.value)

    def is_occupied(self, point):             # occupancygrid.cu:335-341
        k, v = self.get_voxel(point)
        return bool(k and v.prob_log > self.occ_prob_thres_log)

    def is_unknown(self, point):              # occupancygrid.cu:343-348
        return not self.get_voxel(point)[0]

    def has_voxels(self):
        return True

    def to_torch(self):
        """zero-copy [res, res, res] float32 CUDA tensor of the log-odds (NaN = unknown)"""
        import torch
        r = self._resolution
        return torch.as_tensor(DeviceArray((r, r, r), np.float32, ptr=_lib.lib().cphb_occgrid_data(self._h), base=self), device="cuda")

    def __repr__(self):
        return "geometry::OccupancyGrid with %d voxels." % len(self._extract(0)[1])

    def __del__(self):
        try:
            if self._h:
                _lib.lib().cphb_stream_synchronize(None)
                _lib.lib().cphb_occgrid_destroy(self._h)
                self._h = None
        except Exception:
            pass


class DistanceVoxel:
    """geometry::DistanceVoxel (distancetransform.h:30-49; pybind distancetransform.cpp:34-53): nearest_index (3 uint16,
    the nearest site's grid cell) and distance (float32)."""

    def __init__(self, nearest_index=(0, 0, 0), distance=0.0):
        self.nearest_index = np.asarray(nearest_index, np.uint16)
        self.distance = float(np.float32(distance))

    def __repr__(self):
        return "geometry::DistanceVoxel with nearest_index: (%d, %d, %d), distance: %f)" % (*self.nearest_index.tolist(), self.distance)


class DistanceTransform:
    """geometry::DistanceTransform (distancetransform.h:51-78; pybind distancetransform.cpp:55-93): a dense res^3 grid of
    nearest sites and the Euclidean distances to them, on the device.  `voxel_size` and `origin` are plain attributes as
    in the reference; `resolution` is read-only (reconstruct changes it)."""

    def __init__(self, voxel_size=0.05, resolution=512, origin=(0.0, 0.0, 0.0), _handle=None):
        _lib.require_gpu()
        self._voxel_size, self._resolution = float(np.float32(voxel_size)), int(resolution)
        self._origin = np.asarray(origin, np.float32).reshape(3).copy()
        if _handle is not None:
            self._h = _handle
            return
        self._h = C.c_void_p()
        _lib.check(_lib.lib().cphb_dt_create(self._voxel_size, self._resolution, OccupancyGrid._f3(self._origin), None,
                                             C.byref(self._h)))

    voxel_size = property(lambda s: s._voxel_size, lambda s, v: s._set_geometry(voxel_size=v))
    origin = property(lambda s: s._origin, lambda s, v: s._set_geometry(origin=v))
    resolution = property(lambda s: s._resolution)

    def _set_geometry(self, voxel_size=None, origin=None):
        if voxel_size is not None:
            self._voxel_size = float(np.float32(voxel_size))
        if origin is not None:
            self._origin = np.asarray(origin, np.float32).reshape(3).copy()
        _lib.check(_lib.lib().cphb_dt_set_geometry(self._h, self._voxel_size, OccupancyGrid._f3(self._origin)))

    def reconstruct(self, voxel_size, resolution):
        """Reconstruct (densegrid.inl:128-134): the linear prefix of the old cells is kept, the rest are defaults"""
        _lib.check(_lib.lib().cphb_dt_reconstruct(self._h, float(voxel_size), int(resolution), None))
        self._voxel_size, self._resolution = float(np.float32(voxel_size)), int(resolution)
        return self

    def _compute(self, sites, with_distance):
        if isinstance(sites, VoxelGrid):
            keys = sites.voxels_keys
            rc = _lib.lib().cphb_dt_compute_voxel_grid(self._h, keys.ptr if keys is not None else None, len(sites),
                                                       float(sites.voxel_size), OccupancyGrid._f3(sites.origin),
                                                       int(with_distance), None)
            if rc == _lib.CPHB_ERR_INVALID:  # distancetransform.cu:331-337: logged, the grid is unchanged
                print("[cupoch_b200][error] %s" % _lib.lib().cphb_last_error().decode(errors="replace"), file=sys.stderr)
                return self
            _lib.check(rc)
            return self
        if not isinstance(sites, DeviceArray) and not hasattr(sites, "is_cuda"):
            sites = np.asarray(sites, np.int32).reshape(-1, 3)
        d = DeviceArray.wrap(sites, np.int32)
        _lib.check(_lib.lib().cphb_dt_compute_sites(self._h, d.ptr if len(d) else None, len(d), int(with_distance), None))
        return self

    def compute_edt(self, voxel_grid):
        """ComputeEDT(VoxelGrid | [n, 3] int32 grid cells) (distancetransform.cu:320-345)"""
        return self._compute(voxel_grid, True)

    def compute_voronoi_diagram(self, voxel_grid):
        """ComputeVoronoiDiagram(VoxelGrid | [n, 3] int32 grid cells): nearest sites only, every distance 0"""
        return self._compute(voxel_grid, False)

    def get_distances(self, points):
        """GetDistances (:421-435): host or device [n, 3] points -> device float32 [n]; 0 outside the grid or for NaN"""
        q = Vector3fVector(points)
        n = 0 if q is None else len(q)
        out = DeviceArray((n,), np.float32)
        if n:
            _lib.check(_lib.lib().cphb_dt_get_distances(self._h, q.ptr, n, out.ptr, None))
        return out

    def get_distance(self, point):
        """GetDistance (:411-419)"""
        return float(self.get_distances(np.asarray(point, np.float32).reshape(1, 3)).cpu()[0])

    def get_voxel(self, point):
        """-> (found, DistanceVoxel)  (DenseGrid::GetVoxel, densegrid.inl:148-155)"""
        f, nb, st, d = C.c_int(0), (C.c_int32 * 3)(), C.c_int(0), C.c_float(0)
        _lib.check(_lib.lib().cphb_dt_get_voxel(self._h, OccupancyGrid._f3(point), C.byref(f), nb, C.byref(st), C.byref(d), None))
        return bool(f.value), DistanceVoxel(list(nb), d.value)

    @staticmethod
    def create_from_occupancy_grid(occupancy_grid):
        """CreateFromOccupancyGrid (distancetransform_factory.cu:40-62), with the EDT of the occupied cells computed"""
        occupancy_grid._sync_params()
        h = C.c_void_p()
        _lib.check(_lib.lib().cphb_dt_from_occgrid(occupancy_grid._h, None, C.byref(h)))
        return DistanceTransform(occupancy_grid.voxel_size, occupancy_grid.resolution, occupancy_grid.origin, _handle=h)

    def to_torch(self):
        """zero-copy [res, res, res] float32 CUDA tensor of the distances"""
        import torch
        r = self._resolution
        return torch.as_tensor(DeviceArray((r, r, r), np.float32, ptr=_lib.lib().cphb_dt_distance_data(self._h), base=self), device="cuda")

    def __repr__(self):
        return "geometry::DistanceTransform with %d resolution." % self._resolution

    def __del__(self):
        try:
            if self._h:
                _lib.lib().cphb_stream_synchronize(None)
                _lib.lib().cphb_dt_destroy(self._h)
                self._h = None
        except Exception:
            pass


class KDTreeFlann:
    """knn::KDTreeFlann (kdtree_flann.h:43-124), exposed as cupoch.geometry.KDTreeFlann
    (kdtree_flann.cpp:93-95)."""

    def __init__(self, geometry=None):
        self._h = None
        self._n = 0
        if geometry is not None:
            self.set_geometry(geometry)

    def set_geometry(self, geometry):
        pts = geometry.points if isinstance(geometry, PointCloud) else Vector3fVector(geometry)
        self._release()
        n = 0 if pts is None else len(pts)
        h = C.c_void_p()
        _lib.require_gpu()
        _lib.check(_lib.lib().cphb_index_create(pts.ptr if n else None, n, None, C.byref(h)))
        self._h, self._n = h, n
        return True

    def _release(self):
        if self._h:
            _lib.lib().cphb_stream_synchronize(None)
            _lib.lib().cphb_index_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self._release()
        except Exception:
            pass

    # -- batch (device) API: KDTreeFlann::SearchKNN / SearchRadius on device vectors --------------
    def search_knn(self, query, knn):
        return self._search(query, knn, None)

    def search_radius(self, query, radius, max_nn):
        return self._search(query, max_nn, radius)

    search_hybrid = search_radius  # north_star's name (SURVEY.md section 0)

    def _search(self, query, k, radius):
        q = Vector3fVector(query)
        nq = 0 if q is None else len(q)
        if self._h is None or self._n == 0 or nq == 0 or k < 0 or (radius is None and k > NUM_MAX_NN):
            return -1, None, None  # kdtree_flann.cu:46-48,70-72
        idx = DeviceArray((nq, max(k, 1)), np.int32)
        d2 = DeviceArray((nq, max(k, 1)), np.float32)
        cnt = C.c_int64(0)
        L = _lib.lib()
        if radius is None:
            rc = L.cphb_search_knn(self._h, q.ptr, nq, k, idx.ptr, d2.ptr, C.byref(cnt), None)
        else:
            rc = L.cphb_search_radius(self._h, q.ptr, nq, float(radius), k, idx.ptr, d2.ptr, C.byref(cnt), None)
        if rc == -1:  # CPHB_ERR_INVALID == the reference's -1
            return -1, None, None
        _lib.check(rc)
        return int(cnt.value), idx, d2

    # -- single host query API (kdtree_flann.cpp:103-143) ---------------------------------------
    def search_vector_3f(self, query, search_param):
        if isinstance(search_param, KDTreeSearchParamKNN):
            return self.search_knn_vector_3f(query, search_param.knn)
        return self.search_radius_vector_3f(query, search_param.radius, search_param.max_nn)

    def search_knn_vector_3f(self, query, knn):
        k, idx, d2 = self.search_knn(np.asarray(query, np.float32).reshape(1, 3), knn)
        if k < 0:
            raise RuntimeError("search_knn_vector_3f() error!")
        return k, idx.cpu().reshape(-1), d2.cpu().reshape(-1)

    def search_radius_vector_3f(self, query, radius, max_nn):
        k, idx, d2 = self.search_radius(np.asarray(query, np.float32).reshape(1, 3), radius, max_nn)
        if k < 0:
            raise RuntimeError("search_radius_vector_3f() error!")
        return k, idx.cpu().reshape(-1), d2.cpu().reshape(-1)


from . import keypoint  # noqa: E402,F401  (cph.geometry.keypoint: the reference's submodule, keypoint.cpp:76-79)
