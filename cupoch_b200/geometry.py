"""cupoch.geometry mirror (hot-path subset): PointCloud, KDTreeFlann, KDTreeSearchParam*.

Names, argument meaning and error behaviour follow src/python/cupoch_pybind/geometry/
pointcloud.cpp and kdtree_flann.cpp; computation goes through the C ABI only.
"""
import ctypes as C
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


class VoxelGrid:
    """geometry::VoxelGrid (voxelgrid.h:84-160), the part SURVEY 8f ranks next: creation from a point cloud
    (voxelgrid_factory.cu:164-228) and the accessors that need nothing else.  voxels_keys / voxels_colors are
    device arrays ([m, 3] int32 grid indices in lexicographic order, [m, 3] float32 mean colours)."""

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
