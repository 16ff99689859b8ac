"""ctypes loader for the CPU oracle (oracle/oracle.c).

TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__.smoke() and
bench.py's cpu_baseline / --impl reference legs.  The product package
cupoch_b200/ must never import this module.  The library is built by
oracle.build() (oracle/__init__.py).
"""
import ctypes as C

import numpy as np

from . import build as _build, load, ptr as _p

P2P, P2PLANE, SYMMETRIC, COLORED, GICP = 1, 2, 3, 4, 5


def build(force=False):
    return _build("oracle", force)


class IcpResult(C.Structure):
    _fields_ = [("transformation", C.c_float * 16), ("fitness", C.c_float), ("inlier_rmse", C.c_float),
                ("n_corr", C.c_int), ("iterations", C.c_int)]


class IcpParams(C.Structure):
    _fields_ = [("kind", C.c_int), ("max_distance", C.c_float), ("relative_fitness", C.c_float),
                ("relative_rmse", C.c_float), ("max_iteration", C.c_int), ("det_thresh", C.c_float),
                ("lambda_geometric", C.c_float), ("use_kdtree", C.c_int)]


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = load("oracle")
        _lib.orc_search_bruteforce.restype = C.c_long
        _lib.orc_kdtree_build.restype = C.c_void_p
        _lib.orc_kdtree_search.restype = C.c_long
        _lib.orc_kdtree_search.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_void_p, C.c_void_p]
        _lib.orc_kdtree_free.argtypes = [C.c_void_p]
    return _lib


def _f(a):
    return None if a is None else np.ascontiguousarray(a, dtype=np.float32)


def search(tgt, qry, k, radius=-1.0, kdtree=False):
    """-> (idx[n,k] int32, d2[n,k] float32, count)"""
    tgt, qry = _f(tgt).reshape(-1, 3), _f(qry).reshape(-1, 3)
    n = len(qry)
    idx = np.empty((n, k), np.int32)
    d2 = np.empty((n, k), np.float32)
    L = lib()
    if kdtree:
        t = L.orc_kdtree_build(_p(tgt), C.c_int(len(tgt)))
        cnt = L.orc_kdtree_search(t, _p(qry), n, k, C.c_float(radius), _p(idx), _p(d2))
        L.orc_kdtree_free(t)
    else:
        cnt = L.orc_search_bruteforce(_p(tgt), C.c_int(len(tgt)), _p(qry), C.c_int(n), C.c_int(k),
                                      C.c_float(radius), _p(idx), _p(d2))
    return idx, d2, int(cnt)


class KDTree:
    def __init__(self, tgt):
        self.tgt = _f(tgt).reshape(-1, 3)
        self.h = lib().orc_kdtree_build(_p(self.tgt), C.c_int(len(self.tgt)))

    def search(self, qry, k, radius=-1.0):
        qry = _f(qry).reshape(-1, 3)
        n = len(qry)
        idx = np.empty((n, k), np.int32)
        d2 = np.empty((n, k), np.float32)
        cnt = lib().orc_kdtree_search(self.h, _p(qry), n, k, C.c_float(radius), _p(idx), _p(d2))
        return idx, d2, int(cnt)

    def __del__(self):
        if getattr(self, "h", None):
            lib().orc_kdtree_free(self.h)
            self.h = None


def transform_points(p, T):
    p = _f(p).reshape(-1, 3).copy()
    T = _f(T).reshape(16)
    lib().orc_transform_points(_p(p), C.c_int(len(p)), _p(T))
    return p


def transform_normals(p, T):
    p = _f(p).reshape(-1, 3).copy()
    T = _f(T).reshape(16)
    lib().orc_transform_normals(_p(p), C.c_int(len(p)), _p(T))
    return p


def rotate_covariances(c, T):
    c = _f(c).reshape(-1, 9).copy()
    T = _f(T).reshape(16)
    lib().orc_rotate_covariances(_p(c), C.c_int(len(c)), _p(T))
    return c.reshape(-1, 3, 3)


def min_bound(p):
    p = _f(p).reshape(-1, 3)
    o = np.zeros(3, np.float32)
    lib().orc_min_bound(_p(p), C.c_int(len(p)), _p(o))
    return o


def max_bound(p):
    p = _f(p).reshape(-1, 3)
    o = np.zeros(3, np.float32)
    lib().orc_max_bound(_p(p), C.c_int(len(p)), _p(o))
    return o


def voxel_down_sample(pts, voxel, normals=None, colors=None, origin=None):
    """origin=None: the reference's grid origin (min_bound - voxel/2); else a caller-supplied common origin"""
    pts, normals, colors = _f(pts).reshape(-1, 3), _f(normals), _f(colors)
    n = len(pts)
    op = np.empty((n, 3), np.float32)
    on = np.empty((n, 3), np.float32) if normals is not None else None
    oc = np.empty((n, 3), np.float32) if colors is not None else None
    org = None if origin is None else _f(origin).reshape(3)
    m = lib().orc_voxel_down_sample_origin(_p(pts), _p(normals), _p(colors), C.c_int(n), C.c_float(voxel), _p(org), _p(op),
                                           _p(on), _p(oc))
    return op[:m].copy(), (on[:m].copy() if on is not None else None), (oc[:m].copy() if oc is not None else None)


def estimate_normals(pts, knn=30, radius=0.0, max_nn=0):
    pts = _f(pts).reshape(-1, 3)
    out = np.empty_like(pts)
    lib().orc_estimate_normals(_p(pts), C.c_int(len(pts)), C.c_int(knn), C.c_float(radius), C.c_int(max_nn), _p(out))
    return out


def voxel_grid_from_point_cloud(pts, voxel, lo=None, hi=None, colors=None):
    """VoxelGrid::CreateFromPointCloud[WithinBounds] (voxelgrid_factory.cu:164-228) -> (keys[m,3] int32, colors[m,3],
    origin[3])"""
    pts = _f(pts).reshape(-1, 3)
    v = np.float32(voxel)
    if lo is None:  # CreateFromPointCloud: bounds of the cloud widened by half a voxel (:221-228)
        lo = (min_bound(pts) - v * np.float32(0.5)).astype(np.float32)
        hi = (max_bound(pts) + v * np.float32(0.5)).astype(np.float32)
    mn, mx = _f(lo).reshape(3), _f(hi).reshape(3)
    col = None if colors is None else _f(colors).reshape(-1, 3)
    keys = np.empty((len(pts), 3), np.int32)
    out = np.empty((len(pts), 3), np.float32)
    m = lib().orc_voxel_grid_from_point_cloud(_p(pts), _p(col), C.c_int(len(pts)), C.c_float(voxel), _p(mn), _p(mx),
                                              _p(keys), _p(out))
    return keys[:m].copy(), out[:m].copy(), mn.copy()


def gaussian_filter(pts, radius, sigma2, max_nn=50, normals=None, colors=None):
    """PointCloud::GaussianFilter (pointcloud.cu:387-433) -> (points, normals or None, colors or None); empty arrays
    for illegal parameters"""
    pts = _f(pts).reshape(-1, 3)
    nrm = None if normals is None else _f(normals).reshape(-1, 3)
    col = None if colors is None else _f(colors).reshape(-1, 3)
    op = np.empty_like(pts)
    on = None if nrm is None else np.empty_like(pts)
    oc = None if col is None else np.empty_like(pts)
    m = lib().orc_gaussian_filter(_p(pts), _p(nrm), _p(col), C.c_int(len(pts)), C.c_float(radius), C.c_float(sigma2),
                                  C.c_int(max_nn), _p(op), _p(on), _p(oc))
    cut = (lambda a: None if a is None else a[:m])
    return cut(op), cut(on), cut(oc)


def remove_radius_outliers(pts, nb_points, radius):
    """-> ascending indices of the kept points (down_sample.cu:317-354)"""
    pts = _f(pts).reshape(-1, 3)
    out = np.empty(len(pts), np.int32)
    m = lib().orc_remove_radius_outliers(_p(pts), C.c_int(len(pts)), C.c_int(nb_points), C.c_float(radius), _p(out))
    return out[:m].copy()


def remove_statistical_outliers(pts, nb_neighbors, std_ratio):
    """-> (ascending kept indices, per-point mean squared neighbour distance, (mean, std, threshold))
    (down_sample.cu:356-438)"""
    pts = _f(pts).reshape(-1, 3)
    out = np.empty(len(pts), np.int32)
    avg = np.empty(len(pts), np.float32)
    stats = np.zeros(3, np.float32)
    m = lib().orc_remove_statistical_outliers(_p(pts), C.c_int(len(pts)), C.c_int(nb_neighbors), C.c_float(std_ratio),
                                              _p(out), _p(avg), _p(stats))
    return out[:m].copy(), avg, stats


def normals_from_neighbors(pts, nbr):
    pts = _f(pts).reshape(-1, 3)
    nbr = np.ascontiguousarray(nbr, np.int32)
    out = np.empty_like(pts)
    lib().orc_normals_from_neighbors(_p(pts), C.c_int(len(pts)), _p(nbr), C.c_int(nbr.shape[1]), _p(out))
    return out


def covariances_from_normals(nrm, eps=1e-3):
    nrm = _f(nrm).reshape(-1, 3)
    out = np.empty((len(nrm), 9), np.float32)
    lib().orc_covariances_from_normals(_p(nrm), C.c_int(len(nrm)), C.c_float(eps), _p(out))
    return out.reshape(-1, 3, 3)


def color_gradient(pts, nrm, col, nbr):
    pts, nrm, col = _f(pts).reshape(-1, 3), _f(nrm).reshape(-1, 3), _f(col).reshape(-1, 3)
    nbr = np.ascontiguousarray(nbr, np.int32)
    out = np.empty_like(pts)
    lib().orc_color_gradient(_p(pts), _p(nrm), _p(col), C.c_int(len(pts)), _p(nbr), C.c_int(nbr.shape[1]), _p(out))
    return out


def jtj_jtr(kind, src, tgt, corr, src_nrm=None, src_col=None, src_cov=None, tgt_nrm=None, tgt_col=None,
            tgt_grad=None, tgt_cov=None, lambda_geometric=0.968):
    a = [_f(x) for x in (src, src_nrm, src_col, src_cov, tgt, tgt_nrm, tgt_col, tgt_grad, tgt_cov)]
    corr = np.ascontiguousarray(corr, np.int32).reshape(-1, 2)
    sums = np.zeros(32, np.float64)
    lib().orc_jtj_jtr(C.c_int(kind), *[_p(x) for x in a], _p(corr), C.c_int(len(corr)),
                      C.c_float(lambda_geometric), _p(sums))
    return sums


def solve_jtj(jtj21, jtr, det_thresh=1e-6):
    u, b = _f(jtj21).reshape(21), _f(jtr).reshape(6)
    T = np.zeros(16, np.float32)
    ok = lib().orc_solve_jtj(_p(u), _p(b), C.c_float(det_thresh), _p(T))
    return bool(ok), T.reshape(4, 4)


def kabsch(src, tgt, corr, n_model=None):
    src, tgt = _f(src).reshape(-1, 3), _f(tgt).reshape(-1, 3)
    corr = np.ascontiguousarray(corr, np.int32).reshape(-1, 2)
    S = np.zeros(17, np.float64)
    lib().orc_kabsch_sums(_p(src), _p(tgt), _p(corr), C.c_int(len(corr)), _p(S))
    T = np.zeros(16, np.float32)
    lib().orc_kabsch_from_sums(_p(S), C.c_int(len(src) if n_model is None else n_model), _p(T))
    return T.reshape(4, 4), S


def jtj_rows(J, r):
    """utility::ComputeJTJandJTr<.., NumJ> on explicit rows J [n, num_j, 6], r [n, num_j] -> 32 float64 sums"""
    J = np.ascontiguousarray(J, np.float32)
    r = np.ascontiguousarray(r, np.float32).reshape(J.shape[0], -1)
    sums = np.zeros(32, np.float64)
    lib().orc_jtj_rows(_p(J), _p(r), C.c_int(J.shape[0]), C.c_int(r.shape[1]), _p(sums))
    return sums


def weighted_jtj_rows(J, r, sigma2, nu):
    """utility::ComputeWeightedJTJandJTr with the odometry's Student-t weights -> (32 float64 sums, w_sum)"""
    J = np.ascontiguousarray(J, np.float32)
    r = np.ascontiguousarray(r, np.float32).reshape(J.shape[0], -1)
    sums = np.zeros(32, np.float64)
    lib().orc_weighted_jtj_rows.restype = C.c_float
    w = lib().orc_weighted_jtj_rows(_p(J), _p(r), C.c_int(J.shape[0]), C.c_int(r.shape[1]), C.c_float(sigma2), C.c_float(nu), _p(sums))
    return sums, float(w)


def kabsch_weighted(model, target, weight):
    model, target, weight = _f(model).reshape(-1, 3), _f(target).reshape(-1, 3), _f(weight).reshape(-1)
    T = np.zeros(16, np.float32)
    lib().orc_kabsch_weighted(_p(model), _p(target), _p(weight), C.c_int(len(model)), _p(T))
    return T.reshape(4, 4)


def compute_fpfh_feature(pts, nrm, knn=0, radius=0.0, max_nn=0):
    pts, nrm = _f(pts).reshape(-1, 3), _f(nrm).reshape(-1, 3)
    out = np.zeros((len(pts), 33), np.float32)
    lib().orc_compute_fpfh_feature(_p(pts), _p(nrm), C.c_int(len(pts)), C.c_int(knn), C.c_float(radius), C.c_int(max_nn), _p(out))
    return out


def cluster_dbscan(pts, eps, min_points, max_edges=100):
    pts = _f(pts).reshape(-1, 3)
    labels = np.empty(len(pts), np.int32)
    n = lib().orc_cluster_dbscan(_p(pts), C.c_int(len(pts)), C.c_float(eps), C.c_int(min_points), C.c_int(max_edges), _p(labels))
    return labels, int(n)


def correspondences(src, tgt, max_distance, kdtree=True):
    src, tgt = _f(src).reshape(-1, 3), _f(tgt).reshape(-1, 3)
    n = len(src)
    corr = np.empty((n, 2), np.int32)
    nc, fit, rmse = C.c_int(0), C.c_float(0), C.c_float(0)
    kd = lib().orc_kdtree_build(_p(tgt), C.c_int(len(tgt))) if kdtree else None
    lib().orc_correspondences(_p(src), C.c_int(n), _p(tgt), C.c_int(len(tgt)), C.c_void_p(kd), C.c_float(max_distance),
                              _p(corr), C.byref(nc), C.byref(fit), C.byref(rmse))
    if kd:
        lib().orc_kdtree_free(kd)
    return corr[:nc.value].copy(), fit.value, rmse.value


def registration_icp(kind, src, tgt, max_distance, init=None, src_nrm=None, src_col=None, src_cov=None,
                     tgt_nrm=None, tgt_col=None, tgt_grad=None, tgt_cov=None, relative_fitness=1e-6,
                     relative_rmse=1e-6, max_iteration=30, det_thresh=1e-6, lambda_geometric=0.968,
                     use_kdtree=True, trace=False):
    src, tgt = _f(src).reshape(-1, 3), _f(tgt).reshape(-1, 3)
    n, m = len(src), len(tgt)
    init = np.eye(4, dtype=np.float32) if init is None else _f(init).reshape(4, 4)
    prm = IcpParams(kind, max_distance, relative_fitness, relative_rmse, max_iteration, det_thresh,
                    lambda_geometric, 1 if use_kdtree else 0)
    res = IcpResult()
    corr = np.empty((max(n, 1), 2), np.int32)
    tr = np.zeros((max_iteration + 1, 16), np.float32) if trace else None
    a = [_f(x) for x in (src_nrm, src_col, src_cov)]
    b = [_f(x) for x in (tgt_nrm, tgt_col, tgt_grad, tgt_cov)]
    lib().orc_registration_icp(_p(src), _p(a[0]), _p(a[1]), _p(a[2]), C.c_int(n), _p(tgt), _p(b[0]), _p(b[1]),
                               _p(b[2]), _p(b[3]), C.c_int(m), _p(init.reshape(16)), C.byref(prm), C.byref(res),
                               _p(corr), _p(tr))
    out = {
        "transformation": np.array(res.transformation, np.float32).reshape(4, 4),
        "fitness": res.fitness, "inlier_rmse": res.inlier_rmse,
        "correspondence_set": corr[:res.n_corr].copy(), "iterations": res.iterations,
    }
    if trace:
        out["trace"] = tr[:res.iterations + 1].reshape(-1, 4, 4)
    return out


def num_threads():
    return int(lib().orc_num_threads())



class OccupancyGrid:
    """geometry::OccupancyGrid (occupancygrid.h / occupancygrid.cu) restated on numpy arrays: prob[res^3] float32 (NaN =
    unknown), has_index[res^3] uint8, bounds u16[6] = (min_bound_, max_bound_)."""

    def __init__(self, voxel_size=0.05, resolution=512, origin=(0, 0, 0)):
        self.voxel_size, self.resolution = float(voxel_size), int(resolution)
        self.origin = np.asarray(origin, np.float32).reshape(3).copy()
        self.clamping_thres_min, self.clamping_thres_max = -2.0, 3.5
        self.prob_hit_log, self.prob_miss_log, self.occ_prob_thres_log = 0.85, -0.4, 0.0
        n = self.resolution ** 3
        self.prob = np.full(n, np.nan, np.float32)
        self.has_index = np.zeros(n, np.uint8)
        self._stamp = np.zeros(n, np.uint8)
        h = self.resolution // 2
        self.bounds = np.array([h, h, h, h, h, h], np.uint16)

    def _params(self):
        return np.array([self.clamping_thres_min, self.clamping_thres_max, self.prob_hit_log, self.prob_miss_log], np.float32)

    def add_voxels(self, voxels, occupied=False):
        v = np.ascontiguousarray(voxels, np.int32).reshape(-1, 3)
        lib().orc_occgrid_add_voxels(_p(self.prob), _p(self.has_index), _p(self.bounds), C.c_int(self.resolution),
                                     _p(self._params()), _p(v), C.c_int(len(v)), C.c_int(int(occupied)))
        return self

    def insert(self, points, viewpoint, max_range=-1.0, ref_rule=False):
        """ref_rule: walk with the reference's half-voxel boundary instead of the library's (DESIGN §4 item 27)"""
        pts = _f(points).reshape(-1, 3)
        vp = np.asarray(viewpoint, np.float32).reshape(3)
        lib().orc_occgrid_insert(_p(self.prob), _p(self.has_index), _p(self._stamp), _p(self.bounds), C.c_int(self.resolution),
                                 C.c_float(self.voxel_size), _p(self.origin), _p(self._params()), _p(pts), C.c_int(len(pts)),
                                 _p(vp), C.c_float(max_range), C.c_int(int(bool(ref_rule))))
        return self

    def set_free_area(self, min_bound, max_bound):
        lo, hi = np.asarray(min_bound, np.float32).reshape(3), np.asarray(max_bound, np.float32).reshape(3)
        lib().orc_occgrid_set_free_area(_p(self.prob), _p(self.bounds), C.c_int(self.resolution), C.c_float(self.voxel_size),
                                        _p(self.origin), C.c_float(self.prob_miss_log), _p(lo), _p(hi))
        return self

    def extract(self, which):
        """which: 0 known, 1 free, 2 occupied -> (grid_index [m,3] int32, prob_log [m])"""
        b = self.bounds.astype(np.int64)
        cap = int(np.prod(b[3:] - b[:3] + 1))
        idx, pr = np.empty((max(cap, 1), 3), np.int32), np.empty(max(cap, 1), np.float32)
        lib().orc_occgrid_extract.restype = C.c_int
        m = lib().orc_occgrid_extract(_p(self.prob), _p(self.has_index), _p(self.bounds), C.c_int(self.resolution),
                                      C.c_float(self.occ_prob_thres_log), C.c_int(which), _p(idx), _p(pr))
        return idx[:m].copy(), pr[:m].copy()

    def voxel_index(self, point):
        lib().orc_occgrid_voxel_index.restype = C.c_long
        return int(lib().orc_occgrid_voxel_index(C.c_int(self.resolution), C.c_float(self.voxel_size), _p(self.origin),
                                                 _p(np.asarray(point, np.float32).reshape(3))))

    def get_voxel(self, point):
        """-> (known, prob_log)"""
        i = self.voxel_index(point)
        if i < 0:
            return False, float("nan")
        return bool(not np.isnan(self.prob[i])), float(self.prob[i])

    def get_min_bound(self):
        h = self.resolution // 2
        return ((self.bounds[:3].astype(np.int32) - h).astype(np.float32) * np.float32(self.voxel_size) + self.origin).astype(np.float32)

    def get_max_bound(self):
        h = self.resolution // 2
        return ((self.bounds[3:].astype(np.int32) - (h - 1)).astype(np.float32) * np.float32(self.voxel_size) + self.origin).astype(np.float32)
