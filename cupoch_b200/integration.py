"""cupoch.integration mirror: UniformTSDFVolume and ScalableTSDFVolume (integration/{uniform,scalable}_tsdfvolume.h;
pybind integration/integration.cpp).

The volume is a dense resolution^3 grid on the device, owned by a csrc/tsdf.cu handle: a {tsdf, weight} float pair per
voxel and colour planes only when the volume has colour.  Every operation runs there; nothing falls back to the CPU.
"""
import ctypes as C
import enum

import numpy as np

from . import _lib
from .geometry import PointCloud, TriangleMesh, VoxelGrid
from .utility import DeviceArray


class TSDFVolumeColorType(enum.IntEnum):
    """integration::TSDFVolumeColorType (tsdfvolume.h)"""
    NoColor = 0
    RGB8 = 1
    Gray32 = 2


def _m(a, n):
    return (C.c_float * n)(*np.asarray(a, np.float32).reshape(n).tolist())


class UniformTSDFVolume:
    """integration::UniformTSDFVolume(length, resolution, sdf_trunc, color_type, origin = 0): voxel_length = length /
    resolution, voxel k's centre origin + voxel_length (k - resolution / 2) + voxel_length / 2.  A resolution outside
    [2, 1290] or a length or sdf_trunc that is not positive and finite raises."""

    def __init__(self, length, resolution, sdf_trunc, color_type, origin=(0.0, 0.0, 0.0)):
        _lib.require_gpu()
        self._h = C.c_void_p()
        self._length, self._resolution = float(np.float32(length)), int(resolution)
        self._sdf_trunc, self._color_type = float(np.float32(sdf_trunc)), TSDFVolumeColorType(color_type)
        self._origin = np.asarray(origin, np.float32).reshape(3).copy()
        _lib.check(_lib.lib().cphb_tsdf_create(self._length, self._resolution, self._sdf_trunc, int(self._color_type),
                                               _m(self._origin, 3), None, C.byref(self._h)))

    length = property(lambda s: s._length)
    resolution = property(lambda s: s._resolution)
    sdf_trunc = property(lambda s: s._sdf_trunc)
    color_type = property(lambda s: s._color_type)
    origin = property(lambda s: s._origin.copy())
    voxel_length = property(lambda s: float(np.float32(s._length) / np.float32(s._resolution)))

    def __repr__(self):
        return "integration::UniformTSDFVolume " + ("without color." if self._color_type == TSDFVolumeColorType.NoColor
                                                   else "with color.")

    def __del__(self):
        try:
            if self._h:
                _lib.lib().cphb_stream_synchronize(None)
                _lib.lib().cphb_tsdf_destroy(self._h)
                self._h = None
        except Exception:
            pass

    def planes(self):
        """the device planes as borrowed views: tw [res^3, 2] float32 (tsdf, weight) and col [planes, res^3] float32 (3
        planes for RGB8, 1 for Gray32, whose channels are equal; None for NoColor), voxel idx = x res^2 + y res + z"""
        tw, col = C.c_void_p(), C.c_void_p()
        _lib.check(_lib.lib().cphb_tsdf_data(self._h, C.byref(tw), C.byref(col)))
        n = self._resolution ** 3
        planes = {TSDFVolumeColorType.NoColor: 0, TSDFVolumeColorType.RGB8: 3, TSDFVolumeColorType.Gray32: 1}[self._color_type]
        return (DeviceArray((n, 2), np.float32, ptr=tw.value, base=self),
                DeviceArray((planes, n), np.float32, ptr=col.value, base=self) if planes else None)

    def reset(self):
        """Reset: every voxel back to tsdf 0, weight 0, colour (1, 1, 1)"""
        _lib.check(_lib.lib().cphb_tsdf_reset(self._h, None))
        _lib.check(_lib.lib().cphb_stream_synchronize(None))

    def integrate(self, image, intrinsic, extrinsic):
        """Integrate(RGBDImage, intrinsic, extrinsic) (uniform_tsdfvolume.cu:670-701): extrinsic is world-to-camera.
        The depth must be 1-channel float32; RGB8 needs a uint8 RGB colour image and Gray32 a float32 intensity one;
        images that do not match the intrinsic's size raise."""
        d_color, d_depth = image._device()
        dep, col = image._depth_info(), image._color_info()
        _lib.check(_lib.lib().cphb_tsdf_integrate(self._h, d_depth.ptr, *dep, d_color.ptr, *col, int(intrinsic.width),
                                                  int(intrinsic.height), _m(intrinsic.intrinsic_matrix, 9), _m(extrinsic, 16), None))
        _lib.check(_lib.lib().cphb_stream_synchronize(None))

    def _sized(self, fn, *outs_of):
        n = C.c_size_t(0)
        _lib.check(fn(self._h, None, None, None, 0, C.byref(n), None))
        m = n.value
        outs = [DeviceArray((m, 3), dt) if want else None for want, dt in outs_of] if m else []
        if m:
            _lib.check(fn(self._h, *[o.ptr if o is not None else None for o in outs], m, C.byref(n), None))
        return m, outs

    def extract_point_cloud(self):
        """ExtractPointCloud (uniform_tsdfvolume.cu:85-156, 703-737): a point, normal and (with colour) colour per zero
        crossing between neighbouring band voxels, in (x, y, z, axis) order"""
        has_c = self._color_type != TSDFVolumeColorType.NoColor
        m, outs = self._sized(_lib.lib().cphb_tsdf_extract_points, (True, np.float32), (True, np.float32), (has_c, np.float32))
        pc = PointCloud()
        if m:
            pc._points, pc._normals, pc._colors = outs
        return pc

    def extract_triangle_mesh(self):
        """ExtractTriangleMesh (uniform_tsdfvolume.cu:184-350, 739-838), welded: one vertex per crossed grid edge of
        a valid cube (all 8 corner weights nonzero), in (x, y, z, axis) order of the edge's origin voxel, coloured
        unless NoColor; the triangles of each cube in cube index order, oriented so that their right-hand normals
        point from negative to positive tsdf (outwards)."""
        L = _lib.lib()
        has_c = self._color_type != TSDFVolumeColorType.NoColor
        nv, nt = C.c_size_t(0), C.c_size_t(0)
        _lib.check(L.cphb_tsdf_extract_mesh(self._h, None, None, None, 0, 0, C.byref(nv), C.byref(nt), None))
        mesh = TriangleMesh()
        if nv.value:
            v, t = DeviceArray((nv.value, 3), np.float32), DeviceArray((nt.value, 3), np.int32)
            c = DeviceArray((nv.value, 3), np.float32) if has_c else None
            _lib.check(L.cphb_tsdf_extract_mesh(self._h, v.ptr, c.ptr if c is not None else None, t.ptr, nv.value, nt.value,
                                                C.byref(nv), C.byref(nt), None))
            mesh._vertices, mesh._triangles, mesh._vertex_colors = v, t, c
        return mesh

    def extract_voxel_point_cloud(self):
        """ExtractVoxelPointCloud (uniform_tsdfvolume.cu:840-865): the centre of every band voxel, coloured (tsdf + 1) / 2"""
        m, outs = self._sized(_lib.lib().cphb_tsdf_extract_voxels, (False, np.int32), (True, np.float32), (True, np.float32))
        pc = PointCloud()
        if m:
            pc._points, pc._colors = outs[1], outs[2]
        return pc

    def extract_voxel_grid(self):
        """ExtractVoxelGrid (uniform_tsdfvolume.cu:867-895): every band voxel, key = its grid index (lexicographic order),
        colour (tsdf + 1) / 2; origin = origin - (resolution / 2) * voxel_length"""
        m, outs = self._sized(_lib.lib().cphb_tsdf_extract_voxels, (True, np.int32), (False, np.float32), (True, np.float32))
        vg = VoxelGrid()
        vl = np.float32(self._length) / np.float32(self._resolution)
        vg.voxel_size = float(vl)
        vg.origin = (self._origin - np.float32(self._resolution // 2) * vl).astype(np.float32)
        if m:
            vg.voxels_keys, vg.voxels_colors = outs[0], outs[2]
        return vg

    def raycast(self, intrinsic, extrinsic, sdf_trunc, project_valid_depth_only=True):
        """Raycast (uniform_tsdfvolume.cu:509-639, 924-951): one ray per pixel from the camera at extrinsic
        (world-to-camera), marched in steps of sdf_trunc / 2 from where it enters the grid; the surface point, normal and
        colour of each hit.  project_valid_depth_only: the hits in pixel order; otherwise one row per pixel, NaN for a
        miss."""
        w, h = int(intrinsic.width), int(intrinsic.height)
        npx = max(w, 0) * max(h, 0)
        outs = [DeviceArray((npx, 3), np.float32) for _ in range(3)] if npx else [None] * 3
        n = C.c_size_t(0)
        _lib.check(_lib.lib().cphb_tsdf_raycast(self._h, w, h, _m(intrinsic.intrinsic_matrix, 9), _m(extrinsic, 16), float(sdf_trunc),
                                                int(bool(project_valid_depth_only)), *[o.ptr if o else None for o in outs], npx,
                                                C.byref(n), None))
        m = n.value
        pc = PointCloud()
        if m:
            if m < npx:  # keep only the rows written, not the width x height buffers
                outs = [_copy_rows(o, m) for o in outs]
            pc._points, pc._normals, pc._colors = outs
        return pc


class ScalableTSDFVolume:
    """integration::ScalableTSDFVolume(voxel_length, sdf_trunc, color_type, depth_sampling_stride = 4, map_size = 1000):
    16^3-voxel units, unit length voxel_length * 16, allocated on the device near the surfaces each frame observes.
    map_size is the first capacity of the unit pool, which doubles as needed; it changes no result."""

    def __init__(self, voxel_length, sdf_trunc, color_type, depth_sampling_stride=4, map_size=1000):
        _lib.require_gpu()
        self._h = C.c_void_p()
        self._voxel_length, self._sdf_trunc = float(np.float32(voxel_length)), float(np.float32(sdf_trunc))
        self._color_type, self._stride = TSDFVolumeColorType(color_type), int(depth_sampling_stride)
        _lib.check(_lib.lib().cphb_stsdf_create(self._voxel_length, self._sdf_trunc, int(self._color_type), self._stride,
                                                int(map_size), None, C.byref(self._h)))

    voxel_length = property(lambda s: s._voxel_length)
    sdf_trunc = property(lambda s: s._sdf_trunc)
    color_type = property(lambda s: s._color_type)
    depth_sampling_stride = property(lambda s: s._stride)
    volume_unit_length = property(lambda s: float(np.float32(s._voxel_length) * np.float32(16)))

    def __repr__(self):
        return "integration::ScalableTSDFVolume " + ("without color." if self._color_type == TSDFVolumeColorType.NoColor
                                                    else "with color.")

    def __del__(self):
        try:
            if self._h:
                _lib.lib().cphb_stream_synchronize(None)
                _lib.lib().cphb_stsdf_destroy(self._h)
                self._h = None
        except Exception:
            pass

    def reset(self):
        """Reset: no unit is allocated"""
        _lib.check(_lib.lib().cphb_stsdf_reset(self._h, None))
        _lib.check(_lib.lib().cphb_stream_synchronize(None))

    def integrate(self, image, intrinsic, extrinsic):
        """Integrate(RGBDImage, intrinsic, extrinsic) (scalable_tsdfvolume.cu:311-343): allocates the units within
        sdf_trunc of the frame's strided depth points, then updates every allocated voxel.  The image rules of
        UniformTSDFVolume.integrate; a unit key outside [-2^20, 2^20) or a singular extrinsic raises, and a frame that
        raises leaves the volume unchanged."""
        d_color, d_depth = image._device()
        dep, col = image._depth_info(), image._color_info()
        _lib.check(_lib.lib().cphb_stsdf_integrate(self._h, d_depth.ptr, *dep, d_color.ptr, *col, int(intrinsic.width),
                                                   int(intrinsic.height), _m(intrinsic.intrinsic_matrix, 9), _m(extrinsic, 16), None))

    def info(self):
        """(allocated units, pool capacity in units, device bytes of the pool and its table)"""
        u, c, b = C.c_size_t(0), C.c_size_t(0), C.c_size_t(0)
        _lib.check(_lib.lib().cphb_stsdf_info(self._h, C.byref(u), C.byref(c), C.byref(b)))
        return u.value, c.value, b.value

    def units(self):
        """the device state as borrowed views: (keys [units] uint64 packed, tw [units, 4096, 2] float32, col [units,
        planes, 4096] float32 or None); key axis a = ((key >> (42 - 21 a)) & (2^21 - 1)) - 2^20"""
        n, keys, tw, col = C.c_size_t(0), C.c_void_p(), C.c_void_p(), C.c_void_p()
        _lib.check(_lib.lib().cphb_stsdf_data(self._h, C.byref(n), C.byref(keys), C.byref(tw), C.byref(col)))
        u = n.value
        if not u:
            return np.zeros(0, np.uint64), np.zeros((0, 4096, 2), np.float32), None
        planes = {TSDFVolumeColorType.NoColor: 0, TSDFVolumeColorType.RGB8: 3, TSDFVolumeColorType.Gray32: 1}[self._color_type]
        return (DeviceArray((u,), np.uint64, ptr=keys.value, base=self), DeviceArray((u, 4096, 2), np.float32, ptr=tw.value, base=self),
                DeviceArray((u, planes, 4096), np.float32, ptr=col.value, base=self) if planes else None)

    def extract_point_cloud(self):
        """ExtractPointCloud (scalable_tsdfvolume.cu:125-290, 345-366): a point, normal and (with colour) colour per zero
        crossing between a band voxel and its +1 neighbour, across unit faces, in (unit, voxel, axis) order"""
        L = _lib.lib()
        has_c = self._color_type != TSDFVolumeColorType.NoColor
        n = C.c_size_t(0)
        _lib.check(L.cphb_stsdf_extract_points(self._h, None, None, None, 0, C.byref(n), None))
        pc = PointCloud()
        m = n.value
        if m:
            p, nr = DeviceArray((m, 3), np.float32), DeviceArray((m, 3), np.float32)
            c = DeviceArray((m, 3), np.float32) if has_c else None
            _lib.check(L.cphb_stsdf_extract_points(self._h, p.ptr, nr.ptr, c.ptr if c is not None else None, m, C.byref(n), None))
            pc._points, pc._normals, pc._colors = p, nr, c
        return pc

    def extract_voxel_point_cloud(self):
        """ExtractVoxelPointCloud: the centre of every band voxel, coloured (tsdf + 1) / 2, in (unit, voxel) order"""
        L = _lib.lib()
        n = C.c_size_t(0)
        _lib.check(L.cphb_stsdf_extract_voxels(self._h, None, None, 0, C.byref(n), None))
        pc = PointCloud()
        m = n.value
        if m:
            p, c = DeviceArray((m, 3), np.float32), DeviceArray((m, 3), np.float32)
            _lib.check(L.cphb_stsdf_extract_voxels(self._h, p.ptr, c.ptr, m, C.byref(n), None))
            pc._points, pc._colors = p, c
        return pc

    def extract_triangle_mesh(self):
        """not implemented, as in the reference (scalable_tsdfvolume.cu:375-381)"""
        raise NotImplementedError("ScalableTSDFVolume::ExtractTriangleMesh is not implemented")


def _copy_rows(a, m):
    b = DeviceArray((m,) + a.shape[1:], a.dtype)
    _lib.check(_lib.lib().cphb_memcpy_d2d(b.ptr, a.ptr, m * a.nbytes // a.shape[0], None))
    _lib.check(_lib.lib().cphb_stream_synchronize(None))
    return b
