"""cupoch.collision mirror: compute_intersection between VoxelGrids, OccupancyGrids and Box / Sphere / Capsule primitives.

Names follow src/python/cupoch_pybind/collision/{collision,primitives}.cpp; the computation is one call of the C ABI
(cphb_compute_intersection).  In compute_intersection(a, b, margin) `a` is the target and `b` the query: each colliding
element of b gives one pair (smallest colliding index in a, index in b), in ascending query order.  An OccupancyGrid
element's index is its linear cell index x * res^2 + y * res + z; its cell (x, y, z) covers
origin + (x - resolution // 2) * voxel_size on every path.
"""
import copy
import ctypes as C
import sys

import numpy as np

from . import _lib
from .geometry import AxisAlignedBoundingBox, OccupancyGrid, VoxelGrid
from .utility import DeviceArray


class PrimitiveType:
    """collision::Primitive::PrimitiveType (primitives.h:37-44, without Mesh)"""
    Unspecified, Box, Sphere, Capsule, Cylinder = 0, 1, 2, 3, 4


class CollisionType:
    """CollisionResult::CollisionType (collision.h:48-54, without LineSet)"""
    Unspecified, Primitives, VoxelGrid, OccupancyGrid = 0, 1, 2, 3


def _m4(T):
    T = np.asarray(T, np.float32).reshape(4, 4).copy()
    return T


class Primitive:
    """collision::Primitive (primitives.h:36-66): `type` and the 4x4 `transform`"""

    def __init__(self, type=PrimitiveType.Unspecified, transform=None):
        self.type = type
        self.transform = _m4(np.eye(4) if transform is None else transform)

    def get_axis_aligned_bounding_box(self):
        return AxisAlignedBoundingBox()

    def _fields(self):
        return (0.0, 0.0, 0.0), 0.0, 0.0

    def _record(self):
        """this primitive as one cphb_primitive record"""
        lengths, radius, height = self._fields()
        return (int(self.type), _m4(self.transform).reshape(-1), np.asarray(lengths, np.float32).reshape(3), radius, height)

    def __repr__(self):
        return "collision::Primitive type %d" % self.type


def _origin(T):
    return np.asarray(T, np.float32)[:3, 3]


class Box(Primitive):
    """collision::Box(lengths, transform = I) (primitives.h:68-88)"""

    def __init__(self, lengths=(0.0, 0.0, 0.0), transform=None):
        super().__init__(PrimitiveType.Box, transform)
        self.lengths = np.asarray(lengths, np.float32).reshape(3).copy()

    def _fields(self):
        return self.lengths, 0.0, 0.0

    def get_axis_aligned_bounding_box(self):
        """primitives.h:79-85 as written: +-|R * lengths / 2| about the centre"""
        T = _m4(self.transform)
        ra = np.abs(T[:3, :3].astype(np.float32) @ (np.float32(0.5) * self.lengths))
        return AxisAlignedBoundingBox(_origin(T) - ra, _origin(T) + ra)


class Sphere(Primitive):
    """collision::Sphere(radius, center = 0) (primitives.h:90-110)"""

    def __init__(self, radius=0.0, center=None):
        super().__init__(PrimitiveType.Sphere)
        self.radius = float(np.float32(radius))
        if center is not None:
            self.transform[:3, 3] = np.asarray(center, np.float32).reshape(3)

    def _fields(self):
        return (0.0, 0.0, 0.0), self.radius, 0.0

    def get_axis_aligned_bounding_box(self):
        c, r = _origin(self.transform), np.float32(self.radius)
        return AxisAlignedBoundingBox(c - r, c + r)


class Capsule(Primitive):
    """collision::Capsule(radius, height, transform = I) (primitives.h:112-140): the segment of length height along the
    transform's third column, through its translation"""

    def __init__(self, radius=0.0, height=0.0, transform=None):
        super().__init__(PrimitiveType.Capsule, transform)
        self.radius, self.height = float(np.float32(radius)), float(np.float32(height))

    def _fields(self):
        return (0.0, 0.0, 0.0), self.radius, self.height

    def get_axis_aligned_bounding_box(self):
        T = _m4(self.transform)
        pa = T[:3, :3] @ np.array([0, 0, 0.5 * self.height], np.float32)
        r = np.float32(self.radius)
        return AxisAlignedBoundingBox(np.minimum(pa, -pa) - r + _origin(T), np.maximum(pa, -pa) + r + _origin(T))


class Cylinder(Primitive):
    """collision::Cylinder(radius, height, transform = I) (primitives.h:142-180).  It never collides: the reference's
    collision functors fall to their default branch for it."""

    def __init__(self, radius=0.0, height=0.0, transform=None):
        super().__init__(PrimitiveType.Cylinder, transform)
        self.radius, self.height = float(np.float32(radius)), float(np.float32(height))

    def _fields(self):
        return (0.0, 0.0, 0.0), self.radius, self.height

    def get_axis_aligned_bounding_box(self):
        """primitives.h:166-183 as written (its max bound takes the minimum of the two ends)"""
        T = _m4(self.transform)
        pa = T[:3, :3] @ np.array([0, 0, 0.5 * self.height], np.float32)
        pb = -pa
        a = pb - pa
        with np.errstate(invalid="ignore", divide="ignore"):
            e = np.float32(self.radius) * np.sqrt(np.float32(1) - (a * a) / np.dot(a, a))
        return AxisAlignedBoundingBox(np.minimum(pa - e, pb - e) + _origin(T), np.minimum(pa + e, pb + e) + _origin(T))


_RECORD = np.dtype([("type", np.int32), ("transform", np.float32, (16,)), ("lengths", np.float32, (3,)),
                    ("radius", np.float32), ("height", np.float32)])  # cphb_primitive
assert _RECORD.itemsize == C.sizeof(_lib.Primitive)


class PrimitiveArray:
    """collision::PrimitiveArray: primitives built on the host.  append copies the primitive, as the reference's
    device_vector push_back does; the array is uploaded once and again only after the next append."""

    def __init__(self, primitives=()):
        self._items, self._records, self._dev = [], [], None
        for p in primitives:
            self.append(p)

    def append(self, primitive):
        if not isinstance(primitive, Primitive):
            raise TypeError("PrimitiveArray.append needs a collision primitive")
        self._items.append(copy.deepcopy(primitive))
        self._records.append(primitive._record())
        self._dev = None
        return self

    def __len__(self):
        return len(self._items)

    def __getitem__(self, i):
        return self._items[i]

    def __iter__(self):
        return iter(self._items)

    def _device(self):
        if self._dev is None:
            self._dev = DeviceArray.from_numpy(np.array(self._records, _RECORD).view(np.uint8), np.uint8)
        return self._dev


class CollisionResult:
    """collision::CollisionResult (collision.h:47-75): `first` / `second` are the CollisionType of each argument,
    `collision_index_pairs` a device [m, 2] int32 array"""

    def __init__(self, first=CollisionType.Unspecified, second=CollisionType.Unspecified, pairs=None):
        self.first, self.second = first, second
        self.collision_index_pairs = pairs if pairs is not None else DeviceArray((0, 2), np.int32)

    def is_collided(self):
        return len(self.collision_index_pairs) > 0

    def get_collision_index_pairs(self):
        """host [m, 2] int32"""
        return self.collision_index_pairs.cpu()

    def get_first_collision_indices(self):
        """column 0 as it is (not deduplicated), int64 on the host"""
        return self.get_collision_index_pairs()[:, 0].astype(np.int64)

    def get_second_collision_indices(self):
        return self.get_collision_index_pairs()[:, 1].astype(np.int64)

    def __repr__(self):
        return "collision::CollisionResult with %d collisions." % len(self.collision_index_pairs)


def _operand(x, keep):
    op = _lib.CollOperand()
    if isinstance(x, VoxelGrid):
        op.kind = CollisionType.VoxelGrid
        n = len(x)
        op.n = n
        op.voxel_size = float(x.voxel_size)
        op.origin[:] = [float(v) for v in np.asarray(x.origin, np.float32).reshape(3)]
        if n:
            keys = DeviceArray.wrap(x.voxels_keys, np.int32)
            keep.append(keys)
            op.keys = keys.ptr
        return op, n == 0
    if isinstance(x, OccupancyGrid):
        x._sync_params()
        op.kind = CollisionType.OccupancyGrid
        op.occ = x._h
        return op, False
    if isinstance(x, PrimitiveArray):
        op.kind = CollisionType.Primitives
        op.n = len(x)
        if len(x):
            d = x._device()
            keep.append(d)
            op.primitives = d.ptr
        return op, len(x) == 0
    raise TypeError("compute_intersection: unsupported operand %s" % type(x).__name__)


def _log(level, msg):
    print("[cupoch_b200][%s] %s" % (level, msg), file=sys.stderr)


def compute_intersection(a, b, margin=0.0):
    """collision::ComputeIntersection(a, b, margin) (collision.cu:1137-1231) for VoxelGrid x VoxelGrid, VoxelGrid x
    OccupancyGrid (both orders), VoxelGrid x PrimitiveArray (both orders) and OccupancyGrid x PrimitiveArray (both
    orders).  Invalid arguments (a non-finite margin, a voxel size that is not positive and finite, VoxelGrid target
    keys spanning 2^21 or more on an axis) are logged and give an empty result."""
    _lib.require_gpu()
    keep = []
    oa, ea = _operand(a, keep)
    ob, eb = _operand(b, keep)
    out = CollisionResult(oa.kind, ob.kind)
    if oa.kind == ob.kind and oa.kind in (CollisionType.Primitives, CollisionType.OccupancyGrid):
        raise TypeError("compute_intersection: no overload for (%s, %s)" % (type(a).__name__, type(b).__name__))
    L = _lib.lib()
    cnt = C.c_size_t(0)
    # at most one pair per query element: a VoxelGrid or primitive query is answered in one call, an OccupancyGrid
    # query (whose element count is not known up front) is sized first
    cap = 0 if ob.kind == CollisionType.OccupancyGrid else int(ob.n)
    pairs = DeviceArray((max(cap, 1), 2), np.int32)
    rc = L.cphb_compute_intersection(C.byref(oa), C.byref(ob), float(margin), pairs.ptr if cap else None, cap, C.byref(cnt), None)
    if rc == _lib.CPHB_ERR_INVALID:
        _log("error", L.cphb_last_error().decode(errors="replace"))
        return out
    _lib.check(rc)
    if ea or eb:
        _log("warning", "[Intersection::Compute] target or query is empty.")
        return out
    m = int(cnt.value)
    if m and not cap:
        pairs = DeviceArray((m, 2), np.int32)
        _lib.check(L.cphb_compute_intersection(C.byref(oa), C.byref(ob), float(margin), pairs.ptr, m, C.byref(cnt), None))
    if m:
        out.collision_index_pairs = DeviceArray((m, 2), np.int32, ptr=pairs.ptr, base=pairs)
    return out
