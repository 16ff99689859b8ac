"""CPU: the collision restatement (oracle/collision.c) -- the checker of csrc/collision.cu.

- The reference's TEST(Collision, VoxelVoxel) known answer (tests/golden/collision_known.json).
- Sphere, box and capsule tests against float64 closed forms away from ties: squared distance to the box, the
  separating-axis test in numpy, segment-to-box distance by dense sampling.
- At margin 0 cells that share a face or an edge collide and separated cells do not.
- The deliberate deviations of DESIGN.md section 4 item 16: smallest target index, no candidate cap, the margin in both
  argument orders, one placement for OccupancyGrid cells, exact ties at powers of two."""
import json
import os

import numpy as np
import pytest

from oracle import collision_py as OC

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "collision_known.json")


def rot(axis, ang):
    """4x4 rotation about a unit axis (float64)"""
    a = np.asarray(axis, np.float64)
    a = a / np.linalg.norm(a)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    T = np.eye(4)
    T[:3, :3] = np.eye(3) + np.sin(ang) * K + (1 - np.cos(ang)) * K @ K
    return T


def moved(T, t):
    T = np.array(T, np.float64)
    T[:3, 3] = t
    return T


def random_prims(rng, n, span, vs, kinds=(OC.BOX, OC.SPHERE, OC.CAPSULE, OC.CYLINDER)):
    """n random primitives of the given kinds inside [0, span]^3, sizes of a few voxels"""
    out = []
    for i in range(n):
        k = kinds[i % len(kinds)]
        T = moved(rot(rng.normal(size=3), rng.uniform(0, np.pi)), rng.uniform(0, span, 3))
        out.append(OC.prim(k, T, lengths=rng.uniform(0.5, 6, 3) * vs, radius=rng.uniform(0.3, 3) * vs,
                           height=rng.uniform(0, 6) * vs))
    return out


def cell_box(key, vs, o):
    c = (np.asarray(key, np.float64) + 0.5) * vs + np.asarray(o, np.float64)
    return c - vs / 2, c + vs / 2


def test_known_answer_voxel_voxel():
    g = json.load(open(GOLD))
    for step in g["steps"]:
        a = OC.voxel_grid(np.asarray(step["keys1"], np.int32).reshape(-1, 3), g["voxel_size"], g["origin"])
        b = OC.voxel_grid(np.asarray(step["keys2"], np.int32).reshape(-1, 3), g["voxel_size"], g["origin"])
        pairs = OC.compute(a, b, 0.0)
        assert (len(pairs) > 0) == step["collided"]
        if "pairs" in step:
            assert pairs.tolist() == step["pairs"]


def test_sphere_matches_float64_distance():
    rng = np.random.default_rng(1)
    vs, o = 0.25, np.array([0.3, -0.2, 0.1])
    checked = 0
    for _ in range(4000):
        c, r, key = rng.uniform(-2, 2, 3), rng.uniform(0.05, 1.0), rng.integers(-8, 8, 3)
        lo, hi = cell_box(key, vs, o)
        d2 = float(np.sum(np.maximum(0, np.maximum(lo - c, c - hi)) ** 2))
        if abs(d2 - r * r) < 1e-4:
            continue
        assert OC.prim_elem(OC.prim(OC.SPHERE, moved(np.eye(4), c), radius=r), key, vs, o) == (d2 <= r * r)
        checked += 1
    assert checked > 3500


def sat64(e1, R, c1, e2, c2):
    """intersection_test.inl:153-209 in float64 with rot2 = I; returns (collides, smallest slack of the 15 tests)"""
    r, t = R, R @ (c2 - c1)
    ar = np.abs(r) + np.finfo(np.float32).eps
    sl = []
    for i in range(3):
        sl.append(e1[i] + ar[i] @ e2 - abs(t[i]))
    for i in range(3):
        sl.append(ar[:, i] @ e1 + e2[i] - abs(t @ r[:, i]))
    cross = [
        (e1[1] * ar[2, 0] + e1[2] * ar[1, 0], e2[1] * ar[0, 2] + e2[2] * ar[0, 1], t[2] * r[1, 0] - t[1] * r[2, 0]),
        (e1[1] * ar[2, 1] + e1[2] * ar[1, 1], e2[0] * ar[0, 2] + e2[2] * ar[0, 0], t[2] * r[1, 1] - t[1] * r[2, 1]),
        (e1[1] * ar[2, 2] + e1[2] * ar[1, 2], e2[0] * ar[0, 1] + e2[1] * ar[0, 0], t[2] * r[1, 2] - t[1] * r[2, 2]),
        (e1[0] * ar[2, 0] + e1[2] * ar[0, 0], e2[1] * ar[1, 2] + e2[2] * ar[1, 1], t[0] * r[2, 0] - t[2] * r[0, 0]),
        (e1[0] * ar[2, 1] + e1[2] * ar[0, 1], e2[0] * ar[1, 2] + e2[2] * ar[1, 0], t[0] * r[2, 1] - t[2] * r[0, 1]),
        (e1[0] * ar[2, 2] + e1[2] * ar[0, 2], e2[0] * ar[1, 1] + e2[1] * ar[1, 0], t[0] * r[2, 2] - t[2] * r[0, 2]),
        (e1[0] * ar[1, 0] + e1[1] * ar[0, 0], e2[1] * ar[2, 2] + e2[2] * ar[2, 1], t[1] * r[0, 1] - t[0] * r[1, 0]),
        (e1[0] * ar[1, 1] + e1[1] * ar[0, 1], e2[0] * ar[2, 2] + e2[2] * ar[2, 0], t[1] * r[0, 1] - t[0] * r[1, 1]),
        (e1[0] * ar[1, 2] + e1[1] * ar[0, 2], e2[0] * ar[2, 1] + e2[1] * ar[2, 0], t[1] * r[0, 2] - t[0] * r[1, 2]),
    ]
    for ra, rb, v in cross:
        sl.append(ra + rb - abs(v))
    return min(sl) >= 0, min(sl)


def test_box_matches_float64_separating_axes():
    rng = np.random.default_rng(2)
    vs, o = 0.5, np.array([0.1, 0.2, -0.3])
    checked = 0
    for i in range(4000):
        T = moved(rot(rng.normal(size=3), rng.uniform(0, np.pi)) if i % 4 else np.eye(4), rng.uniform(-2, 2, 3))
        L, key, margin = rng.uniform(0.1, 2, 3), rng.integers(-6, 6, 3), [0.0, 0.1][i % 2]
        c2 = (key + 0.5) * vs + o
        hit, slack = sat64(L / 2, T[:3, :3], T[:3, 3], np.full(3, vs / 2 + margin), c2)
        if abs(slack) < 1e-4:
            continue
        p = OC.prim(OC.BOX, T, lengths=L)
        assert OC.prim_elem(p, key, vs, o, margin) == hit
        if i % 4 == 0:  # axis-aligned: the boxes overlap
            lo, hi = cell_box(key, vs, o)
            assert hit == bool(np.all(T[:3, 3] - L / 2 <= hi + margin) and np.all(T[:3, 3] + L / 2 >= lo - margin))
        checked += 1
    assert checked > 3500


def capsule_region64(r, p, d, lo, hi):
    """RayAABB against the box widened by r (float64) -> None (misses, or enters past the segment) or the region code
    u + v of the entry point"""
    elo, ehi = lo - r, hi + r
    tmin, tmax = 0.0, np.finfo(np.float32).max
    for i in range(3):
        if abs(d[i]) < np.finfo(np.float32).eps:
            if p[i] < elo[i] or p[i] > ehi[i]:
                return None
        else:
            t1, t2 = sorted(((elo[i] - p[i]) / d[i], (ehi[i] - p[i]) / d[i]))
            tmin, tmax = max(tmin, t1), min(tmax, t2)
            if tmin > tmax:
                return None
    if tmin > 1:
        return None
    q = p + d * tmin
    return sum(1 << i for i in range(3) if q[i] < lo[i]) + sum(1 << i for i in range(3) if q[i] > hi[i])


def test_capsule_matches_float64_distance_in_face_regions():
    """where the segment enters the widened box through a face region, CapsuleAABB is exact: it collides iff the
    segment comes within r of the box (dense float64 sampling of the segment)"""
    rng = np.random.default_rng(3)
    vs, o = 0.5, np.zeros(3)
    s = np.linspace(0, 1, 4001)[:, None]
    checked = 0
    for _ in range(3000):
        T = moved(rot(rng.normal(size=3), rng.uniform(0, np.pi)), rng.uniform(-1.5, 1.5, 3))
        r, h = rng.uniform(0.05, 0.6), rng.uniform(0, 2)
        key = np.floor(T[:3, 3] / vs).astype(int) + rng.integers(-2, 3, 3)
        z = T[:3, 2]
        p0, d = T[:3, 3] - 0.5 * h * z, h * z
        lo, hi = cell_box(key, vs, o)
        m = capsule_region64(r, p0, d, lo, hi)
        pts = p0 + s * d
        dist = np.sqrt(np.min(np.sum(np.maximum(0, np.maximum(lo - pts, pts - hi)) ** 2, 1)))
        if abs(dist - r) < 2e-3 * max(h, 1e-3) + 1e-4:
            continue
        got = OC.prim_elem(OC.prim(OC.CAPSULE, T, radius=r, height=h), key, vs, o)
        if m is None:
            assert not got and dist > r
            checked += 1
        elif m & (m - 1) == 0:
            assert got == (dist <= r)
            checked += 1
        elif m == 7:
            assert got  # the reference's corner branch reports a hit whatever the distance
    assert checked > 500


def test_touching_faces_and_edges_collide_at_margin_0():
    vs, o = 1.0, np.zeros(3)
    assert OC.elem_elem([0, 0, 0], vs, o, [1, 0, 0], vs, o)      # shared face
    assert OC.elem_elem([0, 0, 0], vs, o, [1, 1, 0], vs, o)      # shared edge
    assert OC.elem_elem([0, 0, 0], vs, o, [1, 1, 1], vs, o)      # shared corner
    assert not OC.elem_elem([0, 0, 0], vs, o, [2, 0, 0], vs, o)  # one cell apart
    assert OC.elem_elem([0, 0, 0], vs, o, [2, 0, 0], vs, o, margin=0.0) is False
    assert OC.elem_elem([0, 0, 0], vs, o, [2, 0, 0], vs, o, margin=1.0)  # the gap closes exactly


def test_sphere_and_box_tangent_to_a_face_collide():
    vs, o = 0.5, np.array([1.0, 2.0, -3.0])  # powers of two and integers: every corner and centre is exact
    lo, hi = cell_box([0, 0, 0], vs, o)
    c = np.array([hi[0] + 0.25, (lo[1] + hi[1]) / 2, (lo[2] + hi[2]) / 2])
    assert OC.prim_elem(OC.prim(OC.SPHERE, moved(np.eye(4), c), radius=0.25), [0, 0, 0], vs, o)
    assert not OC.prim_elem(OC.prim(OC.SPHERE, moved(np.eye(4), c + [0.125, 0, 0]), radius=0.25), [0, 0, 0], vs, o)
    assert OC.prim_elem(OC.prim(OC.BOX, moved(np.eye(4), c), lengths=[0.5, 0.5, 0.5]), [0, 0, 0], vs, o)


def test_cylinder_never_collides():
    assert not OC.prim_elem(OC.prim(OC.CYLINDER, radius=5.0, height=5.0), [0, 0, 0], 1.0, np.zeros(3))


def test_deviation_smallest_target_index():
    t = OC.voxel_grid([[5, 5, 5], [1, 0, 0], [0, 0, 0], [0, 0, 0]], 1.0, np.zeros(3))
    q = OC.voxel_grid([[0, 0, 0]], 1.0, np.zeros(3))
    assert OC.compute(t, q).tolist() == [[1, 0]]  # (1,0,0) touches, and 1 < 2, 3
    sph = OC.prims([OC.prim(OC.SPHERE, radius=3.0)])
    assert OC.compute(t, sph).tolist() == [[1, 0]]


def big_rotated_box_scene():
    """a box rotated 45 degrees about z and x whose AABB covers > 1e5 target cells; every target voxel of the AABB lies
    outside the box except the last one, at its centre"""
    T = moved(rot([0, 0, 1], np.pi / 4) @ rot([1, 0, 0], np.pi / 4), [0.0, 0.0, 0.0])
    L = np.array([120.0, 8.0, 8.0])
    vs = 1.0
    ext = np.abs(T[:3, :3]) @ (L / 2) + 1
    g = np.stack(np.meshgrid(*[np.arange(int(np.floor(-e)), int(np.ceil(e))) for e in ext], indexing="ij"), -1).reshape(-1, 3)
    c = g + 0.5
    # clear of the box by 2 voxels along one of its axes, whether R's columns or its rows are taken as the axes
    far = np.any(np.abs((c - T[:3, 3]) @ T[:3, :3]) > L / 2 + 2.0, 1)
    far &= np.any(np.abs((c - T[:3, 3]) @ T[:3, :3].T) > L / 2 + 2.0, 1)
    keys = np.concatenate([g[far], [[0, 0, 0]]]).astype(np.int32)
    return OC.prim(OC.BOX, T, lengths=L), keys, vs


def test_deviation_no_candidate_cap():
    p, keys, vs = big_rotated_box_scene()
    assert len(keys) > 100_000
    t = OC.voxel_grid(keys, vs, np.zeros(3))
    assert OC.compute(t, OC.prims([p])).tolist() == [[len(keys) - 1, 0]]


def test_deviation_margin_in_both_orders():
    vs = 1.0
    g = OC.voxel_grid([[0, 0, 0]], vs, np.zeros(3))
    s = OC.prims([OC.prim(OC.SPHERE, moved(np.eye(4), [1.75, 0.5, 0.5]), radius=0.5)])  # 0.25 from the voxel
    assert OC.compute(g, s, 0.0).size == 0 and OC.compute(s, g, 0.0).size == 0
    assert OC.compute(g, s, 0.5).tolist() == [[0, 0]]
    assert OC.compute(s, g, 0.5).tolist() == [[0, 0]]


def test_deviation_one_placement_for_occupancy_cells():
    """res 8, voxel 1, origin 0: occupied cell (4, 4, 4) covers [0, 1]^3.  The reference's query-side paths put it at
    [4, 5]^3, where the VoxelGrid voxel (4, 4, 4) is; here it does not collide in either order"""
    prob = np.full((8, 8, 8), np.nan, np.float32)
    prob[4, 4, 4] = 1.0
    occ = OC.occupancy_grid(prob, [0, 0, 0], [7, 7, 7], 0.0, 1.0, np.zeros(3))
    vg = OC.voxel_grid([[4, 4, 4]], 1.0, np.zeros(3))
    assert OC.compute(occ, vg).size == 0 and OC.compute(vg, occ).size == 0
    vg0 = OC.voxel_grid([[0, 0, 0]], 1.0, np.zeros(3))
    assert OC.compute(occ, vg0).tolist() == [[4 * 64 + 4 * 8 + 4, 0]]
    assert OC.compute(vg0, occ).tolist() == [[0, 4 * 64 + 4 * 8 + 4]]
    sph = OC.prims([OC.prim(OC.SPHERE, moved(np.eye(4), [4.5, 4.5, 4.5]), radius=0.4)])
    assert OC.compute(occ, sph).size == 0 and OC.compute(sph, occ).size == 0


def test_occupied_cells_outside_the_bound_box_never_collide():
    prob = np.full((8, 8, 8), np.nan, np.float32)
    prob[1, 1, 1] = prob[6, 6, 6] = 2.0
    vg = OC.voxel_grid(np.array([[-3, -3, -3], [2, 2, 2]], np.int32), 1.0, np.zeros(3))
    full = OC.occupancy_grid(prob, [0, 0, 0], [7, 7, 7], 0.0, 1.0, np.zeros(3))
    assert OC.compute(vg, full)[:, 1].tolist() == [1 * 64 + 9, 6 * 64 + 6 * 8 + 6]
    shrunk = OC.occupancy_grid(prob, [4, 4, 4], [7, 7, 7], 0.0, 1.0, np.zeros(3))
    assert OC.compute(vg, shrunk)[:, 1].tolist() == [6 * 64 + 6 * 8 + 6]
