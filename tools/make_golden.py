#!/usr/bin/env python3
"""Generate tests/golden/reference_vectors.json (and segment_plane_known.json, pointcloud_crop_known.json,
collision_known.json) from the reference's own unit tests.  `make_golden.py collision` writes collision_known.json only.

Run in the development container only (needs /root/reference, which does not
exist on the GPU box).  It reads
  src/tests/test_utility/raw.cpp      -- the 1021-byte deterministic data table
  src/tests/test_utility/rand.cpp     -- (restated below) Rand(Vector3f) = vmin + byte/255*(vmax-vmin)
  src/tests/knn/kdtree_flann.cpp      -- SearchKNN / SearchRadius golden vectors
  src/tests/knn/lbvh_knn.cpp          -- 1-NN golden
  src/tests/geometry/pointcloud.cpp   -- bounds, VoxelDownSample, EstimateNormals goldens
and writes the INPUT arrays (as produced by the reference's generator) plus
the EXPECTED outputs the reference's tests assert.  Only data is extracted;
no reference source is copied into the repository.
"""
import json
import os
import re
import sys

import numpy as np

REF = os.environ.get("CUPOCH_REFERENCE", "/root/reference")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "reference_vectors.json")
OUT_SEG = os.path.join(os.path.dirname(OUT), "segment_plane_known.json")  # kept apart: the vectors above are frozen
OUT_CROP = os.path.join(os.path.dirname(OUT), "pointcloud_crop_known.json")


def read(rel):
    with open(os.path.join(REF, rel)) as f:
        return f.read()


def raw_table():
    src = read("src/tests/test_utility/raw.cpp")
    m = re.search(r"Raw::data_\s*=\s*\{(.*?)\};", src, re.S)
    vals = [int(x) for x in re.findall(r"\d+", m.group(1))]
    assert len(vals) == 1021, len(vals)
    return vals


def rand_vec3f(table, size, vmin, vmax, seed):
    """unit_test::Rand(host_vector<Vector3f>&, vmin, vmax, seed), rand.cpp:115-131 +
    Raw(seed)/Raw::Next<float>, raw.h:30-60, raw.cpp:140-156 (float32 arithmetic)."""
    step = 1 if seed <= 0 else seed
    index = abs(seed) % 1021
    vmin = np.asarray(vmin, np.float32)
    factor = (np.asarray(vmax, np.float32) - vmin).astype(np.float32)
    out = np.zeros((size, 3), np.float32)
    for i in range(size):
        for c in range(3):
            v = np.float32(table[index]) / np.float32(255)
            index = (index + step) % 1021
            out[i, c] = vmin[c] + np.float32(v) * factor[c]
    return out


def brace_numbers(src, name):
    m = re.search(name + r"\[\]\s*=\s*\{(.*?)\};", src, re.S)
    return [float(x) for x in re.findall(r"-?\d+\.?\d*(?:[eE]-?\d+)?", m.group(1))]


def test_body(src, suite, name):
    m = re.search(r"TEST\(%s,\s*%s\)\s*\{" % (suite, name), src)
    start = m.end()
    nxt = re.search(r"\nTEST\(", src[start:])
    return src[start:start + nxt.start()] if nxt else src[start:]


def pushed_vec3(body, var):
    pat = re.compile(var + r"\.push_back\(Vector3f\(\s*(-?[\d.]+)\s*,\s*(-?[\d.]+)\s*,\s*(-?[\d.]+)\s*\)\)")
    return [[float(a), float(b), float(c)] for a, b, c in pat.findall(body)]


def main():
    table = raw_table()
    g = {"source": "neka-nat/cupoch @ae9d6c04 src/tests (see tools/make_golden.py)"}

    # ---- knn/kdtree_flann.cpp:47-135 -------------------------------------
    kd = read("src/tests/knn/kdtree_flann.cpp")
    pts100 = rand_vec3f(table, 100, (0, 0, 0), (10, 10, 10), 0)
    b = test_body(kd, "KDTreeFlann", "SearchKNN")
    g["knn"] = {
        "points": pts100.tolist(),
        "query": [1.647059, 4.392157, 8.784314],
        "k": 30,
        "indices": [int(x) for x in brace_numbers(b, "indices0")],
        "distance2": brace_numbers(b, "distances0"),
        "result": 30,
        "cite": "src/tests/knn/kdtree_flann.cpp:47-91",
    }
    b = test_body(kd, "KDTreeFlann", "SearchRadius")
    g["radius"] = {
        "points": pts100.tolist(),
        "query": [1.647059, 4.392157, 8.784314],
        "radius": 5.0,
        "max_nn": 15,
        "indices": [int(x) for x in brace_numbers(b, "indices0")],
        "distance2": brace_numbers(b, "distances0"),
        "result": 15,
        "cite": "src/tests/knn/kdtree_flann.cpp:93-135",
    }
    g["lbvh_1nn"] = {"points": pts100.tolist(), "query": [1.647059, 4.392157, 8.784314],
                     "index": 27, "cite": "src/tests/knn/lbvh_knn.cpp:47-86"}

    # ---- geometry/pointcloud.cpp -----------------------------------------
    pc = read("src/tests/geometry/pointcloud.cpp")
    pts1000 = rand_vec3f(table, 100, (0, 0, 0), (1000, 1000, 1000), 0)
    g["bounds"] = {
        "points": pts1000.tolist(),
        "min": [19.607843, 0.0, 0.0],
        "max": [996.078431, 996.078431, 996.078431],
        "cite": "src/tests/geometry/pointcloud.cpp:111-141",
    }
    b = test_body(pc, "PointCloud", "VoxelDownSample")
    g["voxel"] = {
        "points": rand_vec3f(table, 20, (0, 0, 0), (1000, 1000, 1000), 0).tolist(),
        "normals": rand_vec3f(table, 20, (0, 0, 0), (10, 10, 10), 0).tolist(),
        "colors": rand_vec3f(table, 20, (0, 0, 0), (255, 255, 255), 0).tolist(),
        "voxel_size": 0.5,
        "ref_points": pushed_vec3(b, "ref_points"),
        "ref_normals": pushed_vec3(b, "ref_normals"),
        "ref_colors": pushed_vec3(b, "ref_colors"),
        "cite": "src/tests/geometry/pointcloud.cpp:371-469",
    }
    assert len(g["voxel"]["ref_points"]) == 20 and len(g["voxel"]["ref_normals"]) == 20
    b = test_body(pc, "PointCloud", "EstimateNormals")
    g["normals"] = {
        "points": rand_vec3f(table, 40, (0, 0, 0), (1000, 1000, 1000), 0).tolist(),
        "knn": 30,
        "ref": pushed_vec3(b, "ref"),
        "cite": "src/tests/geometry/pointcloud.cpp:535-597",
    }
    assert len(g["normals"]["ref"]) == 40
    g["transform"] = {
        "points": rand_vec3f(table, 10, (0, 0, 0), (1000, 1000, 1000), 0).tolist(),
        "tolerance": 5e-4,
        "cite": "src/tests/geometry/pointcloud.cpp:143-174",
    }
    g["kabsch"] = {
        "points": rand_vec3f(table, 20, (0, 0, 0), (1000, 1000, 1000), 0).tolist(),
        "angle_deg_z": 30.0,
        "tolerance": 1e-3,
        "cite": "src/tests/registration/kabsch.cpp:35-55",
    }
    # ---- container / filter known answers (pointcloud.cpp:303-334, 676-693) ----
    b = test_body(pc, "PointCloud", "RemoveRadiusOutliers")
    pat = re.compile(r"points\.push_back\(Eigen::Vector3f\(\{\s*(-?[\d.]+)\s*,\s*(-?[\d.]+)\s*,\s*(-?[\d.]+)\s*\}\)\)")
    rro_pts = [[float(x), float(y), float(z)] for x, y, z in pat.findall(b)]
    m = re.search(r"RemoveRadiusOutliers\((\d+),\s*([\d.]+)\)", b)
    assert len(rro_pts) == 8 and m
    g["radius_outliers"] = {
        "points": rro_pts, "nb_points": int(m.group(1)), "radius": float(m.group(2)),
        "kept_points": [[0.0, 0.0, 0.0]],  # EXPECT_EQ(size, 1); EXPECT_EQ(h_pt[0], (0,0,0))
        "cite": "src/tests/geometry/pointcloud.cpp:676-693",
    }
    b = test_body(pc, "PointCloud", "SelectByIndex")
    g["select_by_index"] = {
        "points": pts1000.tolist(),
        "indices": [int(x) for x in re.findall(r"ref_idx\.push_back\((\d+)\)", b)],
        "cite": "src/tests/geometry/pointcloud.cpp:303-334 (output == the named rows, compared as sorted sets)",
    }
    assert len(g["select_by_index"]["indices"]) == 10
    # ---- SegmentPlane known plane (pointcloud.cpp:659-673): all five coplanar points are inliers ----
    b = test_body(pc, "PointCloud", "SegmentPlaneKnownPlane")
    pat = re.compile(r"ref_points\.push_back\(Eigen::Vector3f\(\{\s*(-?[\d.]+)\s*,\s*(-?[\d.]+)\s*,\s*(-?[\d.]+)\s*\}\)\)")
    sp_pts = [[float(x), float(y), float(z)] for x, y, z in pat.findall(b)]
    m = re.search(r"SegmentPlane\(([\d.]+),\s*(\d+),\s*(\d+)\)", b)
    assert len(sp_pts) == 5 and m and "SelectByIndex(inliers)" in b
    seg = {"source": g["source"], "segment_plane_known": {
        "points": sp_pts, "distance_threshold": float(m.group(1)), "ransac_n": int(m.group(2)),
        "num_iterations": int(m.group(3)),
        # ExpectEQ(SelectByIndex(inliers)->GetPoints(), ref_points).  (The test's comment names x + y + z + 1 = 0, but
        # (1, 1, -1) is not on it; all five points satisfy x = y.)
        "inliers": list(range(len(sp_pts))),
        "cite": "src/tests/geometry/pointcloud.cpp:659-673",
    }}
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    with open(OUT, "w") as f:
        json.dump(g, f)
    with open(OUT_SEG, "w") as f:
        json.dump(seg, f)
    print("wrote", os.path.normpath(OUT_SEG), os.path.getsize(OUT_SEG), "bytes")
    print("wrote", os.path.normpath(OUT), os.path.getsize(OUT), "bytes")
    crop_known(table, pc, g["source"])


def crop_known(table, pc, source):
    """the bounding-box and cleanup known answers (pointcloud.cpp:176-220,264-302,471-533,599-657) -> OUT_CROP"""
    b = test_body(pc, "PointCloud", "GetOrientedBoundingBox")
    pat = re.compile(r"(\w+)\.push_back\(\{\s*(-?[\d.]+)\s*,\s*(-?[\d.]+)\s*,\s*(-?[\d.]+)\s*\}\)")
    rows = {}
    for var, x, y, z in pat.findall(b):
        rows.setdefault(var, []).append([float(x), float(y), float(z)])
    four, eight, box = rows["points"][:4], rows["points"][4:], rows["ref_points"]
    assert len(four) == 4 and len(eight) == 8 and len(box) == 8
    assert "Eigen::Vector3f(1.5, 1, 0.5)" in b and "Eigen::Vector3f(3, 2, 1)" in b and "Matrix3f::Identity()" in b
    out = {"source": source, "tolerance": 1e-4}  # THRESHOLD_1E_4, the default of the reference's ExpectEQ / ExpectLE
    out["oriented_bounding_box"] = {
        "points_4": four, "points_8": eight, "center": [1.5, 1.0, 0.5], "extent": [3.0, 2.0, 1.0],
        "R": [[1.0, 0.0, 0.0], [0.0, 1.0, 0.0], [0.0, 0.0, 1.0]], "box_points": box,
        "cite": "src/tests/geometry/pointcloud.cpp:176-220 (center, extent and R exact; box points as a sorted set)"}
    b = test_body(pc, "PointCloud", "NormalizeNormals")
    out["normalize_normals"] = {"normals": rand_vec3f(table, 20, (0, 0, 0), (1000, 1000, 1000), 0).tolist(),
                                "ref": pushed_vec3(b, "ref"), "cite": "src/tests/geometry/pointcloud.cpp:264-302"}
    b = test_body(pc, "PointCloud", "UniformDownSample")
    out["uniform_down_sample"] = {"points": rand_vec3f(table, 100, (0, 0, 0), (1000, 1000, 1000), 0).tolist(),
                                  "every_k_points": 4, "ref": pushed_vec3(b, "ref"),
                                  "cite": "src/tests/geometry/pointcloud.cpp:471-513"}
    b = test_body(pc, "PointCloud", "CropPointCloud")
    assert "minBound(200.0, 200.0, 200.0)" in b and "maxBound(800.0, 800.0, 800.0)" in b
    out["crop"] = {"points": rand_vec3f(table, 100, (0, 0, 0), (1000, 1000, 1000), 0).tolist(),
                   "min_bound": [200.0] * 3, "max_bound": [800.0] * 3,
                   "cite": "src/tests/geometry/pointcloud.cpp:515-533 (every kept point lies within the bounds)"}
    b = test_body(pc, "PointCloud", "OrientNormalsToAlignWithDirection")
    assert "Vector3f(1.5, 0.5, 3.3)" in b and "EstimateNormals()" in b
    out["orient_normals"] = {"points": rand_vec3f(table, 40, (0, 0, 0), (1000, 1000, 1000), 0).tolist(), "knn": 30,
                             "reference": [1.5, 0.5, 3.3], "ref": pushed_vec3(b, "ref"),
                             "cite": "src/tests/geometry/pointcloud.cpp:599-657 (EstimateNormals with KNN 30 first)"}
    assert len(out["normalize_normals"]["ref"]) == 20 and len(out["uniform_down_sample"]["ref"]) == 25
    assert len(out["orient_normals"]["ref"]) == 40
    with open(OUT_CROP, "w") as f:
        json.dump(out, f)
    print("wrote", os.path.normpath(OUT_CROP), os.path.getsize(OUT_CROP), "bytes")


def collision_known():
    """TEST(Collision, VoxelVoxel) (src/tests/collision/collision.cpp) -> OUT_COLL: its three steps, each with the
    voxel keys the test has added by then (voxel size 1, origin 0) and what it asserts"""
    b = test_body(read("src/tests/collision/collision.cpp"), "Collision", "VoxelVoxel")
    adds = re.findall(r"(voxel[12])\.AddVoxel\(geometry::Voxel\(Eigen::Vector3i\((-?\d+),\s*(-?\d+),\s*(-?\d+)\)\)\)", b)
    assert len(adds) == 4 and "voxel_size_ = 1.0" in b and "Eigen::Vector2i(0, 0)" in b, adds
    keys = {"voxel1": [], "voxel2": []}
    steps = []
    for i, (v, x, y, z) in enumerate(adds):
        keys[v].append([int(x), int(y), int(z)])
        if i % 2 == 1:
            steps.append({"keys1": [list(k) for k in keys["voxel1"]], "keys2": [list(k) for k in keys["voxel2"]]})
    out = {"voxel_size": 1.0, "origin": [0.0, 0.0, 0.0],
           "steps": [{"keys1": [], "keys2": [], "collided": False}] +
                    [dict(steps[0], collided=True), dict(steps[1], collided=True, pairs=[[0, 0]])],
           "cite": "src/tests/collision/collision.cpp TEST(Collision, VoxelVoxel): empty grids do not collide; one "
                   "shared voxel collides; with (5,0,0) and (10,0,0) added there is exactly one pair, (0, 0)"}
    with open(OUT_COLL, "w") as f:
        json.dump(out, f)
    print("wrote", os.path.normpath(OUT_COLL), os.path.getsize(OUT_COLL), "bytes")


OUT_COLL = os.path.join(os.path.dirname(OUT), "collision_known.json")

if __name__ == "__main__":
    if sys.argv[1:] == ["collision"]:  # only the collision known answer; the other files stay as they are
        sys.exit(collision_known())
    rc = main()
    collision_known()
    sys.exit(rc)
