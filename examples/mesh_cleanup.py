"""Merge two TSDF sphere meshes, list where they cut each other, and weld an un-welded copy back together.

    python examples/mesh_cleanup.py
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

import cupoch_b200 as cph  # noqa: E402
from cupoch_b200.testing.datagen import ring_cameras, sphere_depth  # noqa: E402

G, I = cph.geometry, cph.integration


def sphere(res=128):
    w, h = 160, 120
    vol = I.UniformTSDFVolume(2.0, res, 0.06, I.TSDFVolumeColorType.RGB8)
    for K, E in ring_cameras(8, w, h, 2.5):
        d16 = np.round(sphere_depth(K, E, w, h, 0.6) * 1000).astype(np.uint16)
        col = np.full((h, w, 3), 128, np.uint8)
        im = G.RGBDImage.create_from_color_and_depth(G.Image(col), G.Image(d16), 1000.0, 100.0, False)
        vol.integrate(im, cph.camera.PinholeCameraIntrinsic(w, h, K[0, 0], K[1, 1], K[0, 2], K[1, 2]), E)
    return vol.extract_triangle_mesh()


a = sphere()
v, t = a.vertices.cpu(), a.triangles.cpu()
b = G.TriangleMesh(v + np.float32([0.3, 0.1, 0.0]), t)
both = a + b
pairs = both.get_self_intersecting_triangles().cpu()
cross = pairs[(pairs[:, 0] < len(t)) & (pairs[:, 1] >= len(t))]
print("merged: %d triangles, %d intersecting pairs, %d of them between the two spheres" % (len(both.triangles), len(pairs), len(cross)))

soup = G.TriangleMesh(v[t.reshape(-1)], np.arange(3 * len(t), dtype=np.int32).reshape(-1, 3))
print("soup: %d vertices" % len(soup.vertices))
soup.remove_duplicated_vertices().remove_degenerate_triangles().remove_duplicated_triangles()
print("welded: %d vertices, %d triangles (the original had %d and %d)" % (len(soup.vertices), len(soup.triangles), len(v), len(t)))
