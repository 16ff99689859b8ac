"""Mesh filtering (the counterpart of the reference's basic/mesh_filter.py): a sphere fused from noisy synthetic depth
frames is extracted as a mesh, then sharpened and smoothed by the four filters at 100 iterations each.  The reference
example uses meshes.knot() and a viewer; here the mesh comes from a TSDF volume and the result is printed as the
vertices' spread around the true radius.  There is no visualiser and no IO."""
import numpy as np

import cupoch_b200 as cph
from cupoch_b200.testing.datagen import ring_cameras, sphere_depth

W, H, R = 320, 240, 0.6


def noisy_sphere_mesh():
    cams = ring_cameras(8, W, H)
    K = cams[0][0]
    intrinsic = cph.camera.PinholeCameraIntrinsic(W, H, K[0, 0], K[1, 1], K[0, 2], K[1, 2])
    volume = cph.integration.UniformTSDFVolume(2.0, 192, 0.04, cph.integration.TSDFVolumeColorType.RGB8)
    rng = np.random.default_rng(0)
    for _, E in cams:
        d = sphere_depth(K, E, W, H, R)
        d = np.where(d > 0, d + rng.normal(0, 0.004, d.shape), 0)  # a few millimetres of sensor noise
        depth = cph.geometry.Image(np.round(d * 1000).astype(np.uint16))
        color = cph.geometry.Image(rng.integers(0, 256, (H, W, 3), dtype=np.uint8))
        volume.integrate(cph.geometry.RGBDImage.create_from_color_and_depth(color, depth, depth_trunc=4.0,
                                                                            convert_rgb_to_intensity=False), intrinsic, E)
    mesh = volume.extract_triangle_mesh()
    mesh.compute_vertex_normals()
    return mesh


def spread(mesh):
    """standard deviation of the vertices' distance from the sphere's centre, in millimetres"""
    return 1000 * float(np.linalg.norm(mesh.vertices.cpu(), axis=1).std())


def main():
    mesh = noisy_sphere_mesh()
    print("input:", len(mesh.vertices), "vertices,", len(mesh.triangles), "triangles; radius spread %.3f mm" % spread(mesh))
    print("surface area %.4f m^2 (4 pi r^2 = %.4f)" % (mesh.get_surface_area(), 4 * np.pi * R * R))
    S = cph.geometry.FilterScope
    out = mesh.filter_sharpen(number_of_iterations=1, strength=0.05, filter_scope=S.All)
    print("filter_sharpen(1, 0.05): radius spread %.3f mm" % spread(out))
    out = mesh.filter_smooth_simple(number_of_iterations=100)
    print("filter_smooth_simple(100): radius spread %.3f mm, area %.4f" % (spread(out), out.get_surface_area()))
    out = mesh.filter_smooth_laplacian(number_of_iterations=100, lambda_=0.5)
    print("filter_smooth_laplacian(100): radius spread %.3f mm, area %.4f" % (spread(out), out.get_surface_area()))
    out = mesh.filter_smooth_taubin(number_of_iterations=100)
    print("filter_smooth_taubin(100): radius spread %.3f mm, area %.4f (Taubin shrinks less)" % (spread(out), out.get_surface_area()))
    out = mesh.filter_smooth_laplacian(number_of_iterations=10, lambda_=0.5, filter_scope=S.Normal)
    print("filter_smooth_laplacian(10, Normal): vertices unchanged:", bool(np.array_equal(out.vertices.cpu(), mesh.vertices.cpu())))


if __name__ == "__main__":
    main()
