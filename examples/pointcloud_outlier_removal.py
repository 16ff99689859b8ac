"""Counterpart of the reference's examples/python/advanced/pointcloud_outlier_removal.py and basic/clustering.py."""
import numpy as np

from _clouds import pair
import cupoch_b200 as cph

if __name__ == "__main__":
    _, tgt, _, _, _ = pair(200_000)
    rng = np.random.default_rng(0)
    noisy = np.concatenate([tgt, rng.random((2000, 3), dtype=np.float32)])      # 1 % stray points off the surface
    pcd = cph.geometry.PointCloud(noisy)
    print("Downsample the point cloud with a voxel of 0.005")
    voxel_down_pcd = pcd.voxel_down_sample(voxel_size=0.005)
    print("Every 5th point of the point cloud")
    uni_down_pcd = pcd.uniform_down_sample(every_k_points=5)
    print("kept", len(uni_down_pcd), "of", len(pcd))
    print("Statistical outlier removal")
    cl, ind = voxel_down_pcd.remove_statistical_outlier(nb_neighbors=20, std_ratio=2.0)
    print("kept", len(cl), "of", len(voxel_down_pcd))
    print("Radius outlier removal")
    cl, ind = voxel_down_pcd.remove_radius_outlier(nb_points=16, radius=0.02)
    print("kept", len(cl), "of", len(voxel_down_pcd))
    print("DBSCAN clustering")
    labels = cl.cluster_dbscan(eps=0.02, min_points=10).cpu()
    print("clusters:", int(labels.max()) + 1, "noise points:", int((labels < 0).sum()))
