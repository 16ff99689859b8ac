// The reference's known-answer tests for the round-1 "next" rows, written against the header-compatible facade
// exactly as the reference's own tests are written against cupoch:
//   tests/geometry/pointcloud.cpp:676-693  PointCloud.RemoveRadiusOutliers
//   tests/geometry/pointcloud.cpp:303-334  PointCloud.SelectByIndex
//   tests/geometry/voxelgrid.cpp:40-68     VoxelGrid.GetVoxel, VoxelGrid.CreateFromPointCloudWithinBounds
//   tests/geometry/occupancygrid.cpp:30-97 OccupancyGrid.Bounds, .GetVoxel, .Insert, .SetFreeArea
// plus RemoveStatisticalOutliers on a cloud with planted outliers.  Exit code 0 = all expectations met.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <vector>

#include "cupoch/geometry/pointcloud.h"
#include "cupoch/geometry/voxelgrid.h"
#include "facade_check.h"

using namespace cupoch;

int main() {
    {   // RemoveRadiusOutliers
        std::vector<Eigen::Vector3f> points = {{0.0f, 0.0f, 0.0f}, {1.0f, 0.0f, 0.0f}, {-1.0f, 0.0f, 0.0f}, {0.0f, 1.0f, 0.0f},
                                               {0.0f, -1.0f, 0.0f}, {0.0f, 0.0f, 1.0f}, {0.0f, 0.0f, -1.0f}, {2.0f, 0.0f, 0.0f}};
        geometry::PointCloud pcd;
        pcd.SetPoints(points);
        auto res = pcd.RemoveRadiusOutliers(6, 1.1f);
        auto h_pt = std::get<0>(res)->GetPoints();
        EXPECT((int)h_pt.size() == 1);
        if (h_pt.size() == 1) EXPECT(h_pt[0][0] == 0.0f && h_pt[0][1] == 0.0f && h_pt[0][2] == 0.0f);
        auto idx = std::get<1>(res).to_host();
        EXPECT(idx.size() == 1 && idx[0] == 0);
    }
    {   // SelectByIndex (+ invert)
        std::vector<Eigen::Vector3f> points(100);
        for (int i = 0; i < 100; ++i) points[i] = Eigen::Vector3f((float)i, (float)(2 * i), (float)(3 * i));
        geometry::PointCloud pc;
        pc.SetPoints(points);
        std::vector<size_t> ref_idx = {3, 10, 24, 32, 47, 51, 66, 79, 85, 98};
        utility::device_vector<size_t> d_idx(ref_idx);
        auto out = pc.SelectByIndex(d_idx)->GetPoints();
        EXPECT(out.size() == ref_idx.size());
        for (size_t t = 0; t < out.size() && t < ref_idx.size(); ++t) EXPECT(out[t][0] == (float)ref_idx[t]);
        auto inv = pc.SelectByIndex(d_idx, true)->GetPoints();
        EXPECT(inv.size() == 90);
        if (!inv.empty()) EXPECT(inv[0][0] == 0.0f && inv[3][0] == 4.0f);
    }
    {   // RemoveStatisticalOutliers: a 20x20x5 lattice plus three far points
        std::vector<Eigen::Vector3f> points;
        for (int x = 0; x < 20; ++x)
            for (int y = 0; y < 20; ++y)
                for (int z = 0; z < 5; ++z) points.push_back(Eigen::Vector3f(0.1f * x, 0.1f * y, 0.1f * z));
        const size_t n_in = points.size();
        points.push_back(Eigen::Vector3f(10.f, 10.f, 10.f));
        points.push_back(Eigen::Vector3f(-7.f, 3.f, 9.f));
        points.push_back(Eigen::Vector3f(4.f, -8.f, 5.f));
        geometry::PointCloud pcd;
        pcd.SetPoints(points);
        auto res = pcd.RemoveStatisticalOutliers(10, 2.0f);
        auto idx = std::get<1>(res).to_host();
        EXPECT(!idx.empty() && idx.size() <= n_in);
        EXPECT(std::is_sorted(idx.begin(), idx.end()));
        for (size_t i : idx) EXPECT(i < n_in);  // the planted outliers are gone
        EXPECT(std::get<0>(res)->GetPoints().size() == idx.size());
        // GaussianFilter: a lattice point strictly inside keeps its place (symmetric neighbourhood), sizes are kept
        auto smooth = pcd.GaussianFilter(0.15f, 0.01f, 30);
        auto sp = smooth->GetPoints();
        EXPECT(sp.size() == points.size());
        const size_t mid = (10 * 20 + 10) * 5 + 2;  // lattice node (10, 10, 2)
        if (sp.size() == points.size())
            EXPECT(std::fabs(sp[mid][0] - 1.0f) < 1e-4f && std::fabs(sp[mid][1] - 1.0f) < 1e-4f && std::fabs(sp[mid][2] - 0.2f) < 1e-4f);
        EXPECT(pcd.GaussianFilter(0.0f, 0.01f, 30)->IsEmpty());
    }
    {   // VoxelGrid
        geometry::VoxelGrid g;
        g.origin_ = Eigen::Vector3f(0, 0, 0);
        g.voxel_size_ = 5;
        auto v = g.GetVoxel(Eigen::Vector3f(0, 4.9f, 0));
        EXPECT(v[0] == 0 && v[1] == 0 && v[2] == 0);
        v = g.GetVoxel(Eigen::Vector3f(0, 5, 0));
        EXPECT(v[1] == 1);
        v = g.GetVoxel(Eigen::Vector3f(0, 5.1f, 0));
        EXPECT(v[1] == 1);
        geometry::PointCloud pc;
        pc.SetPoints({Eigen::Vector3f(0.5f, 0.5f, 0.5f)});
        auto grid = geometry::VoxelGrid::CreateFromPointCloudWithinBounds(pc, 1.0f, Eigen::Vector3f(-100.0f, -100.0f, -100.0f),
                                                                          Eigen::Vector3f(100.0f, 100.0f, 100.0f));
        EXPECT(grid->voxels_keys_.size() == 1);
        auto kv = grid->GetVoxels();
        if (kv.first.size() == 1) EXPECT(kv.first[0][0] == 100 && kv.second[0].color_[0] == 1.0f);
        auto grid2 = geometry::VoxelGrid::CreateFromPointCloud(pc, 0.5f);
        EXPECT(grid2->voxels_keys_.size() == 1 && grid2->HasVoxels());
    }
    {   // OccupancyGrid: the reference's known-answer tests (tests/geometry/occupancygrid.cpp:30-97)
        geometry::OccupancyGrid og;
        EXPECT(std::fabs(og.voxel_size_ - 0.05f) < 1e-7f && og.resolution_ == 512);
        og.voxel_size_ = 5;
        og.AddVoxel(Eigen::Vector3i(0, 0, 0));
        og.AddVoxel(Eigen::Vector3i(511, 511, 511));
        EXPECT(og.GetMinBound()[0] == -512 * 5 * 0.5f && og.GetMaxBound()[2] == 512 * 5 * 0.5f);
        geometry::OccupancyGrid g2;
        g2.voxel_size_ = 1.0f;
        g2.AddVoxel(Eigen::Vector3i(257, 256, 256), true);
        g2.AddVoxel(Eigen::Vector3i(257, 256, 256), true);
        g2.AddVoxel(Eigen::Vector3i(257, 256, 256), false);
        auto r = g2.GetVoxel(Eigen::Vector3f(1.5f, 0.0f, 0.0f));
        EXPECT(std::get<0>(r) && std::fabs(std::get<1>(r).prob_log_ - (2.0f * g2.prob_hit_log_ + g2.prob_miss_log_)) < 1e-6f);
        geometry::OccupancyGrid g3;
        g3.origin_ = Eigen::Vector3f(-0.5f, -0.5f, 0);
        g3.voxel_size_ = 1.0f;
        g3.Insert(std::vector<Eigen::Vector3f>{Eigen::Vector3f(0.0f, 0.0f, 3.5f)}, Eigen::Vector3f(0, 0, 0));
        EXPECT(g3.ExtractKnownVoxels()->size() == 4);
        EXPECT(std::get<0>(g3.GetVoxel(Eigen::Vector3f(0, 0, 0.5f))) && std::get<0>(g3.GetVoxel(Eigen::Vector3f(0, 0, 3.5f))));
        EXPECT(!std::get<0>(g3.GetVoxel(Eigen::Vector3f(0, 0, 4.5f))) && g3.IsOccupied(Eigen::Vector3f(0, 0, 3.5f)));
        geometry::OccupancyGrid g4;
        g4.SetFreeArea(Eigen::Vector3f(0, 0, 0), Eigen::Vector3f(0.1f, 0.1f, 0.1f));
        EXPECT(g4.ExtractFreeVoxels()->size() == 27);
    }
    {   // DBSCAN, FPFH, KabschWeighted: two well separated blobs of 60 points each
        std::vector<Eigen::Vector3f> pts, nrm;
        for (int b = 0; b < 2; ++b)
            for (int i = 0; i < 60; ++i) {
                pts.push_back(Eigen::Vector3f(10.0f * b + 0.01f * (i % 8), 0.01f * (i / 8), 0.002f * (i % 3)));
                nrm.push_back(Eigen::Vector3f(0, 0, 1));
            }
        geometry::PointCloud pc;
        pc.SetPoints(pts);
        pc.SetNormals(nrm);
        auto labels = pc.ClusterDBSCAN(0.05f, 5);
        auto hl = labels->to_host();
        EXPECT(hl.size() == 120 && hl[0] == 0 && hl[59] == 0 && hl[60] == 1 && hl[119] == 1);
        auto fp = registration::ComputeFPFHFeature(pc, knn::KDTreeSearchParamKNN(10));
        EXPECT(fp->Num() == 120 && fp->Dimension() == 33);
        auto hf = fp->data_.to_host();
        float s0 = 0;
        for (int j = 0; j < 11; ++j) s0 += hf[j];
        EXPECT(std::fabs(s0 - 200.0f) < 1e-2f);  // every 11-bin block of an FPFH row sums to 100 (own SPFH) + 100 (neighbours)
        utility::device_vector<float> w(std::vector<float>(120, 0.5f));
        utility::device_vector<Eigen::Vector3f> moved(pts);
        auto T = registration::KabschWeighted(pc.points_, moved, w);
        EXPECT(std::fabs(T(0, 0) - 1.0f) < 1e-5f && std::fabs(T(0, 3)) < 1e-4f);
    }
    if (fails) return 1;
    std::printf("facade filters: all expectations met\n");
    return 0;
}
