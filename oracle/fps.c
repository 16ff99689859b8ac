/*
 * fps.c -- CPU restatement of cupoch's PointCloud::FarthestPointDownSample (geometry/pointcloud.cu:122-139,301-338).
 * TEST INFRASTRUCTURE ONLY, like oracle.c: loaded by tests/ and tools/bench_ops.py through fps_py.py, never by the
 * product.  Built by fps_py.build() with oracle/Makefile's flags: -ffp-contract=off (no implicit FMA; the squared
 * distance's fused multiply-adds are explicit) and no -ffast-math.
 */
#include <math.h>
#include <stdint.h>
#include <string.h>

/* Under DESIGN.md's arithmetic contract: dist starts at +inf; step t records `far`, sets dist[i] = fminf(dist[i],
 * d2(p_i, p_far)) with d2 in dist2's order (fma(dz,dz, fma(dx,dx, dy*dy))), then takes the argmax with the smallest
 * index among equal distances (the reference's reduction leaves that choice unspecified).  dist is in [+0, +inf], so its
 * bits order like its value and the argmax is the largest key (bits << 32 | 0xFFFFFFFF - i).  One thread, in index order.
 * out_idx [num_samples]; dist [n] ends as every point's squared distance to the nearest selected point (the last step's update is applied, its argmax unused).  n <= 0: nothing. */
void orc_farthest_point_down_sample(const float *pts, int n, long num_samples, int32_t *out_idx, float *dist);

void orc_farthest_point_down_sample(const float *pts, int n, long num_samples, int32_t *out_idx, float *dist) {
    if (n <= 0) return;
    for (int i = 0; i < n; ++i) dist[i] = INFINITY;
    long far = 0;
    for (long t = 0; t < num_samples; ++t) {
        out_idx[t] = (int32_t)far;
        const float fx = pts[3 * far], fy = pts[3 * far + 1], fz = pts[3 * far + 2];
        unsigned long long best = 0ull;
        for (int i = 0; i < n; ++i) {
            const float dx = pts[3 * (long)i] - fx, dy = pts[3 * (long)i + 1] - fy, dz = pts[3 * (long)i + 2] - fz;
            const float d = fminf(dist[i], fmaf(dz, dz, fmaf(dx, dx, dy * dy)));
            dist[i] = d;
            uint32_t b;
            memcpy(&b, &d, sizeof(b));
            const unsigned long long key = ((unsigned long long)b << 32) | (0xffffffffu - (uint32_t)i);
            if (key > best) best = key;
        }
        far = (long)(0xffffffffu - (uint32_t)best);
    }
}
