// cupoch_b200_facade.h -- header-only C++17 facade that reproduces the cupoch
// classes on the ICP / kNN / voxel-grid path on top of the C ABI
// (include/cupoch_b200.h).  Names, argument meaning and error behaviour follow
// the reference headers cited at each declaration; no thrust, no CUDA headers.
//
// Eigen: used when available (cupoch's API types are Eigen's); otherwise
// layout-compatible PODs are declared in namespace Eigen so that the facade
// still builds where Eigen is absent (it is absent in the build container).
#pragma once
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <stdexcept>
#include <algorithm>
#include <array>
#include <tuple>
#include <utility>
#include <limits>
#include <vector>

#include "cupoch_b200.h"

#if __has_include(<Eigen/Core>)
#include <Eigen/Core>
namespace Eigen {
typedef Matrix<float, 4, 4, DontAlign> Matrix4f_u;
}
#else
namespace Eigen {
struct Vector3f {
    float v[3];
    Vector3f() : v{0, 0, 0} {}
    Vector3f(float x, float y, float z) : v{x, y, z} {}
    float &operator[](int i) { return v[i]; }
    float operator[](int i) const { return v[i]; }
    float &operator()(int i) { return v[i]; }
    float operator()(int i) const { return v[i]; }
    static Vector3f Zero() { return Vector3f(); }
};
struct Vector4f {
    float v[4];
    Vector4f() : v{0, 0, 0, 0} {}
    Vector4f(float x, float y, float z, float w) : v{x, y, z, w} {}
    float &operator[](int i) { return v[i]; }
    float operator[](int i) const { return v[i]; }
    float &operator()(int i) { return v[i]; }
    float operator()(int i) const { return v[i]; }
    static Vector4f Zero() { return Vector4f(); }
};
struct Vector3i {
    int v[3];
    Vector3i() : v{0, 0, 0} {}
    Vector3i(int a, int b, int c) : v{a, b, c} {}
    int &operator[](int i) { return v[i]; }
    int operator[](int i) const { return v[i]; }
    int &operator()(int i) { return v[i]; }
    int operator()(int i) const { return v[i]; }
};
struct Vector2i {
    int v[2];
    Vector2i() : v{0, 0} {}
    Vector2i(int a, int b) : v{a, b} {}
    int &operator[](int i) { return v[i]; }
    int operator[](int i) const { return v[i]; }
};
struct Matrix3f {  // column-major like Eigen's default
    float m[9];
    Matrix3f() : m{0, 0, 0, 0, 0, 0, 0, 0, 0} {}
    float &operator()(int r, int c) { return m[3 * c + r]; }
    float operator()(int r, int c) const { return m[3 * c + r]; }
    static Matrix3f Identity() {
        Matrix3f I;
        I.m[0] = I.m[4] = I.m[8] = 1.f;
        return I;
    }
};
struct Matrix4f {  // column-major
    float m[16];
    Matrix4f() { std::memset(m, 0, sizeof(m)); }
    float &operator()(int r, int c) { return m[4 * c + r]; }
    float operator()(int r, int c) const { return m[4 * c + r]; }
    static Matrix4f Identity() {
        Matrix4f I;
        for (int i = 0; i < 4; ++i) I(i, i) = 1.f;
        return I;
    }
    bool isIdentity(float prec = 1e-5f) const {
        for (int r = 0; r < 4; ++r)
            for (int c = 0; c < 4; ++c)
                if (std::fabs((*this)(r, c) - (r == c ? 1.f : 0.f)) > prec) return false;
        return true;
    }
    Matrix4f operator*(const Matrix4f &o) const {
        Matrix4f R;
        for (int r = 0; r < 4; ++r)
            for (int c = 0; c < 4; ++c)
                R(r, c) = (((*this)(r, 0) * o(0, c) + (*this)(r, 1) * o(1, c)) + (*this)(r, 2) * o(2, c)) + (*this)(r, 3) * o(3, c);
        return R;
    }
};
typedef Matrix4f Matrix4f_u;
}  // namespace Eigen
#endif

namespace cupoch {
namespace utility {

inline void LogError(const char *msg) { std::fprintf(stderr, "[cupoch_b200][error] %s\n", msg); }
inline void LogWarning(const char *msg) { std::fprintf(stderr, "[cupoch_b200][warning] %s\n", msg); }
inline void check(int rc) {
    if (rc != CPHB_OK) throw std::runtime_error(std::string("cupoch_b200: ") + cphb_last_error());
}

/// RAII device array (stands in for rmm/thrust device_vector, device_vector.h:67-105).
template <typename T>
class device_vector {
public:
    device_vector() {}
    explicit device_vector(size_t n) { resize(n); }
    device_vector(const std::vector<T> &h) { *this = h; }
    device_vector(const device_vector &o) { copy_from(o); }
    device_vector(device_vector &&o) noexcept : p_(o.p_), n_(o.n_), cap_(o.cap_) { o.p_ = nullptr; o.n_ = o.cap_ = 0; }
    ~device_vector() { cphb_free(p_); }
    device_vector &operator=(const device_vector &o) { if (this != &o) copy_from(o); return *this; }
    device_vector &operator=(device_vector &&o) noexcept {
        if (this != &o) { cphb_free(p_); p_ = o.p_; n_ = o.n_; cap_ = o.cap_; o.p_ = nullptr; o.n_ = o.cap_ = 0; }
        return *this;
    }
    device_vector &operator=(const std::vector<T> &h) {
        resize(h.size());
        if (n_) { check(cphb_memcpy_h2d(p_, h.data(), n_ * sizeof(T), nullptr)); check(cphb_stream_synchronize(nullptr)); }
        return *this;
    }
    void resize(size_t n) {
        if (n > cap_) {
            T *q = static_cast<T *>(cphb_malloc(n * sizeof(T)));
            if (!q) check(CPHB_ERR_CUDA);
            if (n_) check(cphb_memcpy_d2d(q, p_, n_ * sizeof(T), nullptr));
            check(cphb_stream_synchronize(nullptr));
            cphb_free(p_);
            p_ = q;
            cap_ = n;
        }
        n_ = n;
    }
    void clear() { n_ = 0; }
    size_t size() const { return n_; }
    bool empty() const { return n_ == 0; }
    T *data() { return p_; }
    const T *data() const { return p_; }
    std::vector<T> to_host() const {
        std::vector<T> h(n_);
        if (n_) { check(cphb_memcpy_d2h(h.data(), p_, n_ * sizeof(T), nullptr)); check(cphb_stream_synchronize(nullptr)); }
        return h;
    }

private:
    void copy_from(const device_vector &o) {
        resize(o.n_);
        if (n_) { check(cphb_memcpy_d2d(p_, o.p_, n_ * sizeof(T), nullptr)); check(cphb_stream_synchronize(nullptr)); }
    }
    T *p_ = nullptr;
    size_t n_ = 0, cap_ = 0;
};

inline void to_row_major(const Eigen::Matrix4f &M, float out[16]) {
    for (int r = 0; r < 4; ++r)
        for (int c = 0; c < 4; ++c) out[4 * r + c] = M(r, c);
}
inline Eigen::Matrix4f from_row_major(const float in[16]) {
    Eigen::Matrix4f M;
    for (int r = 0; r < 4; ++r)
        for (int c = 0; c < 4; ++c) M(r, c) = in[4 * r + c];
    return M;
}
}  // namespace utility

namespace collision {
namespace detail {
struct Operand;
}  // namespace detail
}  // namespace collision

// --------------------------------------------------------------------------- knn
namespace knn {
static const int NUM_MAX_NN = 100;  // kdtree_search_param.h:26

class KDTreeSearchParam {  // kdtree_search_param.h:28-66
public:
    enum class SearchType { Knn = 0, Radius = 1 };
    virtual ~KDTreeSearchParam() {}
    SearchType GetSearchType() const { return search_type_; }

protected:
    KDTreeSearchParam(SearchType t) : search_type_(t) {}

private:
    SearchType search_type_;
};
class KDTreeSearchParamKNN : public KDTreeSearchParam {
public:
    KDTreeSearchParamKNN(int knn = 30) : KDTreeSearchParam(SearchType::Knn), knn_(knn) {}
    int knn_;
};
class KDTreeSearchParamRadius : public KDTreeSearchParam {
public:
    KDTreeSearchParamRadius(float radius, int max_nn) : KDTreeSearchParam(SearchType::Radius), radius_(radius), max_nn_(max_nn) {}
    float radius_;
    int max_nn_;
};

/// knn::KDTreeFlann (kdtree_flann.h:43-124).  Non-copyable; copies the data like the reference.
class KDTreeFlann {
public:
    KDTreeFlann() {}
    KDTreeFlann(const utility::device_vector<Eigen::Vector3f> &data) { SetRawData(data); }
    ~KDTreeFlann() { release(); }
    KDTreeFlann(const KDTreeFlann &) = delete;
    KDTreeFlann &operator=(const KDTreeFlann &) = delete;

    bool SetRawData(const utility::device_vector<Eigen::Vector3f> &data) {
        release();
        n_ = data.size();
        if (n_ == 0) return false;  // kdtree_flann.inl:128-131
        utility::check(cphb_index_create(reinterpret_cast<const float *>(data.data()), n_, nullptr, &ix_));
        return true;
    }
    int Search(const utility::device_vector<Eigen::Vector3f> &query, const KDTreeSearchParam &param,
               utility::device_vector<int> &indices, utility::device_vector<float> &distance2) const {
        switch (param.GetSearchType()) {
            case KDTreeSearchParam::SearchType::Knn:
                return SearchKNN(query, static_cast<const KDTreeSearchParamKNN &>(param).knn_, indices, distance2);
            case KDTreeSearchParam::SearchType::Radius: {
                const auto &p = static_cast<const KDTreeSearchParamRadius &>(param);
                return SearchRadius(query, p.radius_, p.max_nn_, indices, distance2);
            }
        }
        return -1;
    }
    int SearchKNN(const utility::device_vector<Eigen::Vector3f> &query, int knn, utility::device_vector<int> &indices,
                  utility::device_vector<float> &distance2) const {
        if (!ix_ || n_ == 0 || query.empty() || knn < 0 || knn > NUM_MAX_NN) return -1;  // kdtree_flann.cu:46-48
        indices.resize(query.size() * knn);
        distance2.resize(query.size() * knn);
        int64_t cnt = 0;
        int rc = cphb_search_knn(ix_, reinterpret_cast<const float *>(query.data()), query.size(), knn, indices.data(),
                                 distance2.data(), &cnt, nullptr);
        return rc == CPHB_OK ? (int)cnt : -1;
    }
    int SearchRadius(const utility::device_vector<Eigen::Vector3f> &query, float radius, int max_nn,
                     utility::device_vector<int> &indices, utility::device_vector<float> &distance2) const {
        if (!ix_ || n_ == 0 || query.empty() || max_nn < 0) return -1;  // kdtree_flann.cu:70-72
        indices.resize(query.size() * max_nn);
        distance2.resize(query.size() * max_nn);
        int64_t cnt = 0;
        int rc = cphb_search_radius(ix_, reinterpret_cast<const float *>(query.data()), query.size(), radius, max_nn,
                                    indices.data(), distance2.data(), &cnt, nullptr);
        return rc == CPHB_OK ? (int)cnt : -1;
    }
    /// north_star's name for SearchRadius (SURVEY.md section 0).
    int SearchHybrid(const utility::device_vector<Eigen::Vector3f> &query, float radius, int max_nn,
                     utility::device_vector<int> &indices, utility::device_vector<float> &distance2) const {
        return SearchRadius(query, radius, max_nn, indices, distance2);
    }
    // single host query overloads (kdtree_flann.cu:88-129)
    int SearchKNN(const Eigen::Vector3f &query, int knn, std::vector<int> &indices, std::vector<float> &distance2) const {
        utility::device_vector<Eigen::Vector3f> q(std::vector<Eigen::Vector3f>{query});
        utility::device_vector<int> i;
        utility::device_vector<float> d;
        int k = SearchKNN(q, knn, i, d);
        indices = i.to_host();
        distance2 = d.to_host();
        return k;
    }
    int SearchRadius(const Eigen::Vector3f &query, float radius, int max_nn, std::vector<int> &indices,
                     std::vector<float> &distance2) const {
        utility::device_vector<Eigen::Vector3f> q(std::vector<Eigen::Vector3f>{query});
        utility::device_vector<int> i;
        utility::device_vector<float> d;
        int k = SearchRadius(q, radius, max_nn, i, d);
        indices = i.to_host();
        distance2 = d.to_host();
        return k;
    }

private:
    void release() {
        if (ix_) { cphb_stream_synchronize(nullptr); cphb_index_destroy(ix_); ix_ = nullptr; }
    }
    cphb_index *ix_ = nullptr;
    size_t n_ = 0;
};
}  // namespace knn

// --------------------------------------------------------------------------- camera
namespace camera {
/// camera::PinholeCameraIntrinsicParameters (pinhole_camera_intrinsic.h:33-40): only PrimeSenseDefault is provided
enum class PinholeCameraIntrinsicParameters { PrimeSenseDefault = 0 };
/// camera::PinholeCameraIntrinsic (pinhole_camera_intrinsic.h): width_, height_ and the 3x3 intrinsic_matrix_
class PinholeCameraIntrinsic {
public:
    PinholeCameraIntrinsic() {}
    /// PrimeSenseDefault: 640 x 480, fx = fy = 525, cx = 319.5, cy = 239.5
    PinholeCameraIntrinsic(PinholeCameraIntrinsicParameters) { SetIntrinsics(640, 480, 525.0f, 525.0f, 319.5f, 239.5f); }
    PinholeCameraIntrinsic(int width, int height, float fx, float fy, float cx, float cy) { SetIntrinsics(width, height, fx, fy, cx, cy); }
    void SetIntrinsics(int width, int height, float fx, float fy, float cx, float cy) {
        width_ = width;
        height_ = height;
        intrinsic_matrix_ = Eigen::Matrix3f::Identity();
        intrinsic_matrix_(0, 0) = fx;
        intrinsic_matrix_(1, 1) = fy;
        intrinsic_matrix_(0, 2) = cx;
        intrinsic_matrix_(1, 2) = cy;
    }
    std::pair<float, float> GetFocalLength() const { return std::make_pair(intrinsic_matrix_(0, 0), intrinsic_matrix_(1, 1)); }
    std::pair<float, float> GetPrincipalPoint() const { return std::make_pair(intrinsic_matrix_(0, 2), intrinsic_matrix_(1, 2)); }
    bool IsValid() const { return width_ > 0 && height_ > 0; }

public:
    int width_ = -1;
    int height_ = -1;
    Eigen::Matrix3f intrinsic_matrix_;
};
/// camera::PinholeCameraParameters (pinhole_camera_parameters.h): intrinsic_ and the world-to-camera extrinsic_
class PinholeCameraParameters {
public:
    PinholeCameraIntrinsic intrinsic_;
    Eigen::Matrix4f extrinsic_ = Eigen::Matrix4f::Identity();
};
}  // namespace camera

// --------------------------------------------------------------------------- geometry
namespace geometry {
namespace detail {
inline Eigen::Vector3f v3(float x, float y, float z) { return Eigen::Vector3f(x, y, z); }
// ascending int32 indices from a cphb_*_point_indices call, widened to the reference's size_t
template <class F>
inline utility::device_vector<size_t> point_indices(const utility::device_vector<Eigen::Vector3f> &points, F call) {
    utility::device_vector<size_t> out;
    const size_t n = points.size();
    if (n == 0) return out;
    utility::device_vector<int32_t> idx(n);
    size_t m = 0;
    utility::check(call(reinterpret_cast<const float *>(points.data()), n, idx.data(), &m));
    idx.resize(m);
    std::vector<int32_t> h32 = idx.to_host();
    out = std::vector<size_t>(h32.begin(), h32.end());
    return out;
}
}  // namespace detail

template <int Dim>
class AxisAlignedBoundingBox;

/// geometry::OrientedBoundingBox (boundingvolume.h:40-139): center_, R_ (columns are the box axes), extent_.
class OrientedBoundingBox {
public:
    OrientedBoundingBox() : center_(0, 0, 0), R_(Eigen::Matrix3f::Identity()), extent_(0, 0, 0), color_(0, 0, 0) {}
    OrientedBoundingBox(const Eigen::Vector3f &center, const Eigen::Matrix3f &R, const Eigen::Vector3f &extent)
        : center_(center), R_(R), extent_(extent), color_(0, 0, 0) {}
    float Volume() const { return extent_(0) * extent_(1) * extent_(2); }  // boundingvolume.cu:176-178
    bool IsEmpty() const { return Volume() <= 0; }
    Eigen::Vector3f GetCenter() const { return center_; }
    Eigen::Vector3f GetMinBound() const { return bound(-1.f); }  // boundingvolume.cu:115-123: center -+ 0.5 |R extent|
    Eigen::Vector3f GetMaxBound() const { return bound(1.f); }
    /// GetBoxPoints (boundingvolume.cu:180-194): axis k = R.col(k) * (extent(k) / 2), corners center -+ x -+ y -+ z
    std::array<Eigen::Vector3f, 8> GetBoxPoints() const {
        float ax[3][3];
        for (int k = 0; k < 3; ++k)
            for (int r = 0; r < 3; ++r) ax[k][r] = R_(r, k) * (extent_(k) / 2);
        static const int S[8][3] = {{-1, -1, -1}, {1, -1, -1}, {-1, 1, -1}, {-1, -1, 1}, {1, 1, 1}, {-1, 1, 1}, {1, -1, 1}, {1, 1, -1}};
        std::array<Eigen::Vector3f, 8> p;
        for (int i = 0; i < 8; ++i) {
            float v[3];
            for (int r = 0; r < 3; ++r) {
                v[r] = center_(r);
                for (int k = 0; k < 3; ++k) v[r] = S[i][k] > 0 ? v[r] + ax[k][r] : v[r] - ax[k][r];
            }
            p[i] = detail::v3(v[0], v[1], v[2]);
        }
        return p;
    }
    /// GetPointIndicesWithinBoundingBox (boundingvolume.cu:228-244): the six determinant plane tests (cphb_obb_point_indices)
    utility::device_vector<size_t> GetPointIndicesWithinBoundingBox(const utility::device_vector<Eigen::Vector3f> &points) const {
        const auto bp = GetBoxPoints();
        float box[24];
        for (int i = 0; i < 8; ++i)
            for (int r = 0; r < 3; ++r) box[3 * i + r] = bp[i](r);
        return detail::point_indices(points, [&](const float *p, size_t n, int32_t *idx, size_t *m) {
            return cphb_obb_point_indices(p, n, box, idx, m, nullptr);
        });
    }
    static OrientedBoundingBox CreateFromAxisAlignedBoundingBox(const AxisAlignedBoundingBox<3> &aabox);
    /// CreateFromPoints (boundingvolume.cu:219-269; cphb_oriented_bounding_box): PCA axes by descending eigenvalue, each
    /// signed so its largest-magnitude component is positive; the zero box with R = I for no points.
    static OrientedBoundingBox CreateFromPoints(const utility::device_vector<Eigen::Vector3f> &points) {
        float c[3], R[9], e[3];
        utility::check(cphb_oriented_bounding_box(reinterpret_cast<const float *>(points.data()), points.size(), c, R, e, nullptr));
        Eigen::Matrix3f M;
        for (int r = 0; r < 3; ++r)
            for (int k = 0; k < 3; ++k) M(r, k) = R[3 * r + k];
        return OrientedBoundingBox(detail::v3(c[0], c[1], c[2]), M, detail::v3(e[0], e[1], e[2]));
    }

public:
    Eigen::Vector3f center_;
    Eigen::Matrix3f R_;
    Eigen::Vector3f extent_;
    Eigen::Vector3f color_;

private:
    Eigen::Vector3f bound(float sign) const {
        float v[3];
        for (int r = 0; r < 3; ++r) {
            const float size = std::fabs(R_(r, 0) * extent_(0) + R_(r, 1) * extent_(1) + R_(r, 2) * extent_(2));
            v[r] = center_(r) + sign * 0.5f * size;
        }
        return detail::v3(v[0], v[1], v[2]);
    }
};

/// geometry::AxisAlignedBoundingBox<3> (boundingvolume.h:141-232): min_bound_, max_bound_.
template <>
class AxisAlignedBoundingBox<3> {
public:
    AxisAlignedBoundingBox() : min_bound_(0, 0, 0), max_bound_(0, 0, 0), color_(0, 0, 0) {}
    AxisAlignedBoundingBox(const Eigen::Vector3f &min_bound, const Eigen::Vector3f &max_bound)
        : min_bound_(min_bound), max_bound_(max_bound), color_(0, 0, 0) {}
    Eigen::Vector3f GetMinBound() const { return min_bound_; }
    Eigen::Vector3f GetMaxBound() const { return max_bound_; }
    Eigen::Vector3f GetCenter() const {  // boundingvolume.cu:293-296
        return detail::v3((min_bound_(0) + max_bound_(0)) * 0.5f, (min_bound_(1) + max_bound_(1)) * 0.5f,
                          (min_bound_(2) + max_bound_(2)) * 0.5f);
    }
    Eigen::Vector3f GetExtent() const {
        return detail::v3(max_bound_(0) - min_bound_(0), max_bound_(1) - min_bound_(1), max_bound_(2) - min_bound_(2));
    }
    Eigen::Vector3f GetHalfExtent() const {
        const Eigen::Vector3f e = GetExtent();
        return detail::v3(e(0) * 0.5f, e(1) * 0.5f, e(2) * 0.5f);
    }
    float GetMaxExtent() const {
        const Eigen::Vector3f e = GetExtent();
        return std::max(e(0), std::max(e(1), e(2)));
    }
    float Volume() const {
        const Eigen::Vector3f e = GetExtent();
        return e(0) * e(1) * e(2);
    }
    bool IsEmpty() const { return Volume() <= 0; }
    /// GetBoxPoints (boundingvolume.cu:388-401)
    std::array<Eigen::Vector3f, 8> GetBoxPoints() const {
        const Eigen::Vector3f e = GetExtent(), &lo = min_bound_, &hi = max_bound_;
        return {lo, detail::v3(lo(0) + e(0), lo(1) + 0.f, lo(2) + 0.f), detail::v3(lo(0) + 0.f, lo(1) + e(1), lo(2) + 0.f),
                detail::v3(lo(0) + 0.f, lo(1) + 0.f, lo(2) + e(2)), hi, detail::v3(hi(0) - e(0), hi(1) - 0.f, hi(2) - 0.f),
                detail::v3(hi(0) - 0.f, hi(1) - e(1), hi(2) - 0.f), detail::v3(hi(0) - 0.f, hi(1) - 0.f, hi(2) - e(2))};
    }
    /// GetPointIndicesWithinBoundingBox (boundingvolume.cu:413-425): inclusive bounds, NaN points kept
    utility::device_vector<size_t> GetPointIndicesWithinBoundingBox(const utility::device_vector<Eigen::Vector3f> &points) const {
        const float lo[3] = {min_bound_(0), min_bound_(1), min_bound_(2)}, hi[3] = {max_bound_(0), max_bound_(1), max_bound_(2)};
        return detail::point_indices(points, [&](const float *p, size_t n, int32_t *idx, size_t *m) {
            return cphb_aabb_point_indices(p, n, lo, hi, idx, m, nullptr);
        });
    }
    OrientedBoundingBox GetOrientedBoundingBox() const { return OrientedBoundingBox::CreateFromAxisAlignedBoundingBox(*this); }
    /// CreateFromPoints (boundingvolume.cu:378-395): the min / max bound, the zero box for no points
    static AxisAlignedBoundingBox<3> CreateFromPoints(const utility::device_vector<Eigen::Vector3f> &points) {
        float mn[3] = {0, 0, 0}, mx[3] = {0, 0, 0};
        if (!points.empty())
            utility::check(cphb_min_max_bound(reinterpret_cast<const float *>(points.data()), points.size(), mn, mx, nullptr));
        return AxisAlignedBoundingBox<3>(detail::v3(mn[0], mn[1], mn[2]), detail::v3(mx[0], mx[1], mx[2]));
    }

public:
    Eigen::Vector3f min_bound_, max_bound_, color_;
};

inline OrientedBoundingBox OrientedBoundingBox::CreateFromAxisAlignedBoundingBox(const AxisAlignedBoundingBox<3> &aabox) {
    return OrientedBoundingBox(aabox.GetCenter(), Eigen::Matrix3f::Identity(), aabox.GetExtent());  // boundingvolume.cu:209-217
}

/// geometry::PointCloud (pointcloud.h:43-263), hot-path subset.
class OccupancyGrid;
class Image;
class RGBDImage;
class TriangleMesh;
class PointCloud {
public:
    PointCloud() {}
    /// PointCloud::CreateFromOccupancyGrid (pointcloud_factory.cu:418-430), defined after OccupancyGrid
    static std::shared_ptr<PointCloud> CreateFromOccupancyGrid(const OccupancyGrid &occgrid);
    /// PointCloud::CreateFromDepthImage (pointcloud_factory.cu:43-105, 329-350), defined after RGBDImage: the point of
    /// every stride-th pixel of every stride-th row with depth > 0, in pixel order.  depth: 1-channel uint16 (raw /
    /// int(depth_scale), 0 where that is >= int(depth_trunc)) or float32 metres; another format, stride < 1 or a
    /// singular extrinsic throws.
    static std::shared_ptr<PointCloud> CreateFromDepthImage(const Image &depth, const camera::PinholeCameraIntrinsic &intrinsic,
                                                            const Eigen::Matrix4f &extrinsic = Eigen::Matrix4f::Identity(),
                                                            float depth_scale = 1000.0f, float depth_trunc = 1000.0f, int stride = 1);
    /// PointCloud::CreateFromRGBDImage (pointcloud_factory.cu:107-200, 352-373), defined after RGBDImage: a point and
    /// colour (RGB8 c / 255, Gray32 (g, g, g)) per pixel with depth > 0 (and < depth_cutoff when that is > 0);
    /// compute_normals gives structured normals (0 on the border rows and columns); project_valid_depth_only = false
    /// keeps one row per pixel, NaN where there is no point.
    static std::shared_ptr<PointCloud> CreateFromRGBDImage(const RGBDImage &image, const camera::PinholeCameraIntrinsic &intrinsic,
                                                           const Eigen::Matrix4f &extrinsic = Eigen::Matrix4f::Identity(),
                                                           bool project_valid_depth_only = true, float depth_cutoff = -1.0f,
                                                           bool compute_normals = false);
    PointCloud(const std::vector<Eigen::Vector3f> &points) : points_(points) {}
    virtual ~PointCloud() {}
    bool IsEmpty() const { return points_.empty(); }
    bool HasPoints() const { return !points_.empty(); }
    bool HasNormals() const { return !points_.empty() && normals_.size() == points_.size(); }          // pointcloud.h:82-94
    bool HasColors() const { return !points_.empty() && colors_.size() == points_.size(); }
    bool HasCovariances() const { return !points_.empty() && covariances_.size() == points_.size(); }
    void SetPoints(const std::vector<Eigen::Vector3f> &p) { points_ = p; }
    void SetNormals(const std::vector<Eigen::Vector3f> &p) { normals_ = p; }
    void SetColors(const std::vector<Eigen::Vector3f> &p) { colors_ = p; }
    std::vector<Eigen::Vector3f> GetPoints() const { return points_.to_host(); }
    std::vector<Eigen::Vector3f> GetNormals() const { return normals_.to_host(); }
    std::vector<Eigen::Vector3f> GetColors() const { return colors_.to_host(); }

    Eigen::Vector3f GetMinBound() const { return bound(0); }  // pointcloud.cu:205
    Eigen::Vector3f GetMaxBound() const { return bound(1); }

    PointCloud &Transform(const Eigen::Matrix4f &T) {  // pointcloud.cu:293-299
        float t[16];
        utility::to_row_major(T, t);
        if (!points_.empty())
            utility::check(cphb_transform(fp(points_), HasNormals() ? fp(normals_) : nullptr,
                                          HasCovariances() ? fp(covariances_) : nullptr, 1, points_.size(), t, nullptr));
        utility::check(cphb_stream_synchronize(nullptr));
        return *this;
    }
    std::shared_ptr<PointCloud> VoxelDownSample(float voxel_size) const {  // down_sample.cu:170-273
        auto out = std::make_shared<PointCloud>();
        if (voxel_size <= 0.0) { utility::LogWarning("[VoxelDownSample] voxel_size <= 0."); return out; }
        const size_t n = points_.size();
        if (n == 0) return out;
        const bool hn = HasNormals(), hc = HasColors();
        out->points_.resize(n);
        if (hn) out->normals_.resize(n);
        if (hc) out->colors_.resize(n);
        size_t m = 0;
        utility::check(cphb_voxel_down_sample(cfp(points_), hn ? cfp(normals_) : nullptr, hc ? cfp(colors_) : nullptr, n,
                                              voxel_size, fp(out->points_), hn ? fp(out->normals_) : nullptr,
                                              hc ? fp(out->colors_) : nullptr, &m, nullptr));
        out->points_.resize(m);
        if (hn) out->normals_.resize(m);
        if (hc) out->colors_.resize(m);
        return out;
    }
    bool EstimateNormals(const knn::KDTreeSearchParam &param = knn::KDTreeSearchParamKNN()) {  // estimate_normals.cu:82-127
        if (!HasNormals()) normals_.resize(points_.size());
        int knn = 0, max_nn = 0;
        float radius = 0.f;
        if (param.GetSearchType() == knn::KDTreeSearchParam::SearchType::Knn) knn = static_cast<const knn::KDTreeSearchParamKNN &>(param).knn_;
        else { radius = static_cast<const knn::KDTreeSearchParamRadius &>(param).radius_; max_nn = static_cast<const knn::KDTreeSearchParamRadius &>(param).max_nn_; }
        utility::check(cphb_estimate_normals(cfp(points_), points_.size(), knn, radius, max_nn, fp(normals_), nullptr));
        return true;
    }
    /// PointCloud::SelectByIndex (down_sample.cu:110-127).  Index vectors are size_t like the reference's.
    std::shared_ptr<PointCloud> SelectByIndex(const utility::device_vector<size_t> &indices, bool invert = false) const {
        std::vector<size_t> h = indices.to_host();
        const size_t n = points_.size();
        std::vector<int32_t> sel;
        if (invert) {  // sort + set_difference(0..n, indices) there: ascending complement
            std::vector<char> drop(n, 0);
            for (size_t i : h) if (i < n) drop[i] = 1;
            for (size_t i = 0; i < n; ++i) if (!drop[i]) sel.push_back((int32_t)i);
        } else {
            sel.reserve(h.size());
            for (size_t i : h) sel.push_back((int32_t)i);
        }
        utility::device_vector<int32_t> d;
        d = sel;
        return gather(d, sel.size());
    }
    /// PointCloud::RemoveRadiusOutliers (down_sample.cu:317-354) -> (filtered cloud, kept indices)
    std::tuple<std::shared_ptr<PointCloud>, utility::device_vector<size_t>> RemoveRadiusOutliers(size_t nb_points,
                                                                                                   float search_radius) const {
        if (nb_points < 1 || search_radius <= 0)
            utility::LogError("[RemoveRadiusOutliers] Illegal input parameters, number of points and radius must be positive");
        utility::device_vector<int32_t> kept(points_.size());
        size_t m = 0;
        if (!points_.empty())
            utility::check(cphb_remove_radius_outliers(cfp(points_), points_.size(), (int)nb_points, search_radius, kept.data(), &m,
                                                       nullptr));
        return finish_filter(kept, m);
    }
    /// PointCloud::RemoveStatisticalOutliers (down_sample.cu:356-438) -> (filtered cloud, kept indices)
    std::tuple<std::shared_ptr<PointCloud>, utility::device_vector<size_t>> RemoveStatisticalOutliers(size_t nb_neighbors,
                                                                                                        float std_ratio) const {
        if (nb_neighbors < 1 || std_ratio <= 0)
            utility::LogError("[RemoveStatisticalOutliers] Illegal input parameters, number of neighbors and standard deviation "
                              "ratio must be positive");
        utility::device_vector<int32_t> kept(points_.size());
        size_t m = 0;
        if (!points_.empty())
            utility::check(cphb_remove_statistical_outliers(cfp(points_), points_.size(), (int)nb_neighbors, std_ratio, kept.data(),
                                                            &m, nullptr, nullptr));
        return finish_filter(kept, m);
    }
    /// PointCloud::SegmentPlane (segmentation.cu:187-267) -> (plane [a, b, c, d], ascending inlier indices).  Every
    /// iteration draws its seed with ::rand() as the reference does, so srand() makes a run repeatable.
    std::tuple<Eigen::Vector4f, utility::device_vector<size_t>> SegmentPlane(float distance_threshold = 0.01f, size_t ransac_n = 3,
                                                                             size_t num_iterations = 100) const {
        utility::device_vector<size_t> inliers;
        if (ransac_n < 3) {
            utility::LogError("ransac_n should be set to higher than or equal to 3.");
            return std::make_tuple(Eigen::Vector4f(0.f, 0.f, 0.f, 0.f), std::move(inliers));
        }
        if (points_.size() < ransac_n) {
            utility::LogError("There must be at least 'ransac_n' points.");
            return std::make_tuple(Eigen::Vector4f(0.f, 0.f, 0.f, 0.f), std::move(inliers));
        }
        if (num_iterations > (size_t)std::numeric_limits<int>::max()) utility::check(CPHB_ERR_INVALID);
        std::vector<int32_t> seeds(num_iterations);
        for (int32_t &s : seeds) s = std::rand();
        utility::device_vector<int32_t> kept(points_.size());
        size_t m = 0;
        float h[4];
        utility::check(cphb_segment_plane(cfp(points_), points_.size(), distance_threshold, (int)ransac_n, (int)num_iterations,
                                          seeds.data(), h, kept.data(), &m, nullptr, nullptr, nullptr, nullptr));
        kept.resize(m);
        std::vector<int32_t> h32 = kept.to_host();
        inliers = std::vector<size_t>(h32.begin(), h32.end());
        return std::make_tuple(Eigen::Vector4f(h[0], h[1], h[2], h[3]), std::move(inliers));
    }
    /// PointCloud::FarthestPointDownSample (pointcloud.cu:301-338): num_samples points by farthest-point sampling from
    /// index 0, in pick order.  0 -> empty cloud, points_.size() -> a copy; more samples than points is logged and the
    /// loop runs anyway (the output repeats points), except on an empty cloud, where the result is empty.
    std::shared_ptr<PointCloud> FarthestPointDownSample(size_t num_samples) const {
        const size_t n = points_.size();
        if (num_samples == 0) return std::make_shared<PointCloud>();
        if (num_samples == n) return std::make_shared<PointCloud>(*this);
        if (num_samples > n) {
            char msg[128];
            std::snprintf(msg, sizeof(msg), "Illegal number of samples: %zu, must <= point size: %zu", num_samples, n);
            utility::LogError(msg);
            if (n == 0) return std::make_shared<PointCloud>();
        }
        utility::device_vector<int32_t> idx(num_samples);
        utility::check(cphb_farthest_point_down_sample(cfp(points_), n, num_samples, idx.data(), nullptr, nullptr));
        return gather(idx, num_samples);
    }
    /// PointCloud::ClusterDBSCAN (pointcloud.h:195-199, pointcloud_cluster.cu:84-179): labels, -1 = noise
    std::unique_ptr<utility::device_vector<int>> ClusterDBSCAN(float eps, size_t min_points, bool print_progress = false,
                                                               size_t max_edges = 100) const {
        (void)print_progress;
        auto labels = std::make_unique<utility::device_vector<int>>(points_.size());
        if (!points_.empty())
            utility::check(cphb_cluster_dbscan(cfp(points_), points_.size(), eps, (int)min_points, (int)max_edges,
                                               reinterpret_cast<int32_t *>(labels->data()), nullptr, nullptr));
        return labels;
    }
    /// PointCloud::GaussianFilter (pointcloud.cu:387-433)
    std::shared_ptr<PointCloud> GaussianFilter(float search_radius, float sigma2, size_t num_max_search_points = 50) const {
        auto out = std::make_shared<PointCloud>();
        if (search_radius <= 0 || sigma2 <= 0 || num_max_search_points <= 0) {
            utility::LogError("[GaussianFilter] Illegal input parameters, radius and sigma2 must be positive.");
            return out;
        }
        const size_t n = points_.size();
        if (n == 0) return out;
        const bool hn = HasNormals(), hc = HasColors();
        out->points_.resize(n);
        if (hn) out->normals_.resize(n);
        if (hc) out->colors_.resize(n);
        size_t m = 0;
        utility::check(cphb_gaussian_filter(cfp(points_), hn ? cfp(normals_) : nullptr, hc ? cfp(colors_) : nullptr, n, search_radius,
                                            sigma2, (int)num_max_search_points, fp(out->points_), hn ? fp(out->normals_) : nullptr,
                                            hc ? fp(out->colors_) : nullptr, &m, nullptr));
        return out;
    }
    AxisAlignedBoundingBox<3> GetAxisAlignedBoundingBox() const { return AxisAlignedBoundingBox<3>::CreateFromPoints(points_); }
    OrientedBoundingBox GetOrientedBoundingBox() const { return OrientedBoundingBox::CreateFromPoints(points_); }
    /// PointCloud::Crop (pointcloud.cu:340-356): an empty box is logged and the crop still runs
    std::shared_ptr<PointCloud> Crop(const AxisAlignedBoundingBox<3> &bbox) const {
        if (bbox.IsEmpty()) utility::LogError("[CropPointCloud] AxisAlignedBoundingBox either has zeros size, or has wrong bounds.");
        return SelectByIndex(bbox.GetPointIndicesWithinBoundingBox(points_));
    }
    std::shared_ptr<PointCloud> Crop(const OrientedBoundingBox &bbox) const {
        if (bbox.IsEmpty()) utility::LogError("[CropPointCloud] AxisAlignedBoundingBox either has zeros size, or has wrong bounds.");
        return SelectByIndex(bbox.GetPointIndicesWithinBoundingBox(points_));
    }
    /// PointCloud::PassThroughFilter (pointcloud.cu:436-460): min_bound <= p(axis_no) <= max_bound (NaN kept); axis_no >= 3
    /// is logged and gives an empty cloud.  Like the reference's copy-and-compact, the covariances survive only when no row
    /// is removed.
    std::shared_ptr<PointCloud> PassThroughFilter(size_t axis_no, float min_bound, float max_bound) {
        if (axis_no >= 3) {
            utility::LogError("[PassThroughFilter] Illegal input parameters, axis_no must be 0, 1 or 2.");
            return std::make_shared<PointCloud>();
        }
        float lo[3] = {-INFINITY, -INFINITY, -INFINITY}, hi[3] = {INFINITY, INFINITY, INFINITY};
        lo[axis_no] = min_bound;
        hi[axis_no] = max_bound;
        utility::device_vector<int32_t> kept(points_.size());
        size_t m = 0;
        if (!points_.empty())
            utility::check(cphb_aabb_point_indices(cfp(points_), points_.size(), lo, hi, kept.data(), &m, nullptr));
        auto out = gather(kept, m);
        if (m == points_.size() && HasCovariances()) out->covariances_ = covariances_;
        return out;
    }
    /// PointCloud::RemoveNoneFinitePoints (pointcloud.cu:359-385), in place: points, normals and colours are compacted;
    /// when rows are removed the covariances no longer match and are dropped
    PointCloud &RemoveNoneFinitePoints(bool remove_nan = true, bool remove_infinite = true) {
        const size_t n = points_.size();
        if (n == 0) return *this;
        utility::device_vector<int32_t> kept(n);
        size_t m = 0;
        utility::check(cphb_finite_point_indices(cfp(points_), n, remove_nan, remove_infinite, kept.data(), &m, nullptr));
        if (m == n) return *this;
        const bool hn = HasNormals(), hc = HasColors();
        auto out = gather(kept, m);
        points_ = std::move(out->points_);
        if (hn) normals_ = std::move(out->normals_);
        if (hc) colors_ = std::move(out->colors_);
        covariances_.clear();
        color_gradient_.clear();
        return *this;
    }
    /// PointCloud::UniformDownSample (down_sample.cu:275-300): rows 0, k, 2k, ... -- n / k of them; k == 0 is logged and
    /// gives an empty cloud
    std::shared_ptr<PointCloud> UniformDownSample(size_t every_k_points) const {
        auto out = std::make_shared<PointCloud>();
        if (every_k_points == 0) {
            utility::LogError("[UniformDownSample] Illegal sample rate.");
            return out;
        }
        const size_t n = points_.size(), m = n / every_k_points;
        if (m == 0) return out;
        const bool hn = HasNormals(), hc = HasColors();
        out->points_.resize(m);
        if (hn) out->normals_.resize(m);
        if (hc) out->colors_.resize(m);
        size_t got = 0;
        utility::check(cphb_uniform_down_sample(cfp(points_), hn ? cfp(normals_) : nullptr, hc ? cfp(colors_) : nullptr, n,
                                                every_k_points, fp(out->points_), hn ? fp(out->normals_) : nullptr,
                                                hc ? fp(out->colors_) : nullptr, &got, nullptr));
        utility::check(cphb_stream_synchronize(nullptr));
        return out;
    }
    /// PointCloud::NormalizeNormals (pointcloud.cu:282-285), in place
    PointCloud &NormalizeNormals() {
        if (!normals_.empty()) utility::check(cphb_normalize_normals(fp(normals_), normals_.size(), nullptr));
        utility::check(cphb_stream_synchronize(nullptr));
        return *this;
    }
    /// PointCloud::OrientNormalsToAlignWithDirection (estimate_normals.cu:129-141), in place
    bool OrientNormalsToAlignWithDirection(const Eigen::Vector3f &orientation_reference = Eigen::Vector3f(0.f, 0.f, 1.f)) {
        if (!HasNormals()) {
            utility::LogWarning("[OrientNormalsToAlignWithDirection] No normals in the PointCloud. Call EstimateNormals() first.");
            return false;
        }
        const float r[3] = {orientation_reference(0), orientation_reference(1), orientation_reference(2)};
        utility::check(cphb_orient_normals(fp(normals_), normals_.size(), r, nullptr));
        utility::check(cphb_stream_synchronize(nullptr));
        return true;
    }
    cphb_cloud view() const {
        cphb_cloud c;
        std::memset(&c, 0, sizeof(c));
        c.points = cfp(points_);
        c.n = points_.size();
        c.normals = HasNormals() ? cfp(normals_) : nullptr;
        c.colors = HasColors() ? cfp(colors_) : nullptr;
        c.covariances = HasCovariances() ? cfp(covariances_) : nullptr;
        c.color_gradient = (!points_.empty() && color_gradient_.size() == points_.size()) ? cfp(color_gradient_) : nullptr;
        c.cov_col_major = 1;  // Eigen::Matrix3f default storage
        return c;
    }

public:
    utility::device_vector<Eigen::Vector3f> points_, normals_, colors_;
    utility::device_vector<Eigen::Matrix3f> covariances_;
    utility::device_vector<Eigen::Vector3f> color_gradient_;  // PointCloudForColoredICP (colored_icp.cu:36-40)

private:
    template <class V> static float *fp(V &v) { return reinterpret_cast<float *>(v.data()); }
    template <class V> static const float *cfp(const V &v) { return reinterpret_cast<const float *>(v.data()); }
    std::shared_ptr<PointCloud> gather(const utility::device_vector<int32_t> &idx, size_t m) const {
        auto out = std::make_shared<PointCloud>();
        if (m == 0 || points_.empty()) return out;
        const bool hn = HasNormals(), hc = HasColors();
        out->points_.resize(m);
        if (hn) out->normals_.resize(m);
        if (hc) out->colors_.resize(m);
        utility::check(cphb_select_by_index(cfp(points_), hn ? cfp(normals_) : nullptr, hc ? cfp(colors_) : nullptr, points_.size(),
                                            idx.data(), m, fp(out->points_), hn ? fp(out->normals_) : nullptr,
                                            hc ? fp(out->colors_) : nullptr, nullptr));
        utility::check(cphb_stream_synchronize(nullptr));
        return out;
    }
    std::tuple<std::shared_ptr<PointCloud>, utility::device_vector<size_t>> finish_filter(utility::device_vector<int32_t> &kept,
                                                                                            size_t m) const {
        auto out = gather(kept, m);
        kept.resize(m);
        std::vector<int32_t> h32 = kept.to_host();
        std::vector<size_t> h(h32.begin(), h32.end());  // the reference hands back device_vector<size_t>
        utility::device_vector<size_t> idx;
        idx = h;
        return std::make_tuple(out, std::move(idx));
    }
    Eigen::Vector3f bound(int which) const {
        float mn[3] = {0, 0, 0}, mx[3] = {0, 0, 0};
        if (!points_.empty()) utility::check(cphb_min_max_bound(cfp(points_), points_.size(), mn, mx, nullptr));
        return which ? Eigen::Vector3f(mx[0], mx[1], mx[2]) : Eigen::Vector3f(mn[0], mn[1], mn[2]);
    }
};

/// geometry::Voxel (voxelgrid.h:48-62)
class Voxel {
public:
    Voxel() {}
    Voxel(const Eigen::Vector3i &grid_index) : grid_index_(grid_index) {}
    Voxel(const Eigen::Vector3i &grid_index, const Eigen::Vector3f &color) : grid_index_(grid_index), color_(color) {}
    Eigen::Vector3i grid_index_ = Eigen::Vector3i(0, 0, 0);
    Eigen::Vector3f color_ = Eigen::Vector3f(1.0f, 1.0f, 1.0f);
};

/// geometry::Image (image.h) as a holder of pixels: width_ x height_ x num_of_channels_ channels of bytes_per_channel_
/// bytes each, row-major in data_ (device).  Carving samples a 1-channel float32 image; filters, pyramids and IO are not
/// part of this engine.
class Image {
public:
    Image &Prepare(int width, int height, int num_of_channels, int bytes_per_channel) {
        width_ = width;
        height_ = height;
        num_of_channels_ = num_of_channels;
        bytes_per_channel_ = bytes_per_channel;
        data_.resize((size_t)width * height * num_of_channels * bytes_per_channel);
        return *this;
    }
    bool IsEmpty() const { return data_.size() == 0; }

public:
    int width_ = 0;
    int height_ = 0;
    int num_of_channels_ = 0;
    int bytes_per_channel_ = 0;
    utility::device_vector<uint8_t> data_;
};

/// geometry::VoxelGrid (voxelgrid.h:84-160): creation from a point cloud (voxelgrid_factory.cu:164-228) or a triangle
/// mesh (:229-281) and the
/// accessors, CreateDense, CheckIfIncluded, carving, += / AddVoxels, painting, SelectByIndex and CreateFromOccupancyGrid
/// (voxelgrid.cu:235-475).  Keys and colours are kept as two device vectors (the reference zips keys with
/// Voxel{grid_index, color}); GetVoxels() hands back the reference's pair.
class VoxelGrid {
public:
    bool HasVoxels() const { return voxels_keys_.size() > 0; }
    bool HasColors() const { return true; }  // voxelgrid.h:112-114
    bool IsEmpty() const { return !HasVoxels(); }
    std::pair<std::vector<Eigen::Vector3i>, std::vector<Voxel>> GetVoxels() const {
        std::vector<Eigen::Vector3i> k = voxels_keys_.to_host();
        std::vector<Eigen::Vector3f> c = voxels_colors_.to_host();
        std::vector<Voxel> v(k.size());
        for (size_t i = 0; i < k.size(); ++i) v[i] = Voxel(k[i], c[i]);
        return std::make_pair(std::move(k), std::move(v));
    }
    Eigen::Vector3i GetVoxel(const Eigen::Vector3f &point) const {  // voxelgrid.cu:338-341
        return Eigen::Vector3i((int)std::floor((point[0] - origin_[0]) / voxel_size_), (int)std::floor((point[1] - origin_[1]) / voxel_size_),
                               (int)std::floor((point[2] - origin_[2]) / voxel_size_));
    }
    static std::shared_ptr<VoxelGrid> CreateFromPointCloudWithinBounds(const PointCloud &input, float voxel_size,
                                                                       const Eigen::Vector3f &min_bound,
                                                                       const Eigen::Vector3f &max_bound) {
        auto out = std::make_shared<VoxelGrid>();
        if (voxel_size <= 0.0) utility::LogError("[VoxelGridFromPointCloud] voxel_size <= 0.");
        out->voxel_size_ = voxel_size;
        out->origin_ = min_bound;
        const size_t n = input.points_.size();
        if (n == 0) return out;
        const float mn[3] = {min_bound[0], min_bound[1], min_bound[2]}, mx[3] = {max_bound[0], max_bound[1], max_bound[2]};
        out->voxels_keys_.resize(n);
        out->voxels_colors_.resize(n);
        size_t m = 0;
        utility::check(cphb_voxel_grid_from_point_cloud(
                reinterpret_cast<const float *>(input.points_.data()),
                input.HasColors() ? reinterpret_cast<const float *>(input.colors_.data()) : nullptr, n, voxel_size, mn, mx,
                reinterpret_cast<int32_t *>(out->voxels_keys_.data()), reinterpret_cast<float *>(out->voxels_colors_.data()), &m,
                nullptr));
        out->voxels_keys_.resize(m);
        out->voxels_colors_.resize(m);
        return out;
    }
    static std::shared_ptr<VoxelGrid> CreateFromPointCloud(const PointCloud &input, float voxel_size) {  // :221-228
        const Eigen::Vector3f lo = input.GetMinBound(), hi = input.GetMaxBound();
        const float h = voxel_size * 0.5f;
        return CreateFromPointCloudWithinBounds(input, voxel_size, Eigen::Vector3f(lo[0] - h, lo[1] - h, lo[2] - h),
                                                Eigen::Vector3f(hi[0] + h, hi[1] + h, hi[2] + h));
    }
    /// CreateDense (voxelgrid_factory.cu:134-162): int(round(extent / voxel_size)) voxels per axis in lexicographic order
    static std::shared_ptr<VoxelGrid> CreateDense(const Eigen::Vector3f &origin, float voxel_size, float width, float height, float depth) {
        auto out = std::make_shared<VoxelGrid>();
        out->voxel_size_ = voxel_size;
        out->origin_ = origin;
        size_t n = 0;
        utility::check(cphb_voxel_grid_create_dense(voxel_size, width, height, depth, nullptr, nullptr, 0, &n, nullptr));
        out->voxels_keys_.resize(n);
        out->voxels_colors_.resize(n);
        if (n)
            utility::check(cphb_voxel_grid_create_dense(voxel_size, width, height, depth, out->keys(), out->colors(), n, &n, nullptr));
        return out;
    }
    /// CreateFromOccupancyGrid (voxelgrid_factory.cu:283-305), defined after OccupancyGrid
    static std::shared_ptr<VoxelGrid> CreateFromOccupancyGrid(const OccupancyGrid &input);
    /// CreateFromTriangleMeshWithinBounds (voxelgrid_factory.cu:229-272): int(round(extent / voxel_size)) cells per axis
    /// from min_bound; a cell is a voxel when Akenine-Moeller's triangle/box test says some triangle meets it.  The cell
    /// tested for key k is centred at (k + 0.5) voxel_size + origin, the cell GetVoxel gives (the reference tests the box
    /// centred on the lower corner).  A bad vertex index, voxel size, bounds or count throws.  Defined after TriangleMesh.
    static std::shared_ptr<VoxelGrid> CreateFromTriangleMeshWithinBounds(const TriangleMesh &input, float voxel_size,
                                                                         const Eigen::Vector3f &min_bound, const Eigen::Vector3f &max_bound);
    /// CreateFromTriangleMesh (voxelgrid_factory.cu:274-281): the mesh's vertex bounds widened by half a voxel
    static std::shared_ptr<VoxelGrid> CreateFromTriangleMesh(const TriangleMesh &input, float voxel_size);
    /// CheckIfIncluded (voxelgrid.cu:365-376): whether each query's GetVoxel cell is a voxel (false for non-finite queries)
    std::vector<bool> CheckIfIncluded(const std::vector<Eigen::Vector3f> &queries) const {
        std::vector<bool> out(queries.size(), false);
        if (queries.empty()) return out;
        utility::device_vector<Eigen::Vector3f> q(queries);
        utility::device_vector<uint8_t> d(queries.size());
        const float o[3] = {origin_[0], origin_[1], origin_[2]};
        utility::check(cphb_voxel_grid_check_if_included(keys(), voxels_keys_.size(), voxel_size_, o,
                                                         reinterpret_cast<const float *>(q.data()), q.size(), d.data(), nullptr));
        const auto h = d.to_host();
        for (size_t i = 0; i < h.size(); ++i) out[i] = h[i] != 0;
        return out;
    }
    /// GetVoxelCenterCoordinate (voxelgrid.cu:343-354): the zero vector when idx is not a voxel, as in the reference
    Eigen::Vector3f GetVoxelCenterCoordinate(const Eigen::Vector3i &idx) const {
        const int32_t k[3] = {idx[0], idx[1], idx[2]};
        int found = 0;
        utility::check(cphb_voxel_grid_has_key(keys(), voxels_keys_.size(), k, &found, nullptr));
        if (!found) return Eigen::Vector3f(0.f, 0.f, 0.f);
        return Eigen::Vector3f(((float)idx[0] + 0.5f) * voxel_size_ + origin_[0], ((float)idx[1] + 0.5f) * voxel_size_ + origin_[1],
                               ((float)idx[2] + 0.5f) * voxel_size_ + origin_[2]);
    }
    /// GetVoxelBoundingPoints (voxelgrid.cu:356-363): corner j is the centre + r * (bit 1: x, bit 2: y, bit 0: z ? +1 : -1)
    std::array<Eigen::Vector3f, 8> GetVoxelBoundingPoints(const Eigen::Vector3i &index) const {
        const float r = voxel_size_ * 0.5f;
        const Eigen::Vector3f x = GetVoxelCenterCoordinate(index);
        std::array<Eigen::Vector3f, 8> p;
        for (int j = 0; j < 8; ++j)
            p[j] = Eigen::Vector3f(x[0] + ((j & 2) ? r : -r), x[1] + ((j & 4) ? r : -r), x[2] + ((j & 1) ? r : -r));
        return p;
    }
    /// CarveDepthMap (voxelgrid.cu:378-403)
    VoxelGrid &CarveDepthMap(const Image &depth_map, const camera::PinholeCameraParameters &camera_parameter,
                             bool keep_voxels_outside_image = false) {
        return carve(depth_map, camera_parameter, keep_voxels_outside_image, "depth_map");
    }
    /// CarveSilhouette (voxelgrid.cu:405-430): the reference applies the depth map's test (d > 0 and z >= d)
    VoxelGrid &CarveSilhouette(const Image &silhouette_mask, const camera::PinholeCameraParameters &camera_parameter,
                               bool keep_voxels_outside_image = false) {
        return carve(silhouette_mask, camera_parameter, keep_voxels_outside_image, "silhouette_mask");
    }
    /// operator+= (voxelgrid.cu:235-286): one voxel per key, colours of equal keys averaged (this grid's, then the other's)
    VoxelGrid &operator+=(const VoxelGrid &voxelgrid) {
        merge(voxelgrid, true);
        return *this;
    }
    VoxelGrid operator+(const VoxelGrid &voxelgrid) const { return (VoxelGrid(*this) += voxelgrid); }
    /// AddVoxel / AddVoxels (voxelgrid.cu:288-319): a key already present keeps its voxel
    void AddVoxel(const Voxel &voxel) { AddVoxels(std::vector<Voxel>{voxel}); }
    void AddVoxels(const std::vector<Voxel> &voxels) {
        VoxelGrid other;
        other.voxel_size_ = voxel_size_;
        other.origin_ = origin_;
        std::vector<Eigen::Vector3i> k(voxels.size());
        std::vector<Eigen::Vector3f> c(voxels.size());
        for (size_t i = 0; i < voxels.size(); ++i) {
            k[i] = voxels[i].grid_index_;
            c[i] = voxels[i].color_;
        }
        other.voxels_keys_ = k;
        other.voxels_colors_ = c;
        merge(other, false);
    }
    /// PaintUniformColor / PaintIndexedColor (voxelgrid.cu:321-336); an index outside [0, size) throws, nothing painted
    VoxelGrid &PaintUniformColor(const Eigen::Vector3f &color) {
        const float c[3] = {color[0], color[1], color[2]};
        utility::check(cphb_voxel_grid_paint(colors(), voxels_colors_.size(), nullptr, 0, c, nullptr));
        utility::check(cphb_stream_synchronize(nullptr));
        return *this;
    }
    VoxelGrid &PaintIndexedColor(const utility::device_vector<size_t> &indices, const Eigen::Vector3f &color) {
        const float c[3] = {color[0], color[1], color[2]};
        if (indices.size())
            utility::check(cphb_voxel_grid_paint(colors(), voxels_colors_.size(), reinterpret_cast<const int64_t *>(indices.data()),
                                                 indices.size(), c, nullptr));
        utility::check(cphb_stream_synchronize(nullptr));
        return *this;
    }
    /// SelectByIndex (voxelgrid.cu:432-475): invert gives the voxels not among indices, ascending (repeats allowed);
    /// an index outside [0, size) throws
    std::shared_ptr<VoxelGrid> SelectByIndex(const utility::device_vector<size_t> &indices, bool invert = false) const {
        auto out = std::make_shared<VoxelGrid>();
        out->voxel_size_ = voxel_size_;
        out->origin_ = origin_;
        const size_t rows = invert ? voxels_keys_.size() : indices.size();
        out->voxels_keys_.resize(rows);
        out->voxels_colors_.resize(rows);
        size_t m = 0;
        utility::check(cphb_voxel_grid_select_by_index(keys(), colors(), voxels_keys_.size(),
                                                       reinterpret_cast<const int64_t *>(indices.data()), indices.size(),
                                                       invert ? 1 : 0, out->keys(), out->colors(), &m, nullptr));
        out->voxels_keys_.resize(m);
        out->voxels_colors_.resize(m);
        return out;
    }

public:
    float voxel_size_ = 0.0f;
    Eigen::Vector3f origin_ = Eigen::Vector3f(0.f, 0.f, 0.f);
    utility::device_vector<Eigen::Vector3i> voxels_keys_;
    utility::device_vector<Eigen::Vector3f> voxels_colors_;

private:
    int32_t *keys() { return reinterpret_cast<int32_t *>(voxels_keys_.data()); }
    const int32_t *keys() const { return reinterpret_cast<const int32_t *>(voxels_keys_.data()); }
    float *colors() { return reinterpret_cast<float *>(voxels_colors_.data()); }
    // keys assigned without colours get the default (1, 1, 1)
    const float *colors() const {
        if (voxels_colors_.size() != voxels_keys_.size()) {
            auto &c = const_cast<utility::device_vector<Eigen::Vector3f> &>(voxels_colors_);
            c = std::vector<Eigen::Vector3f>(voxels_keys_.size(), Eigen::Vector3f(1.f, 1.f, 1.f));
        }
        return reinterpret_cast<const float *>(voxels_colors_.data());
    }
    VoxelGrid &carve(const Image &image, const camera::PinholeCameraParameters &cam, bool keep_outside, const char *what) {
        if (image.height_ != cam.intrinsic_.height_ || image.width_ != cam.intrinsic_.width_)
            throw std::runtime_error(std::string("[VoxelGrid] provided ") + what +
                                     " dimensions are not compatible with the provided camera_parameters");
        float K[9], E[16];
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) K[3 * r + c] = cam.intrinsic_.intrinsic_matrix_(r, c);
        utility::to_row_major(cam.extrinsic_, E);
        const float o[3] = {origin_[0], origin_[1], origin_[2]};
        const size_t n = voxels_keys_.size();
        utility::device_vector<Eigen::Vector3i> k(n);
        utility::device_vector<Eigen::Vector3f> c(n);
        size_t m = 0;
        utility::check(cphb_voxel_grid_carve(keys(), static_cast<const VoxelGrid *>(this)->colors(), n, voxel_size_, o,
                                             image.data_.data(), image.width_, image.height_, image.num_of_channels_,
                                             image.bytes_per_channel_, K, E, keep_outside ? 1 : 0,
                                             reinterpret_cast<int32_t *>(k.data()), reinterpret_cast<float *>(c.data()), &m, nullptr));
        k.resize(m);
        c.resize(m);
        voxels_keys_ = k;  // a copy of the m survivors, so a carved grid holds no more than it needs
        voxels_colors_ = c;
        return *this;
    }
    void merge(const VoxelGrid &other, bool average) {
        if (voxel_size_ != other.voxel_size_) throw std::runtime_error("[VoxelGrid] Could not combine VoxelGrid because voxel_size differs");
        if (origin_[0] != other.origin_[0] || origin_[1] != other.origin_[1] || origin_[2] != other.origin_[2])
            throw std::runtime_error("[VoxelGrid] Could not combine VoxelGrid because origin differs");
        const size_t n = voxels_keys_.size() + other.voxels_keys_.size();
        utility::device_vector<Eigen::Vector3i> k(n);
        utility::device_vector<Eigen::Vector3f> c(n);
        size_t m = 0;
        utility::check(cphb_voxel_grid_merge(keys(), static_cast<const VoxelGrid *>(this)->colors(), voxels_keys_.size(), other.keys(),
                                             other.colors(), other.voxels_keys_.size(), average ? 1 : 0,
                                             reinterpret_cast<int32_t *>(k.data()), reinterpret_cast<float *>(c.data()), &m, nullptr));
        k.resize(m);
        c.resize(m);
        voxels_keys_ = std::move(k);
        voxels_colors_ = std::move(c);
    }
};

/// geometry::OccupancyVoxel (occupancygrid.h:33-72)
class OccupancyVoxel {
public:
    OccupancyVoxel() {}
    OccupancyVoxel(const Eigen::Vector3i &grid_index, float prob_log) : grid_index_(grid_index), prob_log_(prob_log) {}
    Eigen::Vector3i grid_index_ = Eigen::Vector3i(0, 0, 0);           // (Vector3ui16 in the reference)
    Eigen::Vector3f color_ = Eigen::Vector3f(0.0f, 0.0f, 1.0f);
    float prob_log_ = std::numeric_limits<float>::quiet_NaN();
};

/// geometry::OccupancyGrid (occupancygrid.h:74-147): dense log-odds grid; Insert ray-casts a scan into it.  The members
/// the reference exposes (voxel_size_, origin_, the probability parameters) are public here too and are handed to the
/// engine at every call.  Extract* return host vectors of voxels (the reference returns device vectors of its 24-byte
/// voxel struct; the engine stores 4.1 bytes per cell and materialises voxels on request).
class OccupancyGrid {
public:
    OccupancyGrid() : OccupancyGrid(0.05f, 512) {}
    OccupancyGrid(float voxel_size, size_t resolution = 512, const Eigen::Vector3f &origin = Eigen::Vector3f(0.f, 0.f, 0.f))
        : voxel_size_(voxel_size), resolution_(resolution), origin_(origin) {
        const float o[3] = {origin[0], origin[1], origin[2]};
        utility::check(cphb_occgrid_create(voxel_size, (int)resolution, o, nullptr, &h_));
    }
    ~OccupancyGrid() { cphb_stream_synchronize(nullptr); cphb_occgrid_destroy(h_); }
    OccupancyGrid(const OccupancyGrid &) = delete;
    OccupancyGrid &operator=(const OccupancyGrid &) = delete;

    OccupancyGrid &Clear() { utility::check(cphb_occgrid_clear(h_, nullptr)); return *this; }
    bool HasVoxels() const { return true; }
    bool HasColors() const { return true; }
    Eigen::Vector3f GetMinBound() const {  // occupancygrid.cu:317-322
        int32_t lo[3], hi[3];
        utility::check(cphb_occgrid_bounds(h_, lo, hi, nullptr));
        const int h = (int)resolution_ / 2;
        return Eigen::Vector3f((lo[0] - h) * voxel_size_ + origin_[0], (lo[1] - h) * voxel_size_ + origin_[1], (lo[2] - h) * voxel_size_ + origin_[2]);
    }
    Eigen::Vector3f GetMaxBound() const {  // occupancygrid.cu:324-333
        int32_t lo[3], hi[3];
        utility::check(cphb_occgrid_bounds(h_, lo, hi, nullptr));
        const int h = (int)resolution_ / 2 - 1;
        return Eigen::Vector3f((hi[0] - h) * voxel_size_ + origin_[0], (hi[1] - h) * voxel_size_ + origin_[1], (hi[2] - h) * voxel_size_ + origin_[2]);
    }
    std::tuple<bool, OccupancyVoxel> GetVoxel(const Eigen::Vector3f &point) const {  // occupancygrid.cu:351-356
        sync();
        const float p[3] = {point[0], point[1], point[2]};
        int known = 0, gi[3];
        float prob = 0.f;
        utility::check(cphb_occgrid_get_voxel(h_, p, &known, &prob, gi, nullptr));
        return std::make_tuple(known != 0, OccupancyVoxel(Eigen::Vector3i(gi[0], gi[1], gi[2]), prob));
    }
    bool IsOccupied(const Eigen::Vector3f &point) const {
        auto r = GetVoxel(point);
        return std::get<0>(r) && std::get<1>(r).prob_log_ > occ_prob_thres_log_;
    }
    bool IsUnknown(const Eigen::Vector3f &point) const { return !std::get<0>(GetVoxel(point)); }
    std::shared_ptr<std::vector<OccupancyVoxel>> ExtractKnownVoxels() const { return extract(0); }
    std::shared_ptr<std::vector<OccupancyVoxel>> ExtractFreeVoxels() const { return extract(1); }
    std::shared_ptr<std::vector<OccupancyVoxel>> ExtractOccupiedVoxels() const { return extract(2); }
    OccupancyGrid &SetFreeArea(const Eigen::Vector3f &min_bound, const Eigen::Vector3f &max_bound) {
        sync();
        const float lo[3] = {min_bound[0], min_bound[1], min_bound[2]}, hi[3] = {max_bound[0], max_bound[1], max_bound[2]};
        utility::check(cphb_occgrid_set_free_area(h_, lo, hi, nullptr));
        return *this;
    }
    OccupancyGrid &Insert(const utility::device_vector<Eigen::Vector3f> &points, const Eigen::Vector3f &viewpoint, float max_range = -1.0f) {
        sync();
        const float v[3] = {viewpoint[0], viewpoint[1], viewpoint[2]};
        if (points.size()) utility::check(cphb_occgrid_insert(h_, reinterpret_cast<const float *>(points.data()), points.size(), v, max_range, nullptr));
        return *this;
    }
    OccupancyGrid &Insert(const std::vector<Eigen::Vector3f> &points, const Eigen::Vector3f &viewpoint, float max_range = -1.0f) {
        return Insert(utility::device_vector<Eigen::Vector3f>(points), viewpoint, max_range);
    }
    OccupancyGrid &Insert(const PointCloud &pointcloud, const Eigen::Vector3f &viewpoint, float max_range = -1.0f) {
        return Insert(pointcloud.points_, viewpoint, max_range);
    }
    OccupancyGrid &AddVoxel(const Eigen::Vector3i &voxel, bool occupied = false) {  // occupancygrid.cu:554-577
        sync();
        const int32_t v[3] = {voxel[0], voxel[1], voxel[2]};
        if (cphb_occgrid_add_voxel(h_, v, occupied ? 1 : 0, nullptr) != CPHB_OK)
            utility::LogError("[OccupancyGrid] a provided voxeld is not occupancy grid range.");
        return *this;
    }
    OccupancyGrid &AddVoxels(const utility::device_vector<Eigen::Vector3i> &voxels, bool occupied = false) {
        sync();
        if (voxels.size()) utility::check(cphb_occgrid_add_voxels(h_, reinterpret_cast<const int32_t *>(voxels.data()), voxels.size(), occupied ? 1 : 0, nullptr));
        return *this;
    }

public:
    float voxel_size_ = 0.05f;
    size_t resolution_ = 512;
    Eigen::Vector3f origin_ = Eigen::Vector3f(0.f, 0.f, 0.f);
    float clamping_thres_min_ = -2.0f;
    float clamping_thres_max_ = 3.5f;
    float prob_hit_log_ = 0.85f;
    float prob_miss_log_ = -0.4f;
    float occ_prob_thres_log_ = 0.0f;
    bool visualize_free_area_ = true;

private:
    friend class DistanceTransform;  // CreateFromOccupancyGrid reads the dense grid
    friend class VoxelGrid;          // and so do VoxelGrid's and PointCloud's
    friend class PointCloud;
    friend struct collision::detail::Operand;  // ComputeIntersection reads it too
    void sync() const {  // the public members are the source of truth, like the reference's
        const float o[3] = {origin_[0], origin_[1], origin_[2]};
        utility::check(cphb_occgrid_set_geometry(h_, voxel_size_, o));
        cphb_occgrid_params p = {clamping_thres_min_, clamping_thres_max_, prob_hit_log_, prob_miss_log_, occ_prob_thres_log_};
        utility::check(cphb_occgrid_set_params(h_, &p));
    }
    std::shared_ptr<std::vector<OccupancyVoxel>> extract(int which) const {
        sync();
        size_t m = 0;
        utility::check(cphb_occgrid_extract(h_, which, nullptr, nullptr, 0, &m, nullptr));
        auto out = std::make_shared<std::vector<OccupancyVoxel>>(m);
        if (!m) return out;
        utility::device_vector<Eigen::Vector3i> idx(m);
        utility::device_vector<float> pr(m);
        utility::check(cphb_occgrid_extract(h_, which, reinterpret_cast<int32_t *>(idx.data()), pr.data(), m, &m, nullptr));
        const auto hi = idx.to_host();
        const auto hp = pr.to_host();
        for (size_t i = 0; i < m; ++i) (*out)[i] = OccupancyVoxel(hi[i], hp[i]);
        return out;
    }
    cphb_occgrid *h_ = nullptr;
};

/// keys = the occupied cells' grid indices (ExtractOccupiedVoxels order), colours (0, 0, 1); origin_ = the grid's origin
/// - (resolution / 2) * voxel_size, so each voxel covers the cell it came from (the reference keeps the grid's origin)
inline std::shared_ptr<VoxelGrid> VoxelGrid::CreateFromOccupancyGrid(const OccupancyGrid &input) {
    auto out = std::make_shared<VoxelGrid>();
    input.sync();
    size_t n = 0;
    float o[3];
    utility::check(cphb_voxel_grid_from_occgrid(input.h_, nullptr, nullptr, 0, &n, o, nullptr));
    out->voxel_size_ = input.voxel_size_;
    out->origin_ = Eigen::Vector3f(o[0], o[1], o[2]);
    out->voxels_keys_.resize(n);
    out->voxels_colors_.resize(n);
    if (n) utility::check(cphb_voxel_grid_from_occgrid(input.h_, out->keys(), out->colors(), n, &n, o, nullptr));
    return out;
}
/// a point per occupied cell at (cell + (float)(-(resolution / 2) + 0.5)) * voxel_size + origin, colour (0, 0, 1)
inline std::shared_ptr<PointCloud> PointCloud::CreateFromOccupancyGrid(const OccupancyGrid &occgrid) {
    auto out = std::make_shared<PointCloud>();
    occgrid.sync();
    size_t n = 0;
    utility::check(cphb_point_cloud_from_occgrid(occgrid.h_, nullptr, nullptr, 0, &n, nullptr));
    out->points_.resize(n);
    out->colors_.resize(n);
    if (n)
        utility::check(cphb_point_cloud_from_occgrid(occgrid.h_, reinterpret_cast<float *>(out->points_.data()),
                                                     reinterpret_cast<float *>(out->colors_.data()), n, &n, nullptr));
    return out;
}

/// geometry::DistanceVoxel (distancetransform.h:30-49)
class DistanceVoxel {
public:
    enum State { HasNext = 1, NotSite = 1 << 1 };
    DistanceVoxel() {}
    DistanceVoxel(const Eigen::Vector3i &nearest_index, unsigned char state) : nearest_index_(nearest_index), state_(state) {}
    bool IsNotSite() const { return state_ & NotSite; }
    bool CheckHasNext() const { return state_ & HasNext; }
    Eigen::Vector3i nearest_index_ = Eigen::Vector3i(0, 0, 0);  // (Vector3ui16 in the reference)
    unsigned char state_ = NotSite;
    float distance_ = 0;
};

/// geometry::DistanceTransform (distancetransform.h:51-78): a dense resolution^3 grid of nearest sites and Euclidean
/// distances.  voxel_size_ and origin_ are public as in the reference and handed to the engine at every call;
/// resolution_ changes only through Reconstruct.  A voxel-size mismatch with the VoxelGrid is logged and leaves the grid
/// unchanged.  Among equidistant sites the lexicographically smallest is the nearest one.
class DistanceTransform {
public:
    DistanceTransform() : DistanceTransform(0.05f, 512) {}
    DistanceTransform(float voxel_size, size_t resolution, const Eigen::Vector3f &origin = Eigen::Vector3f(0.f, 0.f, 0.f))
        : voxel_size_(voxel_size), resolution_(resolution), origin_(origin) {
        const float o[3] = {origin[0], origin[1], origin[2]};
        utility::check(cphb_dt_create(voxel_size, (int)resolution, o, nullptr, &h_));
    }
    ~DistanceTransform() { cphb_stream_synchronize(nullptr); cphb_dt_destroy(h_); }
    DistanceTransform(const DistanceTransform &) = delete;
    DistanceTransform &operator=(const DistanceTransform &) = delete;

    DistanceTransform &Reconstruct(float voxel_size, size_t resolution) {
        utility::check(cphb_dt_reconstruct(h_, voxel_size, (int)resolution, nullptr));
        voxel_size_ = voxel_size;
        resolution_ = resolution;
        return *this;
    }
    DistanceTransform &ComputeEDT(const utility::device_vector<Eigen::Vector3i> &points) { return compute(points, 1); }
    DistanceTransform &ComputeEDT(const VoxelGrid &voxelgrid) { return compute(voxelgrid, 1); }
    DistanceTransform &ComputeVoronoiDiagram(const utility::device_vector<Eigen::Vector3i> &points) { return compute(points, 0); }
    DistanceTransform &ComputeVoronoiDiagram(const VoxelGrid &voxelgrid) { return compute(voxelgrid, 0); }

    float GetDistance(const Eigen::Vector3f &query) const {
        utility::device_vector<Eigen::Vector3f> q(std::vector<Eigen::Vector3f>(1, query));
        return GetDistances(q)->to_host()[0];
    }
    std::unique_ptr<utility::device_vector<float>> GetDistances(const utility::device_vector<Eigen::Vector3f> &queries) const {
        sync();
        auto out = std::make_unique<utility::device_vector<float>>(queries.size());
        if (queries.size())
            utility::check(cphb_dt_get_distances(h_, reinterpret_cast<const float *>(queries.data()), queries.size(), out->data(), nullptr));
        return out;
    }
    std::tuple<bool, DistanceVoxel> GetVoxel(const Eigen::Vector3f &point) const {  // densegrid.inl:148-155
        sync();
        const float p[3] = {point[0], point[1], point[2]};
        int found = 0, state = 0, nb[3];
        float d = 0.f;
        utility::check(cphb_dt_get_voxel(h_, p, &found, nb, &state, &d, nullptr));
        DistanceVoxel v(Eigen::Vector3i(nb[0], nb[1], nb[2]), (unsigned char)state);
        v.distance_ = d;
        return std::make_tuple(found != 0, v);
    }
    /// the reference stamps only the occupied cells; here the EDT of the occupied cells is computed
    static std::shared_ptr<DistanceTransform> CreateFromOccupancyGrid(const OccupancyGrid &input) {
        if (input.voxel_size_ <= 0.0) utility::LogError("[CreateOccupancyGrid] occupancy grid  voxel_size <= 0.");
        input.sync();
        cphb_dt *h = nullptr;
        utility::check(cphb_dt_from_occgrid(input.h_, nullptr, &h));
        return std::shared_ptr<DistanceTransform>(new DistanceTransform(h, input.voxel_size_, input.resolution_, input.origin_));
    }

public:
    float voxel_size_ = 0.05f;
    size_t resolution_ = 512;
    Eigen::Vector3f origin_ = Eigen::Vector3f(0.f, 0.f, 0.f);

private:
    DistanceTransform(cphb_dt *h, float voxel_size, size_t resolution, const Eigen::Vector3f &origin)
        : voxel_size_(voxel_size), resolution_(resolution), origin_(origin), h_(h) {}
    void sync() const {
        const float o[3] = {origin_[0], origin_[1], origin_[2]};
        utility::check(cphb_dt_set_geometry(h_, voxel_size_, o));
    }
    DistanceTransform &compute(const utility::device_vector<Eigen::Vector3i> &points, int with_distance) {
        sync();
        utility::check(cphb_dt_compute_sites(h_, reinterpret_cast<const int32_t *>(points.data()), points.size(), with_distance, nullptr));
        return *this;
    }
    DistanceTransform &compute(const VoxelGrid &vg, int with_distance) {
        sync();
        const float o[3] = {vg.origin_[0], vg.origin_[1], vg.origin_[2]};
        const int rc = cphb_dt_compute_voxel_grid(h_, reinterpret_cast<const int32_t *>(vg.voxels_keys_.data()), vg.voxels_keys_.size(),
                                                  vg.voxel_size_, o, with_distance, nullptr);
        if (rc == CPHB_ERR_INVALID) utility::LogError("Unsupport computing Voronoi diagrams from different voxel size.");
        else utility::check(rc);
        return *this;
    }
    cphb_dt *h_ = nullptr;
};

namespace keypoint {
/// geometry::keypoint::ComputeISSKeypoints (keypoint.h:54-60, iss_keypoints.cu:108-172) -> (the keypoints in ascending
/// index order with their normals and colours, the per-point mask).  salient_radius == 0 or non_max_radius == 0 replaces
/// both from the cloud's resolution.  An empty input, or max_neighbors outside [0, 256], is logged and gives empty results.
inline std::tuple<std::shared_ptr<PointCloud>, std::shared_ptr<utility::device_vector<bool>>> ComputeISSKeypoints(
        const PointCloud &input, float salient_radius = 0.0, float non_max_radius = 0.0, float gamma_21 = 0.975,
        float gamma_32 = 0.975, int min_neighbors = 5, int max_neighbors = knn::NUM_MAX_NN) {
    static_assert(sizeof(bool) == 1, "the mask is written as bytes");
    auto out = std::make_shared<PointCloud>();
    auto mask = std::make_shared<utility::device_vector<bool>>();
    const size_t n = input.points_.size();
    if (n == 0) {
        utility::LogWarning("[ComputeISSKeypoints] Input PointCloud is empty!");
        return std::make_tuple(out, mask);
    }
    if (max_neighbors < 0 || max_neighbors > 256) {
        utility::LogError("[ComputeISSKeypoints] max_neighbors must lie in [0, 256].");
        return std::make_tuple(out, mask);
    }
    mask->resize(n);
    utility::device_vector<int32_t> idx(n);
    size_t m = 0;
    utility::check(cphb_compute_iss_keypoints(reinterpret_cast<const float *>(input.points_.data()), n, salient_radius,
                                              non_max_radius, gamma_21, gamma_32, min_neighbors, max_neighbors,
                                              reinterpret_cast<uint8_t *>(mask->data()), idx.data(), &m, nullptr, nullptr,
                                              nullptr));
    if (m) {  // SelectByMask (down_sample.cu:131-167): points, normals and colours of the masked rows
        const bool hn = input.HasNormals(), hc = input.HasColors();
        out->points_.resize(m);
        if (hn) out->normals_.resize(m);
        if (hc) out->colors_.resize(m);
        utility::check(cphb_select_by_index(
            reinterpret_cast<const float *>(input.points_.data()), hn ? reinterpret_cast<const float *>(input.normals_.data()) : nullptr,
            hc ? reinterpret_cast<const float *>(input.colors_.data()) : nullptr, n, idx.data(), m,
            reinterpret_cast<float *>(out->points_.data()), hn ? reinterpret_cast<float *>(out->normals_.data()) : nullptr,
            hc ? reinterpret_cast<float *>(out->colors_.data()) : nullptr, nullptr));
        utility::check(cphb_stream_synchronize(nullptr));
    }
    return std::make_tuple(out, mask);
}
}  // namespace keypoint
}  // namespace geometry

// --------------------------------------------------------------------------- registration
namespace registration {
typedef utility::device_vector<Eigen::Vector2i> CorrespondenceSet;  // transformation_estimation.h:36

enum class TransformationEstimationType {  // transformation_estimation.h:40-47
    Unspecified = 0, PointToPoint = 1, PointToPlane = 2, SymmetricMethod = 3, ColoredICP = 4, GeneralizedICP = 5,
};

class ICPConvergenceCriteria {  // registration.h:35-49
public:
    ICPConvergenceCriteria(float relative_fitness = 1e-6, float relative_rmse = 1e-6, int max_iteration = 30)
        : relative_fitness_(relative_fitness), relative_rmse_(relative_rmse), max_iteration_(max_iteration) {}
    float relative_fitness_, relative_rmse_;
    int max_iteration_;
};

class RegistrationResult {  // registration.h:51-67
public:
    RegistrationResult(const Eigen::Matrix4f &T = Eigen::Matrix4f::Identity()) : transformation_(T) {}
    std::vector<Eigen::Vector2i> GetCorrespondenceSet() const { return correspondence_set_.to_host(); }
    Eigen::Matrix4f_u transformation_;
    CorrespondenceSet correspondence_set_;
    float inlier_rmse_ = 0.0f;
    float fitness_ = 0.0f;
};

inline cphb_icp_params make_params(int est, float max_dist, const ICPConvergenceCriteria &c, float det_thresh, float lambda) {
    cphb_icp_params p;
    std::memset(&p, 0, sizeof(p));
    p.estimation = est;
    p.max_correspondence_distance = max_dist;
    p.relative_fitness = c.relative_fitness_;
    p.relative_rmse = c.relative_rmse_;
    p.max_iteration = c.max_iteration_;
    p.det_thresh = det_thresh;
    p.lambda_geometric = lambda;
    return p;
}

/// transformation_estimation.h:49-77.  User subclasses (Unspecified) run through the generic loop below.
class TransformationEstimation {
public:
    virtual ~TransformationEstimation() {}
    virtual TransformationEstimationType GetTransformationEstimationType() const = 0;
    virtual float ComputeRMSE(const geometry::PointCloud &source, const geometry::PointCloud &target, const CorrespondenceSet &corres) const = 0;
    virtual Eigen::Matrix4f ComputeTransformation(const geometry::PointCloud &source, const geometry::PointCloud &target, const CorrespondenceSet &corres) const = 0;
    virtual float det_thresh() const { return -1.f; }
    virtual float lambda_geometric() const { return 0.968f; }

protected:
    float rmse_impl(const geometry::PointCloud &s, const geometry::PointCloud &t, const CorrespondenceSet &c) const {
        cphb_cloud sc = s.view(), tc = t.view();
        cphb_icp_params p = make_params((int)GetTransformationEstimationType(), 0.f, ICPConvergenceCriteria(), det_thresh(), lambda_geometric());
        float r = 0.f;
        utility::check(cphb_compute_rmse(p.estimation, &sc, &tc, reinterpret_cast<const int32_t *>(c.data()), c.size(), &p, &r, nullptr));
        return r;
    }
    Eigen::Matrix4f transform_impl(const geometry::PointCloud &s, const geometry::PointCloud &t, const CorrespondenceSet &c) const {
        cphb_cloud sc = s.view(), tc = t.view();
        cphb_icp_params p = make_params((int)GetTransformationEstimationType(), 0.f, ICPConvergenceCriteria(), det_thresh(), lambda_geometric());
        float T[16];
        utility::check(cphb_compute_transformation(p.estimation, &sc, &tc, reinterpret_cast<const int32_t *>(c.data()), c.size(), &p, T, nullptr));
        return utility::from_row_major(T);
    }
};
#define CPHB_FACADE_ESTIMATOR_BODY(TYPE)                                                                        \
    TransformationEstimationType GetTransformationEstimationType() const override { return TransformationEstimationType::TYPE; } \
    float ComputeRMSE(const geometry::PointCloud &s, const geometry::PointCloud &t, const CorrespondenceSet &c) const override { return rmse_impl(s, t, c); } \
    Eigen::Matrix4f ComputeTransformation(const geometry::PointCloud &s, const geometry::PointCloud &t, const CorrespondenceSet &c) const override { return transform_impl(s, t, c); }

class TransformationEstimationPointToPoint : public TransformationEstimation {
public:
    CPHB_FACADE_ESTIMATOR_BODY(PointToPoint)
};
class TransformationEstimationPointToPlane : public TransformationEstimation {
public:
    TransformationEstimationPointToPlane(float det_thresh = 1.0e-6) : det_thresh_(det_thresh) {}
    CPHB_FACADE_ESTIMATOR_BODY(PointToPlane)
    float det_thresh() const override { return det_thresh_; }
    float det_thresh_;
};
class TransformationEstimationSymmetricMethod : public TransformationEstimation {
public:
    TransformationEstimationSymmetricMethod(float det_thresh = 1.0e-6) : det_thresh_(det_thresh) {}
    CPHB_FACADE_ESTIMATOR_BODY(SymmetricMethod)
    float det_thresh() const override { return det_thresh_; }
    float det_thresh_;
};
class TransformationEstimationForGeneralizedICP : public TransformationEstimation {  // generalized_icp.h:14-52
public:
    TransformationEstimationForGeneralizedICP(float epsilon = 1e-3) : epsilon_(epsilon) {}
    CPHB_FACADE_ESTIMATOR_BODY(GeneralizedICP)
    float epsilon_;
};
class TransformationEstimationForColoredICP : public TransformationEstimation {  // colored_icp.cu:42-71
public:
    TransformationEstimationForColoredICP(float lambda_geometric = 0.968, float det_thresh = 1.0e-6)
        : lambda_geometric_(lambda_geometric), det_thresh_(det_thresh) {
        if (lambda_geometric_ < 0 || lambda_geometric_ > 1.0) lambda_geometric_ = 0.968;
    }
    CPHB_FACADE_ESTIMATOR_BODY(ColoredICP)
    float det_thresh() const override { return det_thresh_; }
    float lambda_geometric() const override { return lambda_geometric_; }
    float lambda_geometric_, det_thresh_;
};

inline RegistrationResult to_result(const cphb_icp_result &r, CorrespondenceSet &&corr) {
    RegistrationResult out(utility::from_row_major(r.transformation));
    corr.resize((size_t)r.n_local_correspondences);
    out.correspondence_set_ = std::move(corr);
    out.fitness_ = r.fitness;
    out.inlier_rmse_ = r.inlier_rmse;
    return out;
}

/// registration::EvaluateRegistration (registration.cu:106-119)
inline RegistrationResult EvaluateRegistration(const geometry::PointCloud &source, const geometry::PointCloud &target,
                                               float max_correspondence_distance,
                                               const Eigen::Matrix4f &transformation = Eigen::Matrix4f::Identity()) {
    cphb_cloud sc = source.view(), tc = target.view();
    float T[16];
    utility::to_row_major(transformation, T);
    cphb_icp_result r;
    CorrespondenceSet corr(source.points_.size() ? source.points_.size() : 1);
    utility::check(cphb_evaluate_registration(&sc, &tc, max_correspondence_distance, T, &r, reinterpret_cast<int32_t *>(corr.data()), nullptr));
    return to_result(r, std::move(corr));
}

/// registration::RegistrationICP (registration.cu:121-173).  Built-in estimators run the fused
/// one-launch-per-iteration path; user-defined ones (Unspecified) the generic loop with the
/// caller's virtual ComputeTransformation, exactly as the reference's loop is written.
inline RegistrationResult RegistrationICP(const geometry::PointCloud &source, const geometry::PointCloud &target,
                                          float max_correspondence_distance,
                                          const Eigen::Matrix4f &init = Eigen::Matrix4f::Identity(),
                                          const TransformationEstimation &estimation = TransformationEstimationPointToPoint(),
                                          const ICPConvergenceCriteria &criteria = ICPConvergenceCriteria()) {
    if (max_correspondence_distance <= 0.0) utility::LogError("Invalid max_correspondence_distance.");  // :130-132
    const auto type = estimation.GetTransformationEstimationType();
    if ((type == TransformationEstimationType::PointToPlane || type == TransformationEstimationType::ColoredICP) && !target.HasNormals())
        utility::LogError("TransformationEstimationPointToPlane and TransformationEstimationColoredICP require pre-computed target normal vectors.");
    if (type != TransformationEstimationType::Unspecified) {
        cphb_cloud sc = source.view(), tc = target.view();
        cphb_icp_params p = make_params((int)type, max_correspondence_distance, criteria, estimation.det_thresh(), estimation.lambda_geometric());
        float T[16];
        utility::to_row_major(init, T);
        cphb_icp_result r;
        CorrespondenceSet corr(source.points_.size() ? source.points_.size() : 1);
        utility::check(cphb_registration_icp(&sc, &tc, T, &p, nullptr, &r, reinterpret_cast<int32_t *>(corr.data()), nullptr));
        return to_result(r, std::move(corr));
    }
    // generic loop (registration.cu:145-172) for user-subclassed estimators
    Eigen::Matrix4f transformation = init;
    geometry::PointCloud pcd = source;
    if (!init.isIdentity()) pcd.Transform(init);
    RegistrationResult result = EvaluateRegistration(pcd, target, max_correspondence_distance);
    result.transformation_ = transformation;
    for (int i = 0; i < criteria.max_iteration_; ++i) {
        Eigen::Matrix4f update = estimation.ComputeTransformation(pcd, target, result.correspondence_set_);
        transformation = update * transformation;
        pcd.Transform(update);
        const float bf = result.fitness_, br = result.inlier_rmse_;
        result = EvaluateRegistration(pcd, target, max_correspondence_distance);
        result.transformation_ = transformation;
        if (std::abs(bf - result.fitness_) < criteria.relative_fitness_ && std::abs(br - result.inlier_rmse_) < criteria.relative_rmse_) break;
    }
    return result;
}

/// InitializePointCloudForGeneralizedICP (generalized_icp.cu:37-61)
inline std::shared_ptr<geometry::PointCloud> InitializePointCloudForGeneralizedICP(const geometry::PointCloud &pcd, float epsilon) {
    auto out = std::make_shared<geometry::PointCloud>(pcd);
    if (out->HasCovariances()) return out;
    if (!out->HasNormals()) out->EstimateNormals(knn::KDTreeSearchParamKNN(20));
    out->covariances_.resize(out->points_.size());
    utility::check(cphb_covariances_from_normals(reinterpret_cast<const float *>(out->normals_.data()), out->points_.size(), epsilon,
                                                 reinterpret_cast<float *>(out->covariances_.data()), 1, nullptr));
    return out;
}
/// registration::RegistrationGeneralizedICP (generalized_icp.cu:185-198)
inline RegistrationResult RegistrationGeneralizedICP(const geometry::PointCloud &source, const geometry::PointCloud &target,
                                                     float max_correspondence_distance,
                                                     const Eigen::Matrix4f &init = Eigen::Matrix4f::Identity(),
                                                     const TransformationEstimationForGeneralizedICP &estimation = TransformationEstimationForGeneralizedICP(),
                                                     const ICPConvergenceCriteria &criteria = ICPConvergenceCriteria()) {
    return RegistrationICP(*InitializePointCloudForGeneralizedICP(source, estimation.epsilon_),
                           *InitializePointCloudForGeneralizedICP(target, estimation.epsilon_), max_correspondence_distance,
                           init, estimation, criteria);
}
/// registration::RegistrationColoredICP (colored_icp.cu:329-342)
inline RegistrationResult RegistrationColoredICP(const geometry::PointCloud &source, const geometry::PointCloud &target,
                                                 float max_distance, const Eigen::Matrix4f &init = Eigen::Matrix4f::Identity(),
                                                 const ICPConvergenceCriteria &criteria = ICPConvergenceCriteria(),
                                                 float lambda_geometric = 0.968, float det_thresh = 1.0e-6) {
    geometry::PointCloud target_c = target;  // InitializePointCloudForColoredICP (colored_icp.cu:120-148)
    target_c.color_gradient_.resize(target.points_.size());
    if (target.HasNormals() && target.HasColors())
        utility::check(cphb_color_gradient(reinterpret_cast<const float *>(target_c.points_.data()),
                                           reinterpret_cast<const float *>(target_c.normals_.data()),
                                           reinterpret_cast<const float *>(target_c.colors_.data()), target_c.points_.size(),
                                           max_distance * 2.0f, 30, reinterpret_cast<float *>(target_c.color_gradient_.data()), nullptr));
    else if (!target_c.color_gradient_.empty())
        utility::check(cphb_memset(target_c.color_gradient_.data(), 0, target_c.color_gradient_.size() * 12, nullptr));
    return RegistrationICP(source, target_c, max_distance, init, TransformationEstimationForColoredICP(lambda_geometric, det_thresh), criteria);
}
/// registration::Kabsch (kabsch.h:30-49)
inline Eigen::Matrix4f_u Kabsch(const utility::device_vector<Eigen::Vector3f> &model, const utility::device_vector<Eigen::Vector3f> &target,
                                const CorrespondenceSet &corres) {
    float T[16];
    utility::check(cphb_kabsch(reinterpret_cast<const float *>(model.data()), model.size(), reinterpret_cast<const float *>(target.data()),
                               reinterpret_cast<const int32_t *>(corres.data()), corres.size(), T, nullptr));
    return utility::from_row_major(T);
}
inline Eigen::Matrix4f_u Kabsch(const utility::device_vector<Eigen::Vector3f> &model, const utility::device_vector<Eigen::Vector3f> &target) {
    float T[16];
    utility::check(cphb_kabsch(reinterpret_cast<const float *>(model.data()), model.size(), reinterpret_cast<const float *>(target.data()),
                               nullptr, 0, T, nullptr));
    return utility::from_row_major(T);
}
/// registration::KabschWeighted (kabsch.h:46-49, kabsch.cu:138-201)
inline Eigen::Matrix4f_u KabschWeighted(const utility::device_vector<Eigen::Vector3f> &model,
                                        const utility::device_vector<Eigen::Vector3f> &target, const utility::device_vector<float> &weight) {
    float T[16];
    utility::check(cphb_kabsch_weighted(reinterpret_cast<const float *>(model.data()), reinterpret_cast<const float *>(target.data()),
                                        weight.data(), model.size(), T, nullptr));
    return utility::from_row_major(T);
}
/// registration::Feature<33> (feature.h): one row of 33 floats per point on the device
template <int Dim>
struct Feature {
    utility::device_vector<float> data_;
    size_t num_ = 0;
    void Resize(int n) { num_ = (size_t)n; data_.resize((size_t)n * Dim); }
    size_t Dimension() const { return Dim; }
    size_t Num() const { return num_; }
};
/// registration::ComputeFPFHFeature (feature.h, fpfh.cu:192-229)
inline std::shared_ptr<Feature<33>> ComputeFPFHFeature(const geometry::PointCloud &input,
                                                       const knn::KDTreeSearchParam &search_param = knn::KDTreeSearchParamKNN()) {
    auto feature = std::make_shared<Feature<33>>();
    feature->Resize((int)input.points_.size());
    if (!input.HasNormals()) {
        utility::LogError("[ComputeFPFHFeature] Failed because input point cloud has no normal.");
        return feature;
    }
    int knn = 0, max_nn = 0;
    float radius = 0.f;
    switch (search_param.GetSearchType()) {
        case knn::KDTreeSearchParam::SearchType::Knn: knn = ((const knn::KDTreeSearchParamKNN &)search_param).knn_; break;
        case knn::KDTreeSearchParam::SearchType::Radius:
            radius = ((const knn::KDTreeSearchParamRadius &)search_param).radius_;
            max_nn = ((const knn::KDTreeSearchParamRadius &)search_param).max_nn_;
            break;
        default: utility::LogError("Unsupport search param type."); return feature;
    }
    if (!input.points_.empty())
        utility::check(cphb_compute_fpfh_feature(reinterpret_cast<const float *>(input.points_.data()),
                                                 reinterpret_cast<const float *>(input.normals_.data()), input.points_.size(), knn, radius,
                                                 max_nn, feature->data_.data(), nullptr));
    return feature;
}
/// registration::ComputeSHOTFeature (feature.h:62-66, shot.cu:222-255): one row of 352 floats per point.  `radius` is
/// the descriptor's support, independent of the search.  Missing normals, knn > 100 or max_nn outside [0, 256] are
/// logged and leave the rows unset.
inline std::shared_ptr<Feature<352>> ComputeSHOTFeature(const geometry::PointCloud &input, float radius,
                                                        const knn::KDTreeSearchParam &search_param) {
    auto feature = std::make_shared<Feature<352>>();
    feature->Resize((int)input.points_.size());
    int knn = 0, max_nn = 0;
    float search_radius = 0.f;
    switch (search_param.GetSearchType()) {
        case knn::KDTreeSearchParam::SearchType::Knn: knn = ((const knn::KDTreeSearchParamKNN &)search_param).knn_; break;
        case knn::KDTreeSearchParam::SearchType::Radius:
            search_radius = ((const knn::KDTreeSearchParamRadius &)search_param).radius_;
            max_nn = ((const knn::KDTreeSearchParamRadius &)search_param).max_nn_;
            break;
        default: utility::LogError("Unsupport search param type."); return feature;
    }
    if (input.points_.empty()) return feature;
    if (!input.HasNormals()) {
        utility::LogError("[ComputeSHOTFeature] Failed because input point cloud has no normal.");
        return feature;
    }
    if (knn > knn::NUM_MAX_NN || (knn <= 0 && (max_nn < 0 || max_nn > 256))) {
        utility::LogError("[ComputeSHOTFeature] knn must be <= 100 and max_nn must lie in [0, 256].");
        return feature;
    }
    utility::check(cphb_compute_shot_feature(reinterpret_cast<const float *>(input.points_.data()),
                                             reinterpret_cast<const float *>(input.normals_.data()), input.points_.size(),
                                             radius, knn, search_radius, max_nn, feature->data_.data(), nullptr));
    return feature;
}
}  // namespace registration
// --------------------------------------------------------------------------- collision
namespace collision {

/// collision::Primitive (primitives.h:36-66)
class Primitive {
public:
    enum class PrimitiveType { Unspecified = 0, Box = 1, Sphere = 2, Capsule = 3, Cylinder = 4 };
    Primitive() {}
    Primitive(PrimitiveType type) : type_(type) {}
    Primitive(PrimitiveType type, const Eigen::Matrix4f &transform) : type_(type), transform_(transform) {}
    virtual ~Primitive() {}
    Primitive &Transform(const Eigen::Matrix4f &transform) {  // transform_ = transform_ * transform
        transform_ = transform_ * transform;
        return *this;
    }
    virtual geometry::AxisAlignedBoundingBox<3> GetAxisAlignedBoundingBox() const { return geometry::AxisAlignedBoundingBox<3>(); }
    PrimitiveType type_ = PrimitiveType::Unspecified;
    Eigen::Matrix4f transform_ = Eigen::Matrix4f::Identity();
};

namespace detail {
inline Eigen::Vector3f translation(const Eigen::Matrix4f &T) { return Eigen::Vector3f(T(0, 3), T(1, 3), T(2, 3)); }
}  // namespace detail

/// collision::Box(lengths, transform) (primitives.h:68-88); GetAxisAlignedBoundingBox as written there: +-|R l / 2|
class Box : public Primitive {
public:
    Box() : Primitive(PrimitiveType::Box) {}
    Box(const Eigen::Vector3f &lengths) : Primitive(PrimitiveType::Box), lengths_(lengths) {}
    Box(const Eigen::Vector3f &lengths, const Eigen::Matrix4f &transform) : Primitive(PrimitiveType::Box, transform), lengths_(lengths) {}
    geometry::AxisAlignedBoundingBox<3> GetAxisAlignedBoundingBox() const override {
        float lo[3], hi[3];
        for (int i = 0; i < 3; ++i) {
            float ra = 0.f;
            for (int j = 0; j < 3; ++j) ra += transform_(i, j) * 0.5f * lengths_[j];
            lo[i] = -std::fabs(ra) + transform_(i, 3);
            hi[i] = std::fabs(ra) + transform_(i, 3);
        }
        return geometry::AxisAlignedBoundingBox<3>(Eigen::Vector3f(lo[0], lo[1], lo[2]), Eigen::Vector3f(hi[0], hi[1], hi[2]));
    }
    Eigen::Vector3f lengths_ = Eigen::Vector3f(0.f, 0.f, 0.f);
};

/// collision::Sphere(radius, center) (primitives.h:90-110)
class Sphere : public Primitive {
public:
    Sphere() : Primitive(PrimitiveType::Sphere) {}
    Sphere(float radius) : Primitive(PrimitiveType::Sphere), radius_(radius) {}
    Sphere(float radius, const Eigen::Vector3f &center) : Primitive(PrimitiveType::Sphere), radius_(radius) {
        for (int i = 0; i < 3; ++i) transform_(i, 3) = center[i];
    }
    geometry::AxisAlignedBoundingBox<3> GetAxisAlignedBoundingBox() const override {
        const Eigen::Vector3f c = detail::translation(transform_);
        return geometry::AxisAlignedBoundingBox<3>(Eigen::Vector3f(c[0] - radius_, c[1] - radius_, c[2] - radius_),
                                                   Eigen::Vector3f(c[0] + radius_, c[1] + radius_, c[2] + radius_));
    }
    float radius_ = 0.f;
};

/// collision::Capsule(radius, height, transform) (primitives.h:112-140): the segment of length height along the
/// transform's third column
class Capsule : public Primitive {
public:
    Capsule() : Primitive(PrimitiveType::Capsule) {}
    Capsule(float radius, float height) : Primitive(PrimitiveType::Capsule), radius_(radius), height_(height) {}
    Capsule(float radius, float height, const Eigen::Matrix4f &transform)
        : Primitive(PrimitiveType::Capsule, transform), radius_(radius), height_(height) {}
    geometry::AxisAlignedBoundingBox<3> GetAxisAlignedBoundingBox() const override {
        float lo[3], hi[3];
        for (int i = 0; i < 3; ++i) {
            const float pa = transform_(i, 2) * (0.5f * height_);
            lo[i] = std::min(pa, -pa) - radius_ + transform_(i, 3);
            hi[i] = std::max(pa, -pa) + radius_ + transform_(i, 3);
        }
        return geometry::AxisAlignedBoundingBox<3>(Eigen::Vector3f(lo[0], lo[1], lo[2]), Eigen::Vector3f(hi[0], hi[1], hi[2]));
    }
    float radius_ = 0.f;
    float height_ = 0.f;
};

/// collision::Cylinder(radius, height, transform) (primitives.h:142-185).  It never collides: the reference's collision
/// functors fall to their default branch for it.  GetAxisAlignedBoundingBox as written there (the maximum takes the
/// smaller end).
class Cylinder : public Primitive {
public:
    Cylinder() : Primitive(PrimitiveType::Cylinder) {}
    Cylinder(float radius, float height) : Primitive(PrimitiveType::Cylinder), radius_(radius), height_(height) {}
    Cylinder(float radius, float height, const Eigen::Matrix4f &transform)
        : Primitive(PrimitiveType::Cylinder, transform), radius_(radius), height_(height) {}
    geometry::AxisAlignedBoundingBox<3> GetAxisAlignedBoundingBox() const override {
        float pa[3], a[3], n2 = 0.f, lo[3], hi[3];
        for (int i = 0; i < 3; ++i) {
            pa[i] = transform_(i, 2) * (0.5f * height_);
            a[i] = -pa[i] - pa[i];
            n2 += a[i] * a[i];
        }
        for (int i = 0; i < 3; ++i) {
            const float e = radius_ * std::sqrt(1.f - a[i] * a[i] / n2);
            lo[i] = std::min(pa[i] - e, -pa[i] - e) + transform_(i, 3);
            hi[i] = std::min(pa[i] + e, -pa[i] + e) + transform_(i, 3);
        }
        return geometry::AxisAlignedBoundingBox<3>(Eigen::Vector3f(lo[0], lo[1], lo[2]), Eigen::Vector3f(hi[0], hi[1], hi[2]));
    }
    float radius_ = 0.f;
    float height_ = 0.f;
};

/// collision::PrimitivePack (primitives.h:199-231) and PrimitiveArray: built on the host, uploaded per call
struct PrimitivePack {
    PrimitivePack() {}
    PrimitivePack(const Box &b) : primitive_(b), box_(b) {}
    PrimitivePack(const Sphere &s) : primitive_(s), sphere_(s) {}
    PrimitivePack(const Capsule &c) : primitive_(c), capsule_(c) {}
    PrimitivePack(const Cylinder &c) : primitive_(c), cylinder_(c) {}
    Primitive primitive_;
    Box box_;
    Sphere sphere_;
    Capsule capsule_;
    Cylinder cylinder_;
};
typedef std::vector<PrimitivePack> PrimitiveArray;

/// collision::CollisionResult (collision.h:47-75)
struct CollisionResult {
    enum class CollisionType { Unspecified = 0, Primitives = 1, VoxelGrid = 2, OccupancyGrid = 3 };
    CollisionResult() {}
    CollisionResult(CollisionType first, CollisionType second) : first_(first), second_(second) {}
    bool IsCollided() const { return !collision_index_pairs_.empty(); }
    std::vector<Eigen::Vector2i> GetCollisionIndexPairs() const { return collision_index_pairs_.to_host(); }
    std::vector<size_t> GetFirstCollisionIndices() const { return column(0); }
    std::vector<size_t> GetSecondCollisionIndices() const { return column(1); }
    CollisionType first_ = CollisionType::Unspecified;
    CollisionType second_ = CollisionType::Unspecified;
    utility::device_vector<Eigen::Vector2i> collision_index_pairs_;

private:
    std::vector<size_t> column(int c) const {  // as it is, not deduplicated (host vectors here)
        const std::vector<Eigen::Vector2i> p = GetCollisionIndexPairs();
        std::vector<size_t> out(p.size());
        for (size_t i = 0; i < p.size(); ++i) out[i] = (size_t)p[i][c];
        return out;
    }
};

namespace detail {
struct Operand {
    cphb_coll_operand op{};
    utility::device_vector<cphb_primitive> prims;
    bool empty = false;
    explicit Operand(const geometry::VoxelGrid &g) {
        op.kind = CPHB_COLL_VOXEL_GRID;
        op.keys = reinterpret_cast<const int32_t *>(g.voxels_keys_.data());
        op.n = g.voxels_keys_.size();
        op.voxel_size = g.voxel_size_;
        for (int i = 0; i < 3; ++i) op.origin[i] = g.origin_[i];
        empty = op.n == 0;
    }
    explicit Operand(const geometry::OccupancyGrid &g) {
        g.sync();
        op.kind = CPHB_COLL_OCCUPANCY_GRID;
        op.occ = g.h_;
    }
    explicit Operand(const PrimitiveArray &a) {
        std::vector<cphb_primitive> h(a.size());
        for (size_t i = 0; i < a.size(); ++i) {
            const PrimitivePack &p = a[i];
            cphb_primitive &c = h[i];
            std::memset(&c, 0, sizeof(c));
            c.type = (int32_t)p.primitive_.type_;
            utility::to_row_major(p.primitive_.transform_, c.transform);
            for (int k = 0; k < 3; ++k) c.lengths[k] = p.box_.lengths_[k];
            switch (p.primitive_.type_) {
                case Primitive::PrimitiveType::Sphere: c.radius = p.sphere_.radius_; break;
                case Primitive::PrimitiveType::Capsule: c.radius = p.capsule_.radius_; c.height = p.capsule_.height_; break;
                case Primitive::PrimitiveType::Cylinder: c.radius = p.cylinder_.radius_; c.height = p.cylinder_.height_; break;
                default: break;
            }
        }
        prims = h;
        op.kind = CPHB_COLL_PRIMITIVES;
        op.primitives = prims.data();
        op.n = a.size();
        empty = a.empty();
    }
};

inline std::shared_ptr<CollisionResult> compute(const Operand &a, const Operand &b, float margin) {
    auto out = std::make_shared<CollisionResult>((CollisionResult::CollisionType)a.op.kind, (CollisionResult::CollisionType)b.op.kind);
    // at most one pair per query element: a VoxelGrid or primitive query needs one call, an OccupancyGrid query is sized first
    size_t cap = b.op.kind == CPHB_COLL_OCCUPANCY_GRID ? 0 : b.op.n, m = 0;
    out->collision_index_pairs_.resize(cap);
    int rc = cphb_compute_intersection(&a.op, &b.op, margin, reinterpret_cast<int32_t *>(out->collision_index_pairs_.data()), cap, &m, nullptr);
    if (rc == CPHB_ERR_INVALID) {
        utility::LogError(cphb_last_error());
        out->collision_index_pairs_.resize(0);
        return out;
    }
    utility::check(rc);
    if (a.empty || b.empty) utility::LogWarning("[Intersection::Compute] target or query is empty.");
    if (m && !cap) {
        out->collision_index_pairs_.resize(m);
        utility::check(cphb_compute_intersection(&a.op, &b.op, margin, reinterpret_cast<int32_t *>(out->collision_index_pairs_.data()), m, &m, nullptr));
    }
    out->collision_index_pairs_.resize(m);
    return out;
}
}  // namespace detail

/// collision::ComputeIntersection(a, b, margin) (collision.h:98-146, collision.cu:1137-1231): a is the target, b the query;
/// each colliding query element gives (smallest colliding index in a, index in b), in ascending query order
inline std::shared_ptr<CollisionResult> ComputeIntersection(const geometry::VoxelGrid &voxelgrid1, const geometry::VoxelGrid &voxelgrid2, float margin = 0.0f) {
    return detail::compute(detail::Operand(voxelgrid1), detail::Operand(voxelgrid2), margin);
}
inline std::shared_ptr<CollisionResult> ComputeIntersection(const geometry::VoxelGrid &voxelgrid, const geometry::OccupancyGrid &occgrid, float margin = 0.0f) {
    return detail::compute(detail::Operand(voxelgrid), detail::Operand(occgrid), margin);
}
inline std::shared_ptr<CollisionResult> ComputeIntersection(const geometry::OccupancyGrid &occgrid, const geometry::VoxelGrid &voxelgrid, float margin = 0.0f) {
    return detail::compute(detail::Operand(occgrid), detail::Operand(voxelgrid), margin);
}
inline std::shared_ptr<CollisionResult> ComputeIntersection(const geometry::VoxelGrid &voxelgrid, const PrimitiveArray &primitives, float margin = 0.0f) {
    return detail::compute(detail::Operand(voxelgrid), detail::Operand(primitives), margin);
}
inline std::shared_ptr<CollisionResult> ComputeIntersection(const PrimitiveArray &primitives, const geometry::VoxelGrid &voxelgrid, float margin = 0.0f) {
    return detail::compute(detail::Operand(primitives), detail::Operand(voxelgrid), margin);
}
inline std::shared_ptr<CollisionResult> ComputeIntersection(const geometry::OccupancyGrid &occgrid, const PrimitiveArray &primitives, float margin = 0.0f) {
    return detail::compute(detail::Operand(occgrid), detail::Operand(primitives), margin);
}
inline std::shared_ptr<CollisionResult> ComputeIntersection(const PrimitiveArray &primitives, const geometry::OccupancyGrid &occgrid, float margin = 0.0f) {
    return detail::compute(detail::Operand(primitives), detail::Operand(occgrid), margin);
}
}  // namespace collision

// --------------------------------------------------------------------------- RGBDImage and the TSDF volume
namespace geometry {
/// geometry::RGBDImage (rgbdimage.h): a colour and a depth image of the same size
class RGBDImage {
public:
    RGBDImage() {}
    RGBDImage(const Image &color, const Image &depth) : color_(color), depth_(depth) {}
    bool IsEmpty() const { return depth_.IsEmpty(); }
    /// CreateFromColorAndDepth (rgbdimage_factory.cu:56-72): depth -> float32 metres, raw / int(depth_scale), 0 where it
    /// is >= int(depth_trunc); colour -> float32 weighted intensity when convert_rgb_to_intensity, else kept
    static std::shared_ptr<RGBDImage> CreateFromColorAndDepth(const Image &color, const Image &depth, float depth_scale = 1000.0f,
                                                              float depth_trunc = 3.0f, bool convert_rgb_to_intensity = true) {
        if (color.height_ != depth.height_ || color.width_ != depth.width_)
            throw std::runtime_error("[CreateFromColorAndDepth] Unsupported image format.");
        auto out = std::make_shared<RGBDImage>();
        convert(depth, true, depth_scale, depth_trunc, out->depth_);
        if (convert_rgb_to_intensity)
            convert(color, false, 0.f, 0.f, out->color_);
        else
            out->color_ = color;
        return out;
    }
    static std::shared_ptr<RGBDImage> CreateFromRedwoodFormat(const Image &color, const Image &depth, bool convert_rgb_to_intensity = true) {
        return CreateFromColorAndDepth(color, depth, 1000.0f, 4.0f, convert_rgb_to_intensity);
    }
    static std::shared_ptr<RGBDImage> CreateFromTUMFormat(const Image &color, const Image &depth, bool convert_rgb_to_intensity = true) {
        return CreateFromColorAndDepth(color, depth, 5000.0f, 4.0f, convert_rgb_to_intensity);
    }

public:
    Image color_;
    Image depth_;

private:
    static void convert(const Image &in, bool to_depth, float scale, float trunc, Image &out) {
        out.Prepare(in.width_, in.height_, 1, 4);
        utility::check(cphb_rgbd_convert(in.data_.data(), in.width_, in.height_, in.num_of_channels_, in.bytes_per_channel_, to_depth ? 1 : 0,
                                         scale, trunc, reinterpret_cast<float *>(out.data_.data()), nullptr));
        utility::check(cphb_stream_synchronize(nullptr));
    }
};

namespace detail {
/// cphb_depth_to_points into width / stride x height / stride rows, shrunk to the rows kept
inline std::shared_ptr<PointCloud> depth_to_points(const Image &d, const Image *c, const camera::PinholeCameraIntrinsic &intrinsic,
                                                   const Eigen::Matrix4f &extrinsic, float depth_scale, float depth_trunc, int stride,
                                                   float depth_cutoff, bool normals, bool valid_only) {
    float K[9], E[16];
    for (int r = 0; r < 3; ++r)
        for (int q = 0; q < 3; ++q) K[3 * r + q] = intrinsic.intrinsic_matrix_(r, q);
    utility::to_row_major(extrinsic, E);
    const size_t n = stride >= 1 ? (size_t)std::max(d.width_ / stride, 0) * (size_t)std::max(d.height_ / stride, 0) : 0;
    auto pc = std::make_shared<PointCloud>();
    pc->points_.resize(n);
    if (normals) pc->normals_.resize(n);
    if (c) pc->colors_.resize(n);
    size_t m = 0;
    utility::check(cphb_depth_to_points(d.data_.data(), d.width_, d.height_, d.num_of_channels_, d.bytes_per_channel_, depth_scale, depth_trunc,
                                        stride, c ? c->data_.data() : nullptr, c ? c->width_ : 0, c ? c->height_ : 0,
                                        c ? c->num_of_channels_ : 0, c ? c->bytes_per_channel_ : 0, K, E, depth_cutoff, normals ? 1 : 0,
                                        valid_only ? 1 : 0, (float *)pc->points_.data(), normals ? (float *)pc->normals_.data() : nullptr,
                                        c ? (float *)pc->colors_.data() : nullptr, n, &m, nullptr));
    pc->points_.resize(m);
    if (normals) pc->normals_.resize(m);
    if (c) pc->colors_.resize(m);
    return pc;
}
}  // namespace detail

inline std::shared_ptr<PointCloud> PointCloud::CreateFromDepthImage(const Image &depth, const camera::PinholeCameraIntrinsic &intrinsic,
                                                                    const Eigen::Matrix4f &extrinsic, float depth_scale, float depth_trunc,
                                                                    int stride) {
    return detail::depth_to_points(depth, nullptr, intrinsic, extrinsic, depth_scale, depth_trunc, stride, -1.0f, false, true);
}
inline std::shared_ptr<PointCloud> PointCloud::CreateFromRGBDImage(const RGBDImage &image, const camera::PinholeCameraIntrinsic &intrinsic,
                                                                   const Eigen::Matrix4f &extrinsic, bool project_valid_depth_only,
                                                                   float depth_cutoff, bool compute_normals) {
    if (image.depth_.num_of_channels_ != 1 || image.depth_.bytes_per_channel_ != 4)
        throw std::runtime_error("[PointCloud::CreateFromRGBDImage] the depth image must be 1-channel float32");
    return detail::depth_to_points(image.depth_, &image.color_, intrinsic, extrinsic, 1000.0f, 1000.0f, 1, depth_cutoff, compute_normals,
                                   project_valid_depth_only);
}
}  // namespace geometry

namespace geometry {
/// geometry::MeshBase (meshbase.h): only what TriangleMesh's filters need, FilterScope, so that both
/// MeshBase::FilterScope and TriangleMesh::FilterScope name it.
class MeshBase {
public:
    enum class FilterScope { All, Color, Normal, Vertex };
    virtual ~MeshBase() {}
};

/// geometry::TriangleMesh (trianglemesh.h, meshbase.h): vertices_, vertex_normals_, vertex_colors_, triangles_ (int32
/// vertex indices), triangle_normals_ and edge_list_ on the device.  The two normal computations, ComputeEdgeList,
/// the four vertex filters, GetSurfaceArea, SamplePointsUniformly, GetMinBound / GetMaxBound, the four Remove*
/// cleanup operations, GetSelfIntersectingTriangles and + / += are provided (no IO or primitives).
class TriangleMesh : public MeshBase {
public:
    TriangleMesh() {}
    TriangleMesh(const utility::device_vector<Eigen::Vector3f> &vertices, const utility::device_vector<Eigen::Vector3i> &triangles)
        : vertices_(vertices), triangles_(triangles) {}
    TriangleMesh(const std::vector<Eigen::Vector3f> &vertices, const std::vector<Eigen::Vector3i> &triangles)
        : vertices_(vertices), triangles_(triangles) {}

    bool IsEmpty() const { return !HasVertices(); }
    bool HasVertices() const { return vertices_.size() > 0; }
    bool HasVertexNormals() const { return HasVertices() && vertex_normals_.size() == vertices_.size(); }
    bool HasVertexColors() const { return HasVertices() && vertex_colors_.size() == vertices_.size(); }
    bool HasTriangles() const { return HasVertices() && triangles_.size() > 0; }
    bool HasTriangleNormals() const { return HasTriangles() && triangle_normals_.size() == triangles_.size(); }

    /// ComputeTriangleNormals (trianglemesh.cu:466-477): (v1 - v0) x (v2 - v0), normalised when asked.  A vertex index
    /// outside [0, vertices_.size()) throws.
    TriangleMesh &ComputeTriangleNormals(bool normalized = true) {
        triangle_normals_.resize(triangles_.size());
        if (triangles_.size())
            utility::check(cphb_mesh_triangle_normals((const float *)vertices_.data(), vertices_.size(), (const int32_t *)triangles_.data(),
                                                      triangles_.size(), normalized ? 1 : 0, (float *)triangle_normals_.data(), nullptr));
        return *this;
    }
    /// ComputeVertexNormals (trianglemesh.cu:479-503): the unnormalised triangle normals first when there are none; each
    /// vertex's normal is the sum of its triangles' normals in ascending triangle order, normalised when asked.  A vertex
    /// in no triangle gets a zero normal, so vertex_normals_ stays aligned with vertices_.
    TriangleMesh &ComputeVertexNormals(bool normalized = true) {
        if (!HasTriangleNormals()) ComputeTriangleNormals(false);
        vertex_normals_.resize(vertices_.size());
        if (vertices_.size() || triangles_.size())
            utility::check(cphb_mesh_vertex_normals((const int32_t *)triangles_.data(), triangles_.size(), (const float *)triangle_normals_.data(),
                                                    vertices_.size(), normalized ? 1 : 0, (float *)vertex_normals_.data(), nullptr));
        return *this;
    }

    /// MeshBase::GetMinBound / GetMaxBound: the smallest / largest coordinate of all vertices per axis, (0, 0, 0)
    /// without vertices
    Eigen::Vector3f GetMinBound() const { return Bound(0); }
    Eigen::Vector3f GetMaxBound() const { return Bound(1); }

    bool HasEdgeList() const { return edge_list_.size() > 0; }
    /// ComputeEdgeList (trianglemesh.cu:505-519): the directed edges (a, b) and (b, a) of every triangle edge, sorted and
    /// unique.  A vertex index outside [0, vertices_.size()) throws.
    TriangleMesh &ComputeEdgeList() {
        utility::device_vector<Eigen::Vector2i> buf(6 * triangles_.size());
        size_t n = 0;
        utility::check(cphb_mesh_edge_list((const int32_t *)triangles_.data(), triangles_.size(), vertices_.size(), (int32_t *)buf.data(),
                                           buf.size(), &n, nullptr));
        edge_list_.resize(n);
        if (n) {
            utility::check(cphb_memcpy_d2d(edge_list_.data(), buf.data(), n * sizeof(Eigen::Vector2i), nullptr));
            utility::check(cphb_stream_synchronize(nullptr));
        }
        return *this;
    }
    /// FilterSharpen (trianglemesh.cu:521-599): per iteration v + strength (v N - sum of the N neighbours)
    std::shared_ptr<TriangleMesh> FilterSharpen(int number_of_iterations, float strength, FilterScope scope = FilterScope::All) const {
        return Filter(CPHB_MESH_SHARPEN, number_of_iterations, strength, 0.f, scope);
    }
    /// FilterSmoothSimple (trianglemesh.cu:601-679): per iteration (v + sum of the N neighbours) / (1 + N)
    std::shared_ptr<TriangleMesh> FilterSmoothSimple(int number_of_iterations, FilterScope scope = FilterScope::All) const {
        return Filter(CPHB_MESH_SIMPLE, number_of_iterations, 0.f, 0.f, scope);
    }
    /// FilterSmoothLaplacian (trianglemesh.cu:681-735): per iteration v + lambda (sum w v_nb / sum w - v), w = 1 / (|v -
    /// v_nb| + 1e-12) from the input vertices
    std::shared_ptr<TriangleMesh> FilterSmoothLaplacian(int number_of_iterations, float lambda, FilterScope scope = FilterScope::All) const {
        return Filter(CPHB_MESH_LAPLACIAN, number_of_iterations, lambda, 0.f, scope);
    }
    /// FilterSmoothTaubin (trianglemesh.cu:737-800): per iteration a Laplacian step with lambda, then one with mu
    std::shared_ptr<TriangleMesh> FilterSmoothTaubin(int number_of_iterations, float lambda = 0.5f, float mu = -0.53f,
                                                     FilterScope scope = FilterScope::All) const {
        return Filter(CPHB_MESH_TAUBIN, number_of_iterations, lambda, mu, scope);
    }
    /// GetSurfaceArea (trianglemesh.cu:802-828): the float64 fixed-order sum of 0.5 |(p0 - p1) x (p0 - p2)|, as float
    float GetSurfaceArea() const { return SurfaceArea(nullptr); }
    float GetSurfaceArea(utility::device_vector<float> &triangle_areas) const {
        triangle_areas.resize(triangles_.size());
        return SurfaceArea(triangle_areas.data());
    }
    /// SamplePointsUniformly (trianglemesh.cu:830-901): exactly number_of_points points; with use_triangle_normal the
    /// normalised triangle normals are computed and kept when the mesh has none.  number_of_points 0 or above 2^30 - 1,
    /// no triangles, or a surface area that is not positive and finite throws.
    std::shared_ptr<PointCloud> SamplePointsUniformly(size_t number_of_points, bool use_triangle_normal = false) {
        if (number_of_points == 0) throw std::runtime_error("[SamplePointsUniformly] number_of_points <= 0");
        if (triangles_.size() == 0) throw std::runtime_error("input mesh has no triangles");
        if (use_triangle_normal && !HasTriangleNormals()) ComputeTriangleNormals(true);
        const bool vn = HasVertexNormals(), vc = HasVertexColors();
        auto pc = std::make_shared<PointCloud>();
        pc->points_.resize(number_of_points);
        if (vn || use_triangle_normal) pc->normals_.resize(number_of_points);
        if (vc) pc->colors_.resize(number_of_points);
        utility::check(cphb_mesh_sample_points_uniformly(
            (const float *)vertices_.data(), vertices_.size(), (const int32_t *)triangles_.data(), triangles_.size(),
            vn ? (const float *)vertex_normals_.data() : nullptr, use_triangle_normal ? (const float *)triangle_normals_.data() : nullptr,
            vc ? (const float *)vertex_colors_.data() : nullptr, number_of_points, (float *)pc->points_.data(),
            (vn || use_triangle_normal) ? (float *)pc->normals_.data() : nullptr, vc ? (float *)pc->colors_.data() : nullptr, nullptr));
        return pc;
    }

    /// RemoveDuplicatedVertices (trianglemesh.cu:903-969): the distinct positions (IEEE ==, so -0 and +0 are one) in
    /// lexicographic (x, y, z) order, each keeping the normal and colour of its lowest original index; triangles are
    /// remapped.  A vertex with a NaN coordinate merges with nothing and goes last.  The edge list is recomputed when
    /// the mesh has one.  A vertex index outside [0, vertices_.size()) throws and changes nothing.
    TriangleMesh &RemoveDuplicatedVertices() {
        VertexPass(cphb_mesh_remove_duplicated_vertices);
        if (HasEdgeList()) ComputeEdgeList();
        return *this;
    }
    /// RemoveDuplicatedTriangles (trianglemesh.cu:971-1009): each triangle rotated so its smallest index is first
    /// (orientation kept), sorted, the first of each run kept with its normal; the edge list is recomputed when
    /// triangles were removed
    TriangleMesh &RemoveDuplicatedTriangles() {
        if (TrianglePass(cphb_mesh_remove_duplicated_triangles) && HasEdgeList()) ComputeEdgeList();
        return *this;
    }
    /// RemoveUnreferencedVertices (trianglemesh.cu:1011-1080): the vertices some triangle uses, in order, with their
    /// normals and colours; triangles are remapped; the edge list is recomputed when vertices were removed
    TriangleMesh &RemoveUnreferencedVertices() {
        if (VertexPass(cphb_mesh_remove_unreferenced_vertices) && HasEdgeList()) ComputeEdgeList();
        return *this;
    }
    /// RemoveDegenerateTriangles (trianglemesh.cu:1082-1121): drops, in order, the triangles with two equal indices;
    /// the edge list is recomputed when triangles were removed
    TriangleMesh &RemoveDegenerateTriangles() {
        if (TrianglePass(cphb_mesh_remove_degenerate_triangles) && HasEdgeList()) ComputeEdgeList();
        return *this;
    }
    /// GetSelfIntersectingTriangles (trianglemesh.cu:1123-1141): the pairs i < j, ascending, that share no vertex index,
    /// have only finite vertices and overlapping closed boxes, and that TriangleTriangle3d says intersect
    utility::device_vector<Eigen::Vector2i> GetSelfIntersectingTriangles() const {
        const float *v = (const float *)vertices_.data();
        const int32_t *t = (const int32_t *)triangles_.data();
        size_t n = 0;
        utility::check(cphb_mesh_self_intersecting_triangles(v, vertices_.size(), t, triangles_.size(), nullptr, 0, &n, nullptr, nullptr));
        utility::device_vector<Eigen::Vector2i> out(n);
        if (n)
            utility::check(cphb_mesh_self_intersecting_triangles(v, vertices_.size(), t, triangles_.size(), (int32_t *)out.data(), n, &n,
                                                                 nullptr, nullptr));
        return out;
    }
    /// operator+= (trianglemesh.cu:411-452, meshbase.cu:124-151): other's vertices appended and its triangles shifted by
    /// the old vertex count.  Vertex normals, vertex colours and triangle normals survive when other has them and this
    /// mesh has them or has no vertices (triangles); the edge list is recomputed when this mesh had one.  An empty
    /// other changes nothing; a vertex index outside its mesh's range throws and changes nothing.
    TriangleMesh &operator+=(const TriangleMesh &other) {
        if (other.IsEmpty()) return *this;
        const size_t na = vertices_.size(), nb = other.vertices_.size(), ta = triangles_.size(), tb = other.triangles_.size();
        utility::device_vector<Eigen::Vector3i> tri(ta + tb);
        utility::check(cphb_mesh_append_triangles((const int32_t *)triangles_.data(), ta, na, (const int32_t *)other.triangles_.data(), tb, nb,
                                                  (int32_t *)tri.data(), nullptr));
        const bool vn = (na == 0 || HasVertexNormals()) && other.HasVertexNormals();
        const bool vc = (na == 0 || HasVertexColors()) && other.HasVertexColors();
        const bool tn = (ta == 0 || HasTriangleNormals()) && other.HasTriangleNormals();
        Append(vertex_normals_, na, other.vertex_normals_, vn);
        Append(vertex_colors_, na, other.vertex_colors_, vc);
        Append(triangle_normals_, ta, other.triangle_normals_, tn);
        Append(vertices_, na, other.vertices_, true);
        triangles_ = std::move(tri);
        if (HasEdgeList()) ComputeEdgeList();
        return *this;
    }
    TriangleMesh operator+(const TriangleMesh &other) const { return TriangleMesh(*this) += other; }

public:
    utility::device_vector<Eigen::Vector3f> vertices_;
    utility::device_vector<Eigen::Vector3f> vertex_normals_;
    utility::device_vector<Eigen::Vector3f> vertex_colors_;
    utility::device_vector<Eigen::Vector3i> triangles_;
    utility::device_vector<Eigen::Vector3f> triangle_normals_;
    utility::device_vector<Eigen::Vector2i> edge_list_;

private:
    typedef int (*VertexPassFn)(const float *, const float *, const float *, size_t, const int32_t *, size_t, float *, float *, float *,
                                int32_t *, size_t *, void *);
    typedef int (*TrianglePassFn)(const int32_t *, const float *, size_t, size_t, int32_t *, float *, size_t *, void *);
    // the two vertex removals' common path -> whether vertices were removed
    bool VertexPass(VertexPassFn fn) {
        const size_t n = vertices_.size(), m = triangles_.size();
        const bool vn = HasVertexNormals(), vc = HasVertexColors();
        utility::device_vector<Eigen::Vector3f> ov(n), on(vn ? n : 0), oc(vc ? n : 0);
        utility::device_vector<Eigen::Vector3i> ot(m);
        size_t k = 0;
        utility::check(fn((const float *)vertices_.data(), vn ? (const float *)vertex_normals_.data() : nullptr,
                          vc ? (const float *)vertex_colors_.data() : nullptr, n, (const int32_t *)triangles_.data(), m, (float *)ov.data(),
                          vn ? (float *)on.data() : nullptr, vc ? (float *)oc.data() : nullptr, (int32_t *)ot.data(), &k, nullptr));
        if (n) {
            ov.resize(k);
            vertices_ = std::move(ov);
            if (vn) on.resize(k), vertex_normals_ = std::move(on);
            if (vc) oc.resize(k), vertex_colors_ = std::move(oc);
        }
        if (m) triangles_ = std::move(ot);
        return k < n;
    }
    // the two triangle removals' common path -> whether triangles were removed
    bool TrianglePass(TrianglePassFn fn) {
        const size_t m = triangles_.size();
        if (m == 0) return false;
        const bool tn = HasTriangleNormals();
        utility::device_vector<Eigen::Vector3i> ot(m);
        utility::device_vector<Eigen::Vector3f> otn(tn ? m : 0);
        size_t k = 0;
        utility::check(fn((const int32_t *)triangles_.data(), tn ? (const float *)triangle_normals_.data() : nullptr, m, vertices_.size(),
                          (int32_t *)ot.data(), tn ? (float *)otn.data() : nullptr, &k, nullptr));
        ot.resize(k);
        triangles_ = std::move(ot);
        if (tn) otn.resize(k), triangle_normals_ = std::move(otn);
        return k < m;
    }
    // a += b for one attribute when keep, else a is cleared
    template <class T>
    static void Append(utility::device_vector<T> &a, size_t na, const utility::device_vector<T> &b, bool keep) {
        if (!keep) {
            a.clear();
            return;
        }
        a.resize(na + b.size());
        if (b.size()) {
            utility::check(cphb_memcpy_d2d(a.data() + na, b.data(), b.size() * sizeof(T), nullptr));
            utility::check(cphb_stream_synchronize(nullptr));
        }
    }
    // the filters' common path: a new mesh with the triangles, the edge list (this mesh's own when it has one, checked
    // for range and order) and every vertex attribute, filtered or copied; triangle normals are not carried
    std::shared_ptr<TriangleMesh> Filter(int kind, int iterations, float c0, float c1, FilterScope scope) const {
        auto mesh = std::make_shared<TriangleMesh>();
        mesh->triangles_ = triangles_;
        mesh->vertices_.resize(vertices_.size());
        mesh->edge_list_ = edge_list_;
        if (!mesh->HasEdgeList()) mesh->ComputeEdgeList();
        const int mask = scope == FilterScope::All ? 7 : scope == FilterScope::Vertex ? 1 : scope == FilterScope::Normal ? 2 : 4;
        const bool vn = HasVertexNormals(), vc = HasVertexColors();
        if (vn) mesh->vertex_normals_.resize(vertices_.size());
        if (vc) mesh->vertex_colors_.resize(vertices_.size());
        utility::check(cphb_mesh_filter(kind, iterations, c0, c1, (const int32_t *)mesh->edge_list_.data(), mesh->edge_list_.size(),
                                        vertices_.size(), (const float *)vertices_.data(), vn ? (const float *)vertex_normals_.data() : nullptr,
                                        vc ? (const float *)vertex_colors_.data() : nullptr, mask, (float *)mesh->vertices_.data(),
                                        vn ? (float *)mesh->vertex_normals_.data() : nullptr, vc ? (float *)mesh->vertex_colors_.data() : nullptr,
                                        nullptr));
        return mesh;
    }
    Eigen::Vector3f Bound(int which) const {
        float mn[3] = {0, 0, 0}, mx[3] = {0, 0, 0};
        if (vertices_.size()) utility::check(cphb_min_max_bound((const float *)vertices_.data(), vertices_.size(), mn, mx, nullptr));
        return which ? Eigen::Vector3f(mx[0], mx[1], mx[2]) : Eigen::Vector3f(mn[0], mn[1], mn[2]);
    }
    float SurfaceArea(float *areas) const {
        float a = 0.f;
        if (triangles_.size())
            utility::check(cphb_mesh_surface_area((const float *)vertices_.data(), vertices_.size(), (const int32_t *)triangles_.data(),
                                                  triangles_.size(), areas, &a, nullptr));
        return a;
    }
};

inline std::shared_ptr<VoxelGrid> VoxelGrid::CreateFromTriangleMeshWithinBounds(const TriangleMesh &input, float voxel_size,
                                                                                const Eigen::Vector3f &min_bound,
                                                                                const Eigen::Vector3f &max_bound) {
    auto out = std::make_shared<VoxelGrid>();
    out->voxel_size_ = voxel_size;
    out->origin_ = min_bound;
    const float mn[3] = {min_bound[0], min_bound[1], min_bound[2]}, mx[3] = {max_bound[0], max_bound[1], max_bound[2]};
    const float *v = (const float *)input.vertices_.data();
    const int32_t *t = (const int32_t *)input.triangles_.data();
    const size_t nv = input.vertices_.size(), nt = input.triangles_.size();
    size_t n = 0;
    utility::check(cphb_voxel_grid_from_triangle_mesh(v, nv, t, nt, voxel_size, mn, mx, nullptr, nullptr, 0, &n, nullptr));
    out->voxels_keys_.resize(n);
    out->voxels_colors_.resize(n);
    if (n) utility::check(cphb_voxel_grid_from_triangle_mesh(v, nv, t, nt, voxel_size, mn, mx, out->keys(), out->colors(), n, &n, nullptr));
    return out;
}
inline std::shared_ptr<VoxelGrid> VoxelGrid::CreateFromTriangleMesh(const TriangleMesh &input, float voxel_size) {
    const Eigen::Vector3f lo = input.GetMinBound(), hi = input.GetMaxBound();
    const float h = voxel_size * 0.5f;
    return CreateFromTriangleMeshWithinBounds(input, voxel_size, Eigen::Vector3f(lo[0] - h, lo[1] - h, lo[2] - h),
                                              Eigen::Vector3f(hi[0] + h, hi[1] + h, hi[2] + h));
}
}  // namespace geometry

namespace integration {
/// integration::TSDFVolumeColorType (tsdfvolume.h)
enum class TSDFVolumeColorType { NoColor = 0, RGB8 = 1, Gray32 = 2 };

/// integration::TSDFVolume (tsdfvolume.h): the members the reference's base class holds
class TSDFVolume {
public:
    TSDFVolume(float voxel_length, float sdf_trunc, TSDFVolumeColorType color_type)
        : voxel_length_(voxel_length), sdf_trunc_(sdf_trunc), color_type_(color_type) {}
    virtual ~TSDFVolume() {}
    /// the surface as a welded triangle mesh (tsdfvolume.h:68)
    virtual std::shared_ptr<geometry::TriangleMesh> ExtractTriangleMesh() = 0;

public:
    float voxel_length_;
    float sdf_trunc_;
    TSDFVolumeColorType color_type_;
};

/// integration::UniformTSDFVolume (uniform_tsdfvolume.h): a dense resolution^3 grid owned by a cphb_tsdf handle.
/// Reset restores the initial voxels; a resolution outside [2, 1290] or a length or sdf_trunc that is not positive and
/// finite throws.  Not copyable (the grid stays on the device).
class UniformTSDFVolume : public TSDFVolume {
public:
    UniformTSDFVolume(float length, int resolution, float sdf_trunc, TSDFVolumeColorType color_type,
                      const Eigen::Vector3f &origin = Eigen::Vector3f(0.f, 0.f, 0.f))
        : TSDFVolume(length / (float)resolution, sdf_trunc, color_type), origin_(origin), length_(length), resolution_(resolution),
          voxel_num_((size_t)(resolution > 0 ? resolution : 0) * (resolution > 0 ? resolution : 0) * (resolution > 0 ? resolution : 0)) {
        const float o[3] = {origin[0], origin[1], origin[2]};
        utility::check(cphb_tsdf_create(length, resolution, sdf_trunc, (int)color_type, o, nullptr, &h_));
    }
    UniformTSDFVolume(const UniformTSDFVolume &) = delete;
    UniformTSDFVolume &operator=(const UniformTSDFVolume &) = delete;
    ~UniformTSDFVolume() override {
        if (h_) {
            cphb_stream_synchronize(nullptr);
            cphb_tsdf_destroy(h_);
        }
    }
    void Reset() {
        utility::check(cphb_tsdf_reset(h_, nullptr));
        utility::check(cphb_stream_synchronize(nullptr));
    }
    /// Integrate (uniform_tsdfvolume.cu:670-701); extrinsic is world-to-camera
    void Integrate(const geometry::RGBDImage &image, const camera::PinholeCameraIntrinsic &intrinsic, const Eigen::Matrix4f &extrinsic) {
        float K[9], E[16];
        intrinsic9(intrinsic, K);
        utility::to_row_major(extrinsic, E);
        const geometry::Image &d = image.depth_, &c = image.color_;
        utility::check(cphb_tsdf_integrate(h_, reinterpret_cast<const float *>(d.data_.data()), d.width_, d.height_, d.num_of_channels_,
                                           d.bytes_per_channel_, c.data_.data(), c.width_, c.height_, c.num_of_channels_,
                                           c.bytes_per_channel_, intrinsic.width_, intrinsic.height_, K, E, nullptr));
        utility::check(cphb_stream_synchronize(nullptr));
    }
    /// ExtractPointCloud (uniform_tsdfvolume.cu:703-737): points, normals and (with colour) colours of the crossings
    std::shared_ptr<geometry::PointCloud> ExtractPointCloud() {
        auto pc = std::make_shared<geometry::PointCloud>();
        size_t n = 0;
        utility::check(cphb_tsdf_extract_points(h_, nullptr, nullptr, nullptr, 0, &n, nullptr));
        if (n) {
            pc->points_.resize(n);
            pc->normals_.resize(n);
            if (color_type_ != TSDFVolumeColorType::NoColor) pc->colors_.resize(n);
            utility::check(cphb_tsdf_extract_points(h_, (float *)pc->points_.data(), (float *)pc->normals_.data(),
                                                    color_type_ != TSDFVolumeColorType::NoColor ? (float *)pc->colors_.data() : nullptr,
                                                    n, &n, nullptr));
        }
        return pc;
    }
    /// ExtractTriangleMesh (uniform_tsdfvolume.cu:739-838), welded: one vertex per crossed grid edge of a valid cube,
    /// coloured unless NoColor; triangles cube by cube, their right-hand normals pointing from negative to positive tsdf
    std::shared_ptr<geometry::TriangleMesh> ExtractTriangleMesh() override {
        auto mesh = std::make_shared<geometry::TriangleMesh>();
        const bool has_c = color_type_ != TSDFVolumeColorType::NoColor;
        size_t nv = 0, nt = 0;
        utility::check(cphb_tsdf_extract_mesh(h_, nullptr, nullptr, nullptr, 0, 0, &nv, &nt, nullptr));
        if (nv) {
            mesh->vertices_.resize(nv);
            if (has_c) mesh->vertex_colors_.resize(nv);
            mesh->triangles_.resize(nt);
            utility::check(cphb_tsdf_extract_mesh(h_, (float *)mesh->vertices_.data(), has_c ? (float *)mesh->vertex_colors_.data() : nullptr,
                                                  (int32_t *)mesh->triangles_.data(), nv, nt, &nv, &nt, nullptr));
        }
        return mesh;
    }
    /// ExtractVoxelPointCloud (uniform_tsdfvolume.cu:840-865): band voxel centres coloured (tsdf + 1) / 2
    std::shared_ptr<geometry::PointCloud> ExtractVoxelPointCloud() const {
        auto pc = std::make_shared<geometry::PointCloud>();
        size_t n = 0;
        utility::check(cphb_tsdf_extract_voxels(h_, nullptr, nullptr, nullptr, 0, &n, nullptr));
        if (n) {
            pc->points_.resize(n);
            pc->colors_.resize(n);
            utility::check(cphb_tsdf_extract_voxels(h_, nullptr, (float *)pc->points_.data(), (float *)pc->colors_.data(), n, &n, nullptr));
        }
        return pc;
    }
    /// ExtractVoxelGrid (uniform_tsdfvolume.cu:867-895): band voxels, origin = origin - (resolution / 2) * voxel_length
    std::shared_ptr<geometry::VoxelGrid> ExtractVoxelGrid() const {
        auto vg = std::make_shared<geometry::VoxelGrid>();
        vg->voxel_size_ = voxel_length_;
        const float half = (float)(resolution_ / 2) * voxel_length_;
        vg->origin_ = Eigen::Vector3f(origin_[0] - half, origin_[1] - half, origin_[2] - half);
        size_t n = 0;
        utility::check(cphb_tsdf_extract_voxels(h_, nullptr, nullptr, nullptr, 0, &n, nullptr));
        if (n) {
            vg->voxels_keys_.resize(n);
            vg->voxels_colors_.resize(n);
            utility::check(cphb_tsdf_extract_voxels(h_, (int32_t *)vg->voxels_keys_.data(), nullptr, (float *)vg->voxels_colors_.data(), n, &n,
                                                    nullptr));
        }
        return vg;
    }
    /// Raycast (uniform_tsdfvolume.cu:924-951): one ray per pixel from the camera at extrinsic (world-to-camera)
    std::shared_ptr<geometry::PointCloud> Raycast(const camera::PinholeCameraIntrinsic &intrinsic, const Eigen::Matrix4f &extrinsic,
                                                  float sdf_trunc, bool project_valid_depth_only = true) const {
        float K[9], E[16];
        intrinsic9(intrinsic, K);
        utility::to_row_major(extrinsic, E);
        const size_t npx = (size_t)std::max(intrinsic.width_, 0) * (size_t)std::max(intrinsic.height_, 0);
        utility::device_vector<Eigen::Vector3f> p(npx), nr(npx), c(npx);
        size_t n = 0;
        utility::check(cphb_tsdf_raycast(h_, intrinsic.width_, intrinsic.height_, K, E, sdf_trunc, project_valid_depth_only ? 1 : 0,
                                         (float *)p.data(), (float *)nr.data(), (float *)c.data(), npx, &n, nullptr));
        auto pc = std::make_shared<geometry::PointCloud>();
        pc->points_.resize(n);
        pc->normals_.resize(n);
        pc->colors_.resize(n);
        if (n) {
            utility::check(cphb_memcpy_d2d(pc->points_.data(), p.data(), 12 * n, nullptr));
            utility::check(cphb_memcpy_d2d(pc->normals_.data(), nr.data(), 12 * n, nullptr));
            utility::check(cphb_memcpy_d2d(pc->colors_.data(), c.data(), 12 * n, nullptr));
            utility::check(cphb_stream_synchronize(nullptr));
        }
        return pc;
    }

public:
    Eigen::Vector3f origin_;
    float length_;
    int resolution_;
    size_t voxel_num_;

private:
    static void intrinsic9(const camera::PinholeCameraIntrinsic &in, float K[9]) {
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) K[3 * r + c] = in.intrinsic_matrix_(r, c);
    }
    cphb_tsdf *h_ = nullptr;
};

/// integration::ScalableTSDFVolume (scalable_tsdfvolume.h): 16^3-voxel units allocated on the device near observed
/// surfaces, owned by a cphb_stsdf handle.  map_size is the first capacity of the unit pool, which doubles as needed.
/// Argument errors, a rejected frame (which leaves the volume unchanged) and ExtractTriangleMesh (not implemented, as
/// in the reference) throw.  Not copyable.
class ScalableTSDFVolume : public TSDFVolume {
public:
    ScalableTSDFVolume(float voxel_length, float sdf_trunc, TSDFVolumeColorType color_type, int depth_sampling_stride = 4,
                       int map_size = 1000)
        : TSDFVolume(voxel_length, sdf_trunc, color_type), volume_unit_length_(voxel_length * 16.0f),
          depth_sampling_stride_(depth_sampling_stride) {
        utility::check(cphb_stsdf_create(voxel_length, sdf_trunc, (int)color_type, depth_sampling_stride, map_size, nullptr, &h_));
    }
    ScalableTSDFVolume(const ScalableTSDFVolume &) = delete;
    ScalableTSDFVolume &operator=(const ScalableTSDFVolume &) = delete;
    ~ScalableTSDFVolume() override {
        if (h_) {
            cphb_stream_synchronize(nullptr);
            cphb_stsdf_destroy(h_);
        }
    }
    void Reset() {
        utility::check(cphb_stsdf_reset(h_, nullptr));
        utility::check(cphb_stream_synchronize(nullptr));
    }
    /// Integrate (scalable_tsdfvolume.cu:311-343); extrinsic is world-to-camera
    void Integrate(const geometry::RGBDImage &image, const camera::PinholeCameraIntrinsic &intrinsic, const Eigen::Matrix4f &extrinsic) {
        float K[9], E[16];
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) K[3 * r + c] = intrinsic.intrinsic_matrix_(r, c);
        utility::to_row_major(extrinsic, E);
        const geometry::Image &d = image.depth_, &c = image.color_;
        utility::check(cphb_stsdf_integrate(h_, reinterpret_cast<const float *>(d.data_.data()), d.width_, d.height_, d.num_of_channels_,
                                            d.bytes_per_channel_, c.data_.data(), c.width_, c.height_, c.num_of_channels_,
                                            c.bytes_per_channel_, intrinsic.width_, intrinsic.height_, K, E, nullptr));
    }
    /// ExtractPointCloud (scalable_tsdfvolume.cu:345-366): points, normals and (with colour) colours of the crossings
    std::shared_ptr<geometry::PointCloud> ExtractPointCloud() {
        auto pc = std::make_shared<geometry::PointCloud>();
        const bool has_c = color_type_ != TSDFVolumeColorType::NoColor;
        size_t n = 0;
        utility::check(cphb_stsdf_extract_points(h_, nullptr, nullptr, nullptr, 0, &n, nullptr));
        if (n) {
            pc->points_.resize(n);
            pc->normals_.resize(n);
            if (has_c) pc->colors_.resize(n);
            utility::check(cphb_stsdf_extract_points(h_, (float *)pc->points_.data(), (float *)pc->normals_.data(),
                                                     has_c ? (float *)pc->colors_.data() : nullptr, n, &n, nullptr));
        }
        return pc;
    }
    /// ExtractVoxelPointCloud: band voxel centres coloured (tsdf + 1) / 2
    std::shared_ptr<geometry::PointCloud> ExtractVoxelPointCloud() const {
        auto pc = std::make_shared<geometry::PointCloud>();
        size_t n = 0;
        utility::check(cphb_stsdf_extract_voxels(h_, nullptr, nullptr, 0, &n, nullptr));
        if (n) {
            pc->points_.resize(n);
            pc->colors_.resize(n);
            utility::check(cphb_stsdf_extract_voxels(h_, (float *)pc->points_.data(), (float *)pc->colors_.data(), n, &n, nullptr));
        }
        return pc;
    }
    /// not implemented, as in the reference (scalable_tsdfvolume.cu:375-381)
    std::shared_ptr<geometry::TriangleMesh> ExtractTriangleMesh() override {
        throw std::runtime_error("ScalableTSDFVolume::ExtractTriangleMesh is not implemented");
    }
    /// the number of allocated units
    size_t UnitCount() const {
        size_t u = 0, cap = 0, bytes = 0;
        utility::check(cphb_stsdf_info(h_, &u, &cap, &bytes));
        return u;
    }

public:
    float volume_unit_length_;
    int depth_sampling_stride_;

private:
    cphb_stsdf *h_ = nullptr;
};
}  // namespace integration
}  // namespace cupoch
