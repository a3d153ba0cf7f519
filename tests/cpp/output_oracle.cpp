// output_oracle.cpp -- TEST INFRASTRUCTURE ONLY: the CPU checker of the node's published clouds, restated from the reference's
// description (src/laserMapping.cpp:209-220 pointBodyToWorld, :561-636 publish_frame_world / publish_frame_body / publish_effect_world,
// :1013-1020 and :1050-1051 laserCloudOri) and PCL's VoxelGrid<PointXYZINormal> with downsample_all_data_ (the default). Shares no
// code with the product. Build: g++ -O3 -ffp-contract=off (no FMA contraction, like the reference's x86-64 build).
//
// Records are PointType (pcl::PointXYZINormal) as 12 floats: x y z data[3] | normal_x normal_y normal_z data_n[3] | intensity
// curvature data_c[2] data_c[3].
#include <algorithm>
#include <cmath>
#include <cstring>
#include <limits>
#include <vector>

namespace {

struct PointType {
    float x = 0.f, y = 0.f, z = 0.f, d3 = 1.f;                 // PointXYZINormal(): data[3] = 1
    float normal_x = 0.f, normal_y = 0.f, normal_z = 0.f, dn3 = 0.f;
    float intensity = 0.f, curvature = 0.f, dc2 = 0.f, dc3 = 0.f;
};
static_assert(sizeof(PointType) == 48, "PointType is 48 bytes");

struct State {
    double R[9], p[3], RLI[9], TLI[3];
};

PointType load(const float* r) {
    PointType q;
    memcpy(&q, r, sizeof(q));
    return q;
}

// pointBodyToWorld: p_global = rot_end * (offset_R_L_I * p_body + offset_T_L_I) + pos_end, each matrix-vector product as Eigen
// evaluates it for a 3x3 times 3-vector (row by row, left to right), no contraction
void pointBodyToWorld(const State& s, const PointType* pi, PointType* po) {
    const double b[3] = {pi->x, pi->y, pi->z};
    double t[3], g[3];
    for (int r = 0; r < 3; r++) t[r] = s.RLI[3 * r] * b[0] + s.RLI[3 * r + 1] * b[1] + s.RLI[3 * r + 2] * b[2] + s.TLI[r];
    for (int r = 0; r < 3; r++) g[r] = s.R[3 * r] * t[0] + s.R[3 * r + 1] * t[1] + s.R[3 * r + 2] * t[2] + s.p[r];
    po->x = (float)g[0];
    po->y = (float)g[1];
    po->z = (float)g[2];
    po->normal_x = pi->normal_x;
    po->normal_y = pi->normal_y;
    po->normal_z = pi->normal_z;
    po->intensity = pi->intensity;
}

State state_of(const double* R, const double* p, const double* RLI, const double* TLI) {
    State s;
    memcpy(s.R, R, sizeof(s.R));
    memcpy(s.p, p, sizeof(s.p));
    memcpy(s.RLI, RLI, sizeof(s.RLI));
    memcpy(s.TLI, TLI, sizeof(s.TLI));
    return s;
}

}  // namespace

extern "C" {

// publish_frame_world: PointCloudXYZI(size, 1) filled by pointBodyToWorld
void oo_to_world(const float* in12, int n, const double* R, const double* p, const double* RLI, const double* TLI, float* out12) {
    const State s = state_of(R, p, RLI, TLI);
    for (int i = 0; i < n; i++) {
        const PointType a = load(in12 + 12 * (size_t)i);
        PointType w;
        pointBodyToWorld(s, &a, &w);
        memcpy(out12 + 12 * (size_t)i, &w, sizeof(w));
    }
}

// publish_frame_body: feats_undistort as it is (the padding of a PointType made by the preprocess: data[3] = 1, the rest 0)
void oo_frame_body(const float* in12, int n, float* out12) {
    for (int i = 0; i < n; i++) {
        const PointType a = load(in12 + 12 * (size_t)i);
        PointType b;
        b.x = a.x; b.y = a.y; b.z = a.z;
        b.normal_x = a.normal_x; b.normal_y = a.normal_y; b.normal_z = a.normal_z;
        b.intensity = a.intensity; b.curvature = a.curvature;
        memcpy(out12 + 12 * (size_t)i, &b, sizeof(b));
    }
}

// VoxelGrid<PointXYZINormal>::applyFilter with downsample_all_data_: bounding box of the finite points, leaf index of every finite
// point, stable sort by leaf index, per leaf the input-order float sum of every field divided by the count. Returns the number of
// leaves (out12 must hold n records), -1 when the grid overflows int32.
int oo_voxel_grid(const float* in12, int n, float leaf, float* out12) {
    const float inv = 1.0f / leaf;
    float mn[3] = {std::numeric_limits<float>::max(), std::numeric_limits<float>::max(), std::numeric_limits<float>::max()};
    float mx[3] = {-std::numeric_limits<float>::max(), -std::numeric_limits<float>::max(), -std::numeric_limits<float>::max()};
    std::vector<PointType> P(n);
    for (int i = 0; i < n; i++) P[i] = load(in12 + 12 * (size_t)i);
    auto finite = [](const PointType& q) { return std::isfinite(q.x) && std::isfinite(q.y) && std::isfinite(q.z); };
    int nf = 0;
    for (int i = 0; i < n; i++) {
        if (!finite(P[i])) continue;
        nf++;
        const float v[3] = {P[i].x, P[i].y, P[i].z};
        for (int a = 0; a < 3; a++) { mn[a] = std::min(mn[a], v[a]); mx[a] = std::max(mx[a], v[a]); }
    }
    if (nf == 0) return 0;
    long long minb[3], div[3];
    for (int a = 0; a < 3; a++) {
        minb[a] = (long long)std::floor(mn[a] * inv);
        const long long maxb = (long long)std::floor(mx[a] * inv);
        div[a] = maxb - minb[a] + 1;
    }
    if (div[0] * div[1] * div[2] > std::numeric_limits<int>::max()) return -1;
    const int mul1 = (int)div[0], mul2 = (int)(div[0] * div[1]);
    std::vector<std::pair<unsigned, int>> idx;
    for (int i = 0; i < n; i++) {
        if (!finite(P[i])) continue;
        const int i0 = (int)(std::floor(P[i].x * inv) - (float)minb[0]);
        const int i1 = (int)(std::floor(P[i].y * inv) - (float)minb[1]);
        const int i2 = (int)(std::floor(P[i].z * inv) - (float)minb[2]);
        idx.emplace_back((unsigned)(i0 + i1 * mul1 + i2 * mul2), i);
    }
    std::stable_sort(idx.begin(), idx.end(), [](const std::pair<unsigned, int>& a, const std::pair<unsigned, int>& b) { return a.first < b.first; });
    int m = 0;
    for (size_t f = 0; f < idx.size();) {
        size_t l = f;
        float sx = 0.f, sy = 0.f, sz = 0.f, snx = 0.f, sny = 0.f, snz = 0.f, si = 0.f;
        while (l < idx.size() && idx[l].first == idx[f].first) {
            const PointType& q = P[idx[l].second];
            sx += q.x; sy += q.y; sz += q.z;
            snx += q.normal_x; sny += q.normal_y; snz += q.normal_z;
            si += q.intensity;
            l++;
        }
        const float c = (float)(l - f);
        PointType o;
        o.x = sx / c; o.y = sy / c; o.z = sz / c;
        o.normal_x = snx / c; o.normal_y = sny / c; o.normal_z = snz / c;
        o.intensity = si / c;
        memcpy(out12 + 12 * (size_t)m, &o, sizeof(o));
        m++;
        f = l;
    }
    return m;
}

// publish_effect_world: laserCloudOri = the selected points of feats_down_body in index order (:1013-1020), intensity sqrt(R_inv)
// with R_inv = 1000 (:1050-1051), then pointBodyToWorld into PointCloudXYZI(effect_feat_num, 1). Returns effect_feat_num.
int oo_effect(const float* down12, const unsigned char* selected, int n, const double* R, const double* p, const double* RLI, const double* TLI,
              float* out12) {
    const State s = state_of(R, p, RLI, TLI);
    int k = 0;
    for (int i = 0; i < n; i++) {
        if (!selected[i]) continue;
        PointType ori = load(down12 + 12 * (size_t)i);
        const double R_inv = 1000;
        ori.intensity = (float)std::sqrt(R_inv);
        PointType w;
        pointBodyToWorld(s, &ori, &w);
        memcpy(out12 + 12 * (size_t)k, &w, sizeof(w));
        k++;
    }
    return k;
}

}  // extern "C"
