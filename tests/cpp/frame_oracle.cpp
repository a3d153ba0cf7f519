// frame_oracle.cpp -- TEST INFRASTRUCTURE: the CPU checker of the cut-frame preprocess (Preprocess::process_cut_frame_livox /
// process_cut_frame_pcl2, src/preprocess.cpp:50-335), restated literally and sequentially: the same loops, the same float / double
// mix, std::stable_sort for the sort, the per-ring loop of the constant-rotation model. It shares no code with the product.
// Built with -ffp-contract=off (no FMA contraction, as the reference's x86-64 build).
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <type_traits>
#include <vector>

using namespace std;

namespace {

struct Pt {   // the PointType fields the cut uses; PointXYZINormal() zero-initialises them
    float x = 0.f, y = 0.f, z = 0.f, intensity = 0.f, curvature = 0.f;
};

template <class T>
T rd(const uint8_t* p) {
    T v;
    memcpy(&v, p, sizeof(T));
    return v;
}

// `abs` and `atan2` of floats under `using namespace std` resolve to the float overloads, as in preprocess.cpp
static_assert(is_same<decltype(abs(float())), float>::value, "abs(float) is the float overload");
static_assert(is_same<decltype(atan2(float(), float())), float>::value, "atan2(float, float) is the float overload");

struct Out {
    float* pts;      // [cap_pts][5]: x, y, z, intensity, curvature
    int cap_pts;
    int* sub_n;
    double* sub_tbeg;
    float* sub_end;
    int cap_sub;
    int n_sub = 0, n_pts = 0;
};

// preprocess.cpp:84-112 / 304-334 on pl_surf
int cut(vector<Pt>& pl_surf, double stamp, int required_frame_num, int scan_count, int threshold, Out& o) {
    stable_sort(pl_surf.begin(), pl_surf.end(), [](const Pt& a, const Pt& b) { return a.curvature < b.curvature; });
    double last_frame_end_time = stamp * 1000;
    unsigned valid_num = 0;
    unsigned cut_num = 0;
    unsigned valid_pcl_size = pl_surf.size();
    int required_cut_num = required_frame_num;
    if (scan_count < threshold) required_cut_num = 1;
    vector<Pt> pcl_cut;
    for (unsigned i = 1; i < valid_pcl_size; i++) {
        valid_num++;
        pl_surf[i].curvature += stamp * 1000 - last_frame_end_time;
        pcl_cut.push_back(pl_surf[i]);
        if (valid_num == (int((cut_num + 1) * valid_pcl_size / required_cut_num) - 1)) {
            cut_num++;
            if (o.n_sub >= o.cap_sub || o.n_pts + (int)pcl_cut.size() > o.cap_pts) return -3;
            o.sub_tbeg[o.n_sub] = last_frame_end_time / double(1000);   // time_buffer (laserMapping.cpp:334)
            o.sub_end[o.n_sub] = pcl_cut.back().curvature;
            o.sub_n[o.n_sub] = (int)pcl_cut.size();
            for (const Pt& p : pcl_cut) {
                float* q = o.pts + 5 * (size_t)o.n_pts++;
                q[0] = p.x; q[1] = p.y; q[2] = p.z; q[3] = p.intensity; q[4] = p.curvature;
            }
            o.n_sub++;
            last_frame_end_time += pl_surf[i].curvature;
            pcl_cut.clear();
        }
    }
    return 0;
}

}  // namespace

extern "C" {

// Livox CustomMsg records {u32 offset_time; f32 x, y, z; u8 reflectivity, tag, line}, `stride` bytes apart.
int frame_oracle_livox(const uint8_t* msg, int stride, int plsize, int N_SCANS, double blind, int point_filter_num, int required_frame_num,
                       int scan_count, double stamp, float* pts, int cap_pts, int* sub_n, double* sub_tbeg, float* sub_end, int cap_sub,
                       int* n_sub, int* n_pts) {
    vector<Pt> pl_surf, pl_full(plsize);
    int valid_point_num = 0;
    for (unsigned i = 1; i < (unsigned)plsize; i++) {
        const uint8_t* r = msg + (size_t)i * stride;
        const uint8_t tag = r[17], line = r[18];
        if ((line < N_SCANS) && ((tag & 0x30) == 0x10 || (tag & 0x30) == 0x00)) {
            valid_point_num++;
            if (valid_point_num % point_filter_num == 0) {
                pl_full[i].x = rd<float>(r + 4);
                pl_full[i].y = rd<float>(r + 8);
                pl_full[i].z = rd<float>(r + 12);
                pl_full[i].intensity = r[16];
                pl_full[i].curvature = rd<uint32_t>(r) / float(1000000);
                double dist = pl_full[i].x * pl_full[i].x + pl_full[i].y * pl_full[i].y + pl_full[i].z * pl_full[i].z;
                if (dist < blind * blind) continue;
                if ((abs(pl_full[i].x - pl_full[i - 1].x) > 1e-7) || (abs(pl_full[i].y - pl_full[i - 1].y) > 1e-7) ||
                    (abs(pl_full[i].z - pl_full[i - 1].z) > 1e-7)) {
                    pl_surf.push_back(pl_full[i]);
                }
            }
        }
    }
    Out o{pts, cap_pts, sub_n, sub_tbeg, sub_end, cap_sub};
    int r = cut(pl_surf, stamp, required_frame_num, scan_count, 5, o);
    *n_sub = o.n_sub;
    *n_pts = o.n_pts;
    return r;
}

// PointCloud2 data of lidar_type 2 (Velodyne), 3 (Ouster), 5 (Pandar), 6 (Robosense). offs: byte offsets of x, y, z, intensity,
// time, ring (-1: absent, reads 0). Returns -1 when the rotation model meets a ring >= 128 (the reference's arrays overrun).
int frame_oracle_pcl2(const uint8_t* data, int point_step, const int* offs, int lidar_type, int plsize, int N_SCANS, double blind,
                      int point_filter_num, int required_frame_num, int scan_count, double stamp, float* pts, int cap_pts, int* sub_n,
                      double* sub_tbeg, float* sub_end, int cap_sub, int* n_sub, int* n_pts) {
    *n_sub = *n_pts = 0;
    if (plsize == 0) return 0;
    struct Raw {
        float x, y, z, fintensity;
        uint8_t u8intensity;
        float ftime;
        uint32_t utime;
        double dtime;
        unsigned ring;
    };
    vector<Raw> pl_orig(plsize);
    for (int i = 0; i < plsize; i++) {   // fromROSMsg
        const uint8_t* r = data + (size_t)i * point_step;
        Raw& p = pl_orig[i];
        memset(&p, 0, sizeof(p));
        if (offs[0] >= 0) p.x = rd<float>(r + offs[0]);
        if (offs[1] >= 0) p.y = rd<float>(r + offs[1]);
        if (offs[2] >= 0) p.z = rd<float>(r + offs[2]);
        if (offs[3] >= 0) {
            if (lidar_type == 6) p.u8intensity = r[offs[3]];
            else p.fintensity = rd<float>(r + offs[3]);
        }
        if (offs[4] >= 0) {
            if (lidar_type == 2) p.ftime = rd<float>(r + offs[4]);
            else if (lidar_type == 3) p.utime = rd<uint32_t>(r + offs[4]);
            else p.dtime = rd<double>(r + offs[4]);
        }
        if (offs[5] >= 0) p.ring = lidar_type == 3 ? r[offs[5]] : rd<uint16_t>(r + offs[5]);
    }
    const bool rotation = lidar_type == 2 || lidar_type == 6;
    bool given_offset_time = true;
    bool is_first[128];
    double yaw_fp[128] = {0};
    double omega_l = 3.61;
    float yaw_last[128] = {0.0};
    float time_last[128] = {0.0};
    if (rotation) {
        const bool pos = lidar_type == 2 ? pl_orig[plsize - 1].ftime > 0 : pl_orig[plsize - 1].dtime > 0;
        if (!pos) {
            given_offset_time = false;
            memset(is_first, true, sizeof(is_first));
        }
    }
    vector<Pt> pl_surf;
    for (int i = 0; i < plsize; i++) {
        const Raw& o = pl_orig[i];
        Pt added_pt;
        added_pt.x = o.x;
        added_pt.y = o.y;
        added_pt.z = o.z;
        added_pt.intensity = lidar_type == 6 ? o.u8intensity : o.fintensity;
        if (lidar_type == 2) added_pt.curvature = o.ftime * 1000.0;
        else if (lidar_type == 3) added_pt.curvature = o.utime / 1e6;
        else if (lidar_type == 5) added_pt.curvature = (o.dtime - pl_orig[0].dtime) * 1000;
        else added_pt.curvature = (o.dtime - stamp + 0.1) * 1000.0;
        double dist = added_pt.x * added_pt.x + added_pt.y * added_pt.y + added_pt.z * added_pt.z;
        if (dist < blind * blind || isnan(added_pt.x) || isnan(added_pt.y) || isnan(added_pt.z)) continue;
        if (!given_offset_time) {
            int layer = o.ring;
            if (layer >= 128) return -1;
            double yaw_angle = atan2(added_pt.y, added_pt.x) * 57.2957;
            if (is_first[layer]) {
                yaw_fp[layer] = yaw_angle;
                is_first[layer] = false;
                added_pt.curvature = 0.0;
                yaw_last[layer] = yaw_angle;
                time_last[layer] = added_pt.curvature;
                continue;
            }
            if (yaw_angle <= yaw_fp[layer]) {
                added_pt.curvature = (yaw_fp[layer] - yaw_angle) / omega_l;
            } else {
                added_pt.curvature = (yaw_fp[layer] - yaw_angle + 360.0) / omega_l;
            }
            if (added_pt.curvature < time_last[layer]) added_pt.curvature += 360.0 / omega_l;
            yaw_last[layer] = yaw_angle;
            time_last[layer] = added_pt.curvature;
        }
        if (i % point_filter_num == 0 && (int)o.ring < N_SCANS) pl_surf.push_back(added_pt);
    }
    (void)yaw_last;
    Out out{pts, cap_pts, sub_n, sub_tbeg, sub_end, cap_sub};
    int r = cut(pl_surf, stamp, required_frame_num, scan_count, 20, out);
    *n_sub = out.n_sub;
    *n_pts = out.n_pts;
    return r;
}

}  // extern "C"
