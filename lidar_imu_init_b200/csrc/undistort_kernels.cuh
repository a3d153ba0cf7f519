// undistort_kernels.cuh -- per-point motion compensation on the device (SURVEY.md section 8f row N3).
//
// Replaces the two back-propagation loops of src/IMU_Processing.hpp:
//   * constant-velocity model without IMU, Forward_propagation_without_imu :246-266 (LO mode; bias_g holds the angular
//     velocity): P' = Exp(omega, -dt_j) P_j - (rot_end^T vel_end) dt_j,  dt_j = t_end - t_j;
//   * IMU model, propagation_and_undist :390-415: every point is carried from the IMU pose that precedes it to the scan-end
//     frame, P' = R_LI^T ( rot_end^T ( R_i (R_LI p + T_LI) + P_i - pos_end ) - T_LI ),
//     R_i = R_head Exp(gyr_head, dt), P_i = pos_head + vel_head dt + 0.5 acc_head dt^2, dt = t_j - t_head.
// The reference walks the time-sorted cloud backwards; per point the result only depends on the point's own time stamp
// (PointType.curvature, milliseconds), so one thread per point needs no sort. Loop quirks kept: the CV loop never touches
// the earliest point (`it_pcl != begin`), the IMU loop leaves points with t_j <= t_head0 untouched and never uses the last
// pose of the table as head. All arithmetic in double, float store, as the reference.
#pragma once
#include "common.cuh"

// so3_math.h:39-59  Exp(ang_vel, dt)
__device__ __forceinline__ void li_so3_exp_dt(const double w[3], double dt, double R[9]) {
    const double n = sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
    R[0] = R[4] = R[8] = 1.0;
    R[1] = R[2] = R[3] = R[5] = R[6] = R[7] = 0.0;
    if (n > 0.0000001) {
        const double r0 = w[0] / n, r1 = w[1] / n, r2 = w[2] / n;
        const double a = n * dt;
        const double s = sin(a), c = 1.0 - cos(a);
        // K = [r]x ; R = I + s K + c K K
        const double K[9] = {0.0, -r2, r1, r2, 0.0, -r0, -r1, r0, 0.0};
        double KK[9];
#pragma unroll
        for (int i = 0; i < 3; i++)
#pragma unroll
            for (int j = 0; j < 3; j++) KK[3 * i + j] = K[3 * i] * K[j] + K[3 * i + 1] * K[3 + j] + K[3 * i + 2] * K[6 + j];
#pragma unroll
        for (int i = 0; i < 9; i++) R[i] = R[i] + s * K[i] + c * KK[i];
    }
}

struct CvParams {
    double omega[3];    // state.bias_g (angular velocity in the CV model)
    double vb[3];       // rot_end^T * vel_end
};

// pts.w = time offset in milliseconds (PointType.curvature). tmax / tmin_idx: results of k_time_range.
__global__ void k_undistort_cv(float4* __restrict__ pts, int n, CvParams P, const int* __restrict__ tmax,
                               const unsigned long long* __restrict__ tmin_idx) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (i == (int)(unsigned)(*tmin_idx & 0xffffffffull)) return;   // the earliest point is never reached by the reference loop (:250)
    int o = *tmax;
    const float t_last = __int_as_float(o >= 0 ? o : o ^ 0x7fffffff);
    const double t_end = (double)t_last / 1000.0;                  // pcl_end_offset_time (:212)
    float4 p = pts[i];
    const double dt_j = t_end - (double)p.w / 1000.0;
    double R[9];
    li_so3_exp_dt(P.omega, -dt_j, R);
    const double x = p.x, y = p.y, z = p.z;
    const double cx = R[0] * x + R[1] * y + R[2] * z + (-P.vb[0] * dt_j);
    const double cy = R[3] * x + R[4] * y + R[5] * z + (-P.vb[1] * dt_j);
    const double cz = R[6] * x + R[7] * y + R[8] * z + (-P.vb[2] * dt_j);
    pts[i] = make_float4((float)cx, (float)cy, (float)cz, p.w);
}

// Pose6D (msg/Pose6D.msg; common_lib.h:184-199), flat: offset_time, acc[3], gyr[3], vel[3], pos[3], rot[9] = 22 doubles
#define LI_POSE6D_DOUBLES 22

// the head pose of a point at time t [s]: the last pose k <= npose-2 with offset_time < t (-1: none)
__device__ __forceinline__ int li_imu_head(const double* __restrict__ poses, int npose, double t) {
    int head = -1;
    for (int k = 0; k <= npose - 2; k++)
        if (t > poses[(size_t)k * LI_POSE6D_DOUBLES]) head = k;
    return head;
}

// the point (x, y, z) at time t [s] carried from the head pose h to the scan-end frame of S (rot_end, pos_end, R_LI, T_LI); shared by
// k_undistort_imu and the timed assessment (assess_time_kernels.cuh), so both round alike
__device__ __forceinline__ float3 li_undistort_imu_point(const double* __restrict__ h, double t, const PoseD& S, float px, float py, float pz) {
    const double dt = t - h[0];
    double E[9], Ri[9];
    li_so3_exp_dt(h + 4, dt, E);
    const double* Rh = h + 13;
#pragma unroll
    for (int a = 0; a < 3; a++)
#pragma unroll
        for (int b = 0; b < 3; b++) Ri[3 * a + b] = Rh[3 * a] * E[b] + Rh[3 * a + 1] * E[3 + b] + Rh[3 * a + 2] * E[6 + b];
    double Pi[3];
#pragma unroll
    for (int a = 0; a < 3; a++) Pi[a] = h[10 + a] + h[7 + a] * dt + 0.5 * h[1 + a] * dt * dt;
    const double x = px, y = py, z = pz;
    double q[3], u[3], v[3], w[3];
#pragma unroll
    for (int a = 0; a < 3; a++) q[a] = S.RLI[3 * a] * x + S.RLI[3 * a + 1] * y + S.RLI[3 * a + 2] * z + S.TLI[a];
#pragma unroll
    for (int a = 0; a < 3; a++) u[a] = Ri[3 * a] * q[0] + Ri[3 * a + 1] * q[1] + Ri[3 * a + 2] * q[2] + Pi[a] - S.p[a];
#pragma unroll
    for (int a = 0; a < 3; a++) v[a] = S.R[a] * u[0] + S.R[3 + a] * u[1] + S.R[6 + a] * u[2] - S.TLI[a];   // rot_end^T u - T_LI
#pragma unroll
    for (int a = 0; a < 3; a++) w[a] = S.RLI[a] * v[0] + S.RLI[3 + a] * v[1] + S.RLI[6 + a] * v[2];        // R_LI^T v
    return make_float3((float)w[0], (float)w[1], (float)w[2]);
}

__global__ void k_undistort_imu(float4* __restrict__ pts, int n, const double* __restrict__ poses, int npose, PoseD S) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float4 p = pts[i];
    const double t = (double)p.w / 1000.0;
    const int head = li_imu_head(poses, npose, t);
    if (head < 0) return;
    const float3 w = li_undistort_imu_point(poses + (size_t)head * LI_POSE6D_DOUBLES, t, S, p.x, p.y, p.z);
    pts[i] = make_float4(w.x, w.y, w.z, p.w);
}

// pointBodyToWorld (laserMapping.cpp:209-220) over the staged cloud, one thread per point, packed xyz out in upload order
// (publish_frame_world / pcd_save on feats_undistort, :560-603).
__global__ void k_raw_to_world(const float4* __restrict__ pts, int n, PoseD P, float* __restrict__ out) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 p = pts[i];
    float wx, wy, wz;
    li_body_to_world(P, p.x, p.y, p.z, wx, wy, wz);
    out[3 * (size_t)i] = wx;
    out[3 * (size_t)i + 1] = wy;
    out[3 * (size_t)i + 2] = wz;
}

// time range of the staged cloud: min time + its first index, max time (ordered-int atomics on non-negative floats)
__global__ void k_time_range(const float4* __restrict__ pts, int n, unsigned long long* __restrict__ tmin_idx, int* __restrict__ tmax) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float t = pts[i].w;
    int o = __float_as_int(t);
    o = o >= 0 ? o : o ^ 0x7fffffff;
    atomicMax(tmax, o);
    unsigned long long key = ((unsigned long long)(unsigned)(o ^ 0x80000000) << 32) | (unsigned)i;   // (time, index) ascending
    atomicMin(tmin_idx, key);
}
